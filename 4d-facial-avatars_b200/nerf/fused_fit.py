"""Fused fitting step (DESIGN.md 8d): a FROZEN avatar (both networks fixed) fitted to photos by optimising each frame's camera
pose, expression and latent code — what the drop-in loop of tools/fit_bench.py does with get_ray_bundle + run_one_iter_of_nerf +
torch MSE + loss.backward() + torch.optim.Adam — as kernel launches of libnfb over K images per step, with no autograd graph and
no torch.optim, capturable as one CUDA graph:

    sample rays of K images (1) -> fold K frames (1) -> multi-frame training forward (1) -> loss gradient (1)
    -> input-only multi-frame backward (ray, expression and latent gradients only; no parameter gradient)
    -> pose / expression rows (nfb_fit_rows_grad) -> latent rows + regulariser (nfb_latent_rows_grad) -> Adam per fitted table

The parameters are three tables in ONE flat FP32 bucket, [poses N x 12 | expressions N x 76 | latents N x 32] (each padded to
64 floats); gradients and Adam's moments are buckets of the same layout.  The sampler reads the pose and expression tables and
the latent table IN PLACE (ray_sampler.TrainImages.alias_tables), so every step and every replay draws rays from the current
estimates.  torch is used for memory and the noise draws (in the reference's order)."""
import torch

from . import _capi as capi
from . import _engine
from . import ray_sampler
from .fused_train import _capture, _check_epoch, _draw_noise, _image_buffers

TABLES = ("pose", "expression", "latent")
_WIDTH = dict(pose=12, expression=76, latent=32)


def _pad(n):
    return (n + 63) // 64 * 64


class FusedFitter:
    """Fit per-image pose, expression and latent of a frozen avatar to images.

    model_coarse / model_fine: the avatar's networks (never changed; model_fine may be None).  images [N,H,W,3] (device, or host
    memory that is pinned and read in place), bboxs (N boxes of the importance maps), intrinsics [fx, fy, cx, cy]: the training
    set as ray_sampler.TrainImages takes it.  poses [N,12] / [N,3,4] / [N,4,4] camera-to-world, expressions [N,76], latents
    [N,32]: the initial estimates, copied into the fit bucket.  background: optional [H,W,3].
    fit: which tables are optimised, any non-empty subset of ("pose", "expression", "latent"); the others stay bitwise
    unchanged.  lr_pose / lr_expression / lr_latent: each table's constant Adam learning rate (defaults 1e-4, 1e-4 and 1e-4:
    tools/fit_bench.py's 1e-4 for pose and expression, and the same for the latent code).  betas, eps: Adam's.  latent_reg:
    weight of the latent regulariser (latent_reg / K) * sum_k ||latent[image_index[k]]|| (default 0.005 = the reference's
    10 * 0.0005); only when the latent table is fitted.  Render options as FusedTrainer's (precision None: the module's mode).

    The step is torch.optim.Adam with three parameter groups, one per fitted table, each table one leaf (every row moves every
    step, as torch does): loss = mse(rgb_c, t) + mse(rgb_f, t) + the regulariser over the K * n rays of the step.  The pose
    parameter is the raw 3x4 camera-to-world matrix, what get_ray_bundle differentiates."""

    def __init__(self, model_coarse, model_fine, images, bboxs, intrinsics, poses, expressions, latents, background=None,
                 fit=TABLES, lr_pose=1e-4, lr_expression=1e-4, lr_latent=1e-4, betas=(0.9, 0.999), eps=1e-8, latent_reg=0.005,
                 num_coarse=64, num_fine=64, perturb=True, noise_std=0.1, near=0.2, far=0.8, white_bkgd=False, precision=None):
        fit = tuple(fit) if not isinstance(fit, str) else (fit,)
        if not fit:
            raise ValueError("nothing to fit: name at least one of 'pose', 'expression', 'latent'")
        if any(f not in TABLES for f in fit):
            raise ValueError(f"fit takes 'pose', 'expression' and 'latent', not {[f for f in fit if f not in TABLES]}")
        if precision is not None and precision not in _engine.PRECISIONS:
            raise ValueError(f"precision must be 'fast', 'exact' or 'exact_grad', not {precision!r}")
        n_img = images.shape[0]
        poses = poses.detach().reshape(n_img, -1)
        if poses.shape[1] not in (12, 16) or expressions.shape != (n_img, 76) or latents.shape != (n_img, 32):
            raise ValueError("poses [N,12] (or [N,3,4], [N,4,4]), expressions [N,76] and latents [N,32] for the N images")
        dev = next(model_coarse.parameters()).device
        self.eng = _engine.renderer_for(dev)
        self.dev, self.mc, self.mf = dev, model_coarse, model_fine
        self.fit = tuple(t for t in TABLES if t in fit)
        self.lr = dict(pose=float(lr_pose), expression=float(lr_expression), latent=float(lr_latent))
        self.betas, self.eps = betas, eps
        self.latent_reg = float(latent_reg)
        self.opts = dict(near=float(near), far=float(far), num_coarse=int(num_coarse), num_fine=int(num_fine) if model_fine is not None else 0,
                         perturb=bool(perturb), noise_std=float(noise_std), white_bkgd=bool(white_bkgd), precision=precision)
        self._iter = 0

        # ---- the fit bucket and its three tables
        self.n_images = int(n_img)
        self._off, off = {}, 0
        for t in TABLES:
            self._off[t] = off
            off += _pad(n_img * _WIDTH[t])
        self.params = torch.zeros(off, device=dev, dtype=torch.float32)
        self.grads = torch.zeros_like(self.params)
        self.exp_avg = torch.zeros_like(self.params)
        self.exp_avg_sq = torch.zeros_like(self.params)
        self.poses, self.expressions, self.latents = (self._table(self.params, t) for t in TABLES)
        self.poses.copy_(poses[:, :12].to(device=dev, dtype=torch.float32))
        self.expressions.copy_(expressions.detach().to(device=dev, dtype=torch.float32))
        self.latents.copy_(latents.detach().to(device=dev, dtype=torch.float32))

        # ---- the training set, its pose and expression tables aliased to the bucket's rows
        self.data = ray_sampler.TrainImages(images, self.poses, self.expressions, bboxs, intrinsics, background=background, device=dev)
        self.data.alias_tables(self.poses, self.expressions)

        # ---- frozen networks: FP32 copies the backward reads and the re-pack packs (their addresses are baked into graphs)
        self._pc = [_engine._f32c(t, dev).clone() for t in self.eng._params(model_coarse)]
        self._pf = [_engine._f32c(t, dev).clone() for t in self.eng._params(model_fine)] if model_fine is not None else None
        self._synced = None

        # ---- one NfbAdamDev per fitted table: constant learning rate (decay factor 1), no regulariser row
        self._adam = {}
        for t in self.fit:
            st = capi.NfbAdamDev(step=0, pad=0, lr0=self.lr[t], decay_factor=1.0, decay_steps=1.0, beta1=self.betas[0],
                                 beta2=self.betas[1], eps=self.eps, grad_scale=1.0, reg_weight=0.0, table_offset=-1, row=None,
                                 lr_over_bc1=0.0, sqrt_bc2=1.0, reg_offset=-1)
            self._adam[t] = torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(dev)
        self.loss = torch.zeros(4, device=dev, dtype=torch.float32)
        # pixels the sampler repeated because an image's selection came up short, per batch slot, since construction
        self.shortfall = torch.zeros(capi.NFB_MAX_STEP_IMAGES, device=dev, dtype=torch.int64)
        self._bufs = {}
        self._graph = None
        self._own_engine()

    def _table(self, bucket, name):
        n = self.n_images * _WIDTH[name]
        return bucket[self._off[name]:self._off[name] + n].view(self.n_images, _WIDTH[name])

    @property
    def iter(self):
        """Steps taken so far."""
        return self._iter

    def _fingerprint(self):
        return (self.eng._fingerprint(self.mc), self.eng._fingerprint(self.mf) if self.mf is not None else None)

    def _own_engine(self):
        """The device's renderer holds ONE set of packed weights.  Re-pack this fitter's networks (eagerly, never inside a graph)
        when someone else's are in place (a FusedTrainer step, a drop-in render of other models) or when the models' parameters
        changed since they were packed (their in-place version or storage, as the drop-in API checks)."""
        fp = self._fingerprint()
        if self.eng.packed_owner is self and fp == self._synced:
            return
        for dst, src in zip(self._pc + (self._pf or []), self.eng._params(self.mc) + (self.eng._params(self.mf) if self.mf is not None else [])):
            dst.copy_(src.detach())
        self.eng.repack(self._pc, self._pf)
        self.eng.mark_synced(self.mc, self.mf)
        self.eng.packed_owner = self
        self._synced = fp

    def _check(self, k, n, image_index=None, draws=None, max_rounds=32):
        """Argument checks of a step, all before any launch."""
        if not 1 <= k <= capi.NFB_MAX_STEP_IMAGES:
            raise ValueError(f"1 <= K <= {capi.NFB_MAX_STEP_IMAGES} images per step")
        if not 1 <= n <= 2048 or n > self.data.H * self.data.W:
            raise ValueError("1 <= n_per_image <= 2048 rays per image (and no more than the frame's pixels)")
        if max_rounds < 1:
            raise ValueError("max_rounds >= 1")
        if image_index is not None and any(not 0 <= int(i) < self.n_images for i in image_index):
            raise ValueError("image index out of range")
        if draws is not None and draws.numel() < k * max_rounds * n:
            raise ValueError("draws must hold K * max_rounds * n_per_image values")

    def _buffers(self, k, n):
        """Per-step buffers (cached per shape), with the input-gradient buffers of the fitted tables."""
        extra = dict(pose=dict(gro=(k * n, 3), grd=(k * n, 3)), expression=dict(gexpr=(k, 76)), latent=dict(glat=(k, 32)))
        shapes = dict(pixel_rc=((k * n, 2), torch.int32))
        for t in self.fit:
            shapes.update(extra[t])
        return _image_buffers(self._bufs, self.dev, self.data, k, n, self.shortfall, **shapes)

    def _sample(self, sb, n, draws, max_rounds):
        """nfb_sample_rays_images into the step's buffers (those named like NfbImageBatch's members), the latent rows read from
        the fit bucket."""
        self.eng.sample_images(self.data, sb["img"], n, draws, max_rounds, self.latents, sb)

    def _gradients(self, sb, k, n):
        """Fold, noise, forward, loss and input-only backward of the sampled batch, then the fitted tables' gradient rows."""
        eng, o, fit = self.eng, self.opts, self.fit
        N = k * n
        eng.set_frames(sb["expressions"], sb["latents"])
        out = eng.render(sb["ray_origins"], sb["ray_directions"], o["near"], o["far"], o["num_coarse"], o["num_fine"], perturb=o["perturb"],
                         noise_std=o["noise_std"], white_bkgd=o["white_bkgd"], background=sb["background"],
                         noise=_draw_noise(o, self.dev, N), precision=o["precision"], train=True, frame_index=sb["frame_index"])
        g1 = sb["g1"] if o["num_fine"] > 0 else None
        self.loss.zero_()
        eng.loss_mse_grad(out["rgb_coarse"], out.get("rgb_fine"), sb["target"], N, sb["g0"], g1, self.loss)
        pose, expr, lat = ("pose" in fit), ("expression" in fit), ("latent" in fit)
        eng.backward_into((sb["g0"], None, None, g1, None, None, None), self._pc, self._pf, None, None, sb.get("glat"), frames=True,
                          grad_expressions=sb.get("gexpr"), grad_ray_origins=sb.get("gro"), grad_ray_directions=sb.get("grd"))
        if pose or expr:
            eng.fit_rows_grad(self.data, sb["img"], n, sb["pixel_rc"], sb.get("gro"), sb.get("grd"),
                              self._table(self.grads, "pose") if pose else None, sb.get("gexpr"),
                              self._table(self.grads, "expression") if expr else None)
        if lat:
            eng.latent_rows_grad(sb["glat"], sb["img"], self.latents, self._table(self.grads, "latent"), self.latent_reg / k)
        return out

    def _adam_step(self):
        """Adam on every fitted table with its own device state; zeroes the table's gradients."""
        for t in self.fit:
            p, g, m, v = (self._table(b, t).view(-1) for b in (self.params, self.grads, self.exp_avg, self.exp_avg_sq))
            self.eng.adam_step_dev(p, g, m, v, self._adam[t])

    def _prepare(self, image_index, n_per_image, draws, max_rounds):
        k, n = len(image_index), int(n_per_image)
        self._check(k, n, image_index, draws, max_rounds)
        sb = self._buffers(k, n)
        sb["img"].copy_(torch.tensor([int(i) for i in image_index], dtype=torch.int32))
        if draws is None:
            draws = torch.rand(k * max_rounds * n, dtype=torch.float64, device=self.dev)
        self._own_engine()
        self._sample(sb, n, draws, max_rounds)
        found = sb["state"][:, 0].cpu()
        if bool((found < n).any()):
            short = [(int(image_index[j]), int(found[j])) for j in range(k) if int(found[j]) < n]
            raise RuntimeError(f"ray sampler: {max_rounds} rounds of draws found fewer than {n} distinct pixels for (image, found) "
                               f"{short}; raise max_rounds")
        return sb, k, n

    def gradients(self, image_index, n_per_image, draws=None, max_rounds=32):
        """Forward and backward of one step's batch into the fit bucket's gradients (self.grads, zeroed first): the pose,
        expression and latent rows of the fitted tables (regulariser included), nothing else.  No optimizer step.  Returns the
        device tensor [mse_coarse, mse_fine]; the step's buffers stay in self._bufs (rays, pixel_rc, the per-ray gradients)."""
        sb, k, n = self._prepare(image_index, n_per_image, draws, max_rounds)
        self.grads.zero_()
        self._last = sb
        self._gradients(sb, k, n)
        return self.loss[:2]

    def step(self, image_index, n_per_image, draws=None, max_rounds=32):
        """One fitting step on n_per_image rays of each of the K images image_index (host ints, repeats allowed).  draws: float64
        CUDA [K * max_rounds * n] as FusedTrainer.step_images takes them (None: torch.rand on the device).  Raises RuntimeError,
        before any gradient is formed, when an image's selection came up short of n distinct pixels.  Returns the device tensor
        [mse_coarse, mse_fine].
        Launches per step (within the memory budget; +1 the first time the sampler's scratch grows), by fitted tables:
        (pose): 14, (expression): 14, (latent): 14, (pose, expression): 19, (pose, latent): 20, (expression, latent): 17,
        (pose, expression, latent): 22 — sample 1, set_frames 1, forward 1, loss 1, backward 4 (compositing 2, dX chain 1,
        reduction 1) + 3 with expression or latent (per-ray and per-frame sums 2, per-frame gradients 1) + 2 with pose (input
        rows and rays), pose / expression rows 2 with pose, else 1 with expression, latent rows 1 with latent, Adam 2 per table."""
        sb, k, n = self._prepare(image_index, n_per_image, draws, max_rounds)
        self._gradients(sb, k, n)
        self._adam_step()
        self._iter += 1
        return self.loss[:2]

    def capture(self, k, n_per_image, has_background=True, max_rounds=32, device_draws=True):
        """Capture a whole K-image fitting step into a CUDA graph: sampler (draws from torch.rand(float64) inside the graph, or
        with device_draws=False from a static buffer step_graph fills), fold, noise, forward, loss, backward, rows, Adam.  Only the
        K image indices change between replays; the tables are read in place, so writes into fit.poses / expressions / latents
        between replays take effect.  An incomplete selection does not stop the graph: the missing slots repeat the image's first
        pixels and self.shortfall[k] counts them.  The graph holds the renderer's buffers as sized at capture: when a later call on
        the device re-allocates them, step_graph raises RuntimeError (capture again).  Never re-packs inside the graph: step_graph
        re-packs eagerly, before the replay, when needed."""
        n = int(n_per_image)
        self._check(k, n, max_rounds=max_rounds)
        if has_background != (self.data.background is not None):
            raise ValueError("has_background must say whether the training set has a background")
        sb = dict(self._buffers(k, n))  # own copies: eager steps must not write into a graph's buffers
        for name, t in list(sb.items()):
            if t is not None and name != "shortfall":
                sb[name] = torch.zeros_like(t)
        sb["draws"] = None if device_draws else torch.zeros(k * max_rounds * n, device=self.dev, dtype=torch.float64)

        def body():
            draws = torch.rand(k * max_rounds * n, dtype=torch.float64, device=self.dev) if device_draws else sb["draws"]
            self._sample(sb, n, draws, max_rounds)
            return self._gradients(sb, k, n), draws

        sb["img"].copy_(torch.arange(k, dtype=torch.int32) % self.n_images)
        if not device_draws:
            sb["draws"].uniform_()
        before = self.shortfall.clone()
        g = _capture(self._own_engine, self.eng, self.grads, body, self._adam_step)
        self.shortfall.copy_(before)  # the warm-up's selections are not a step's
        self._graph = dict(g, sb=sb, k=k, n=n)
        return self

    def step_graph(self, image_index, draws=None):
        """One fitting step by replaying the graph of capture(): copies the K image indices (host ints, or an int32 CUDA / pinned
        tensor) and, when captured with device_draws=False, the draws, re-packs the networks eagerly if another owner's weights
        are in place, then replays.  Raises RuntimeError before it copies or launches anything when the renderer buffers the
        graph points at were re-allocated since capture."""
        g = self._graph
        if g is None:
            raise RuntimeError("capture() first")
        _check_epoch(self.eng, g)
        sb = g["sb"]
        if len(image_index) != g["k"]:
            raise ValueError(f"the graph was captured for {g['k']} images per step")
        if sb["draws"] is not None and draws is None:
            raise ValueError("the graph was captured with device_draws=False: pass the draws")
        idx = image_index if torch.is_tensor(image_index) else torch.tensor([int(i) for i in image_index], dtype=torch.int32)
        sb["img"].copy_(idx, non_blocking=True)
        if sb["draws"] is not None:
            sb["draws"].copy_(draws.reshape(-1)[:sb["draws"].numel()], non_blocking=True)
        self._own_engine()
        g["graph"].replay()
        self._iter += 1
        return self.loss[:2]
