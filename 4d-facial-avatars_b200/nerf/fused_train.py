"""Fused training step (SURVEY.md §8f rank 2): what train_transformed_rays.py:336-400 does per iteration — render in train
mode, mse(rgb_coarse) + mse(rgb_fine) + 10 * 0.0005 * ||latent||, loss.backward(), optimizer.step(), zero_grad(), LR decay —
as kernel launches of libnfb on ONE flat FP32 parameter bucket, with no torch.autograd graph, no torch.optim and no
gradient copies:

    set_frame (1 launch) -> training forward (1) -> loss gradient (1) -> backward (writes into the flat gradient bucket)
    -> [one NCCL all-reduce of that bucket when the batch is sharded over ranks] -> Adam + zero_grad (2: schedule, update)
    -> re-pack (2: fold, pack)

The models keep their reference `state_dict` (their parameters become views of the bucket), so checkpoints, `.parameters()`
and the drop-in `run_one_iter_of_nerf` keep working on the same objects.  torch is used for memory, the noise draws (in the
reference's order) and torch.distributed."""
import torch
import torch.distributed as dist

from . import _capi as capi
from . import _engine
from . import train_utils
from ._engine import PARAM_ORDER


def _draw_noise(opts, dev, n):
    """The reference's draws for one chunk of n rays (train chunksize = num_random_rays in the shipped YAML, so a batch is one
    chunk); None when neither perturbation nor sigma noise is on.  Shared by the fused training and fitting steps."""
    return train_utils._draw_noise(n, opts, dev, opts["num_fine"] > 0) if (opts["perturb"] or opts["noise_std"] > 0.0) else None


def _capture(own_engine, eng, grads, body, tail):
    """The capture skeleton of the fused steps: own the renderer's packed weights, body() once eagerly (the warm-up sizes the
    library's buffers: cudaMalloc is not capturable), read the buffer epoch, zero the gradient bucket, then body() and tail()
    captured into a CUDA graph.  Returns the graph, what the captured body returned (its buffers must outlive the graph) and
    the epoch."""
    own_engine()
    body()
    epoch = eng.buffer_epoch()
    grads.zero_()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        keep = body()
        tail()
    return dict(graph=graph, keep=keep, epoch=epoch)


def _check_epoch(eng, g):
    """Refuse to replay a graph whose renderer buffers were re-allocated or refilled since capture (nfb_buffer_epoch)."""
    if eng.buffer_epoch() != g["epoch"]:
        raise RuntimeError("a call on this device since capture re-allocated renderer buffers the graph points at (a larger "
                           "step, more frames or more images per step, on any trainer): capture again")


def _image_buffers(cache, dev, data, k, n, shortfall, **extra):
    """Per-step buffers of a K-image step, cached per (K, n, background): the sampler's outputs for N = K * n rays, the
    loss-gradient buffers g0 / g1 [N,3] and the caller's `extra` buffers, name -> shape (float32) or (shape, dtype).  The chunked backward re-reads
    rays and frame indices, so they outlive the step."""
    key = (k, n, data.background is not None)
    sb = cache.get(key)
    if sb is None:
        N = k * n
        z = lambda *shape, dt=torch.float32: torch.zeros(shape, device=dev, dtype=dt)  # noqa: E731
        sb = cache[key] = dict(
            img=z(k, dt=torch.int32), ray_origins=z(N, 3), ray_directions=z(N, 3), target=z(N, 3),
            background=z(N, 3) if data.background is not None else None, frame_index=z(N, dt=torch.int32),
            expressions=z(k, 76), latents=z(k, 32), state=z(k, 3, dt=torch.int32), shortfall=shortfall[:k],
            g0=z(N, 3), g1=z(N, 3),
            **{name: (z(*s[0], dt=s[1]) if isinstance(s[-1], torch.dtype) else z(*s)) for name, s in extra.items()})
    return sb


class FusedTrainer:
    background = None      # the learned background's [H,W,3] rows (None: the training set's background, if any, is fixed)
    background_loss = 0.0  # the supervised background term's weight

    def __init__(self, model_coarse, model_fine, n_latent, lr=5e-4, lr_decay_steps=250000, lr_decay_factor=0.1,
                 betas=(0.9, 0.999), eps=1e-8, num_coarse=64, num_fine=64, perturb=True, noise_std=0.1, near=0.2, far=0.8,
                 latent_reg=0.005, white_bkgd=False, latent_codes=None, precision=None, background=None, background_loss=0.0):
        """background: the initial [H,W,3] image of a background this trainer LEARNS (train_transformed_rays.py:128-157,
        train_background): it joins the bucket as its own rows, steps over several images gather it at their pixels and Adam
        updates it with everything else (the reference's second parameter group has the same learning rate and decay).  None: the
        background, if any, is the training set's fixed one.  background_loss: the weight of the supervised term
        weight * mean(w_last * ||bg - target||^2) (supervised_train_background; 0.001 in the reference, 0: off).  Initialise it
        as the reference does from the training images [N,H,W,3]:  bg = images.mean(0)  (optionally blurred first:
        nerf.GaussianSmoothing(3, 11, 11)(bg.permute(2, 0, 1)[None])[0].permute(1, 2, 0))."""
        self.background_loss = float(background_loss)  # checked before the renderer is touched
        if background is not None:
            background = torch.as_tensor(background)
            if background.dim() != 3 or background.shape[2] != 3:
                raise ValueError("background must be an [H,W,3] image")
        elif self.background_loss != 0.0:
            raise ValueError("background_loss supervises a learned background: pass background=")
        if self.background_loss < 0.0:
            raise ValueError("background_loss must be >= 0")
        dev = next(model_coarse.parameters()).device
        self.eng = _engine.renderer_for(dev)
        self.dev, self.mc, self.mf = dev, model_coarse, model_fine
        self.lr0, self.decay_steps, self.decay_factor = float(lr), float(lr_decay_steps), float(lr_decay_factor)
        self.betas, self.eps = betas, eps
        self.opts = dict(near=float(near), far=float(far), num_coarse=int(num_coarse), num_fine=int(num_fine) if model_fine is not None else 0,
                         perturb=bool(perturb), noise_std=float(noise_std), white_bkgd=bool(white_bkgd), precision=precision)
        self.latent_reg = float(latent_reg)
        self._iter = 0

        # ---- flat bucket: [coarse 26 tensors | fine 26 tensors | pad to 256 | latent table n_latent x 32
        #                    (| pad to 256 | learned background H x W x 3)]
        models = [model_coarse] + ([model_fine] if model_fine is not None else [])
        tensors = [dict(m.named_parameters())[k] for m in models for k in PARAM_ORDER]
        n_mlp = sum(t.numel() for t in tensors)
        self.lat_off = (n_mlp + 255) // 256 * 256
        self._lat_end = n_total = self.lat_off + n_latent * 32
        self.bg_off = None
        if background is not None:
            self.bg_off = (n_total + 255) // 256 * 256
            n_total = self.bg_off + background.numel()
        self.params = torch.zeros(n_total, device=dev, dtype=torch.float32)
        self.grads = torch.zeros_like(self.params)
        self.exp_avg = torch.zeros_like(self.params)
        self.exp_avg_sq = torch.zeros_like(self.params)
        off = 0
        self._views, self._gviews = [], []
        for t in tensors:
            n = t.numel()
            view = self.params[off:off + n].view(t.shape)
            view.copy_(t.detach().to(device=dev, dtype=torch.float32))
            t.data = view  # the module's parameter now IS a slice of the bucket
            self._views.append(view)
            self._gviews.append(self.grads[off:off + n].view(t.shape))
            off += n
        self.latent_codes = self.params[self.lat_off:self._lat_end].view(n_latent, 32)
        if latent_codes is not None:
            self.latent_codes.copy_(latent_codes.detach().to(dev))
        # the learned background: an [H,W,3] view of its rows (what a reference-format checkpoint stores under "background")
        self.background = self._bg_grads = None
        if background is not None:
            self.background = self.params[self.bg_off:].view(background.shape)
            self.background.copy_(background.detach().to(device=dev, dtype=torch.float32))
            self._bg_grads = self.grads[self.bg_off:].view(background.shape)
        npar = len(PARAM_ORDER)
        skip = [k.startswith("layers_dir.3") for k in PARAM_ORDER]  # unused by the forward (models.py:257): no gradient
        self._pc, self._pf = self._views[:npar], (self._views[npar:] if model_fine is not None else None)
        self._gc = [None if s else g for s, g in zip(skip, self._gviews[:npar])]
        self._gf = [None if s else g for s, g in zip(skip, self._gviews[npar:])] if model_fine is not None else None
        self.loss = torch.zeros(4, device=dev, dtype=torch.float32)
        # pixels the K-image sampler repeated because an image's selection came up short, per batch slot, since construction
        self.shortfall = torch.zeros(64, device=dev, dtype=torch.int64)
        self._g_rgb = {}
        self._image_bufs = {}
        # ONE optimizer state on the device (NfbAdamDev) for every kind of step — eager, captured, one image or several — so
        # all of them take one step counter and one learning-rate schedule (nfb_adam_step_dev).  Each step writes the latent
        # row its regulariser applies to into self._row first (-1: none).
        self._row = torch.full((1,), -1, device=dev, dtype=torch.int64)
        st = capi.NfbAdamDev(step=0, pad=0, lr0=self.lr0, decay_factor=self.decay_factor, decay_steps=self.decay_steps,
                             beta1=self.betas[0], beta2=self.betas[1], eps=self.eps, grad_scale=1.0, reg_weight=self.latent_reg,
                             table_offset=self.lat_off if self.latent_reg > 0.0 else -1, row=self._row.data_ptr(),
                             lr_over_bc1=0.0, sqrt_bc2=1.0, reg_offset=-1)
        self._adam = torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(dev)
        self._own_engine()

    @property
    def iter(self):
        """Optimizer steps taken so far (the host's copy of the device state's step counter)."""
        return self._iter

    @iter.setter
    def iter(self, value):
        """Set the step counter, e.g. on resume: the next step takes the schedule's step value + 1."""
        self._iter = int(value)
        self._adam[:4].copy_(torch.tensor([self._iter], dtype=torch.int32).view(torch.uint8))

    def _own_engine(self):
        """The device's renderer holds ONE set of packed weights: (re-)pack this trainer's if someone else's are in place (another
        trainer, or other models rendered through the drop-in API since the last step)."""
        if self.eng.packed_owner is not self:
            self.eng.repack(self._pc, self._pf)
            self.eng.mark_synced(self.mc, self.mf)
            self.eng.packed_owner = self

    def _draw_noise(self, n):
        return _draw_noise(self.opts, self.dev, n)

    def _latent_grads(self):
        """The latent table's rows of the gradient bucket, [n_latent,32]."""
        return self.grads[self.lat_off:self._lat_end].view(-1, 32)

    def _single_image(self, name):
        if self.background is not None:
            raise ValueError(f"{name}() takes background rays gathered by the caller and no pixel indices, so it cannot learn a "
                             "background: a trainer built with background= steps with step_images / capture_images")

    def _forward_backward(self, expressions, latents, frame_index, ro, rd, background, target, n_total, noise, g, grad_latent,
                          grad_background=None):
        """Frame fold, training forward, loss gradient and backward of one batch into the flat gradient bucket, d latent into
        grad_latent.  frame_index None: one frame (expressions [76], latents [32]); otherwise ray i is conditioned on frame
        frame_index[i] of expressions [F,76] and latents [F,32], and grad_latent is [F,32].  g: the [n,3] loss-gradient buffers
        (g0, g1), and with the supervised background term also its [n,3] background and [n] w_last gradient buffers.
        grad_background: [n,3] receives the per-ray background gradient of the render (a learned background)."""
        eng, o = self.eng, self.opts
        frames = frame_index is not None
        if frames:
            eng.set_frames(expressions, latents)
        else:
            eng.set_frame(expressions, latents)
        out = eng.render(ro, rd, o["near"], o["far"], o["num_coarse"], o["num_fine"], perturb=o["perturb"], noise_std=o["noise_std"],
                         white_bkgd=o["white_bkgd"], background=background, noise=noise, precision=o["precision"], train=True,
                         frame_index=frame_index)
        g1 = g[1] if o["num_fine"] > 0 else None
        self.loss.zero_()
        eng.loss_mse_grad(out["rgb_coarse"], out.get("rgb_fine"), target, n_total, g[0], g1, self.loss)
        g_wlast = None
        if len(g) > 2:  # the supervised background term on the last pass's w_last; its share goes to loss[2]
            eng.loss_background_grad(background, target, out["w_last"], n_total, self.background_loss, g[2], g[3], self.loss[2:3])
            g_wlast = g[3]
        eng.backward_into((g[0], None, None, g1, None, None, g_wlast), self._pc, self._pf, self._gc, self._gf, grad_latent,
                          frames=frames, grad_background=grad_background)
        return out

    def _stepped(self):
        """Host bookkeeping after an optimizer step: the step counter, and the packed streams now hold this trainer's weights."""
        self._iter += 1
        self.eng.mark_synced(self.mc, self.mf)
        self.eng.packed_owner = self

    def _adam_repack(self, row):
        """Adam on the trainer's device state with the latent regulariser on `row` (an int, -1 for none, or a device tensor
        holding it), zero_grad, then the re-pack."""
        if torch.is_tensor(row):
            self._row.copy_(row)
        else:
            self._row.fill_(row)
        self.eng.adam_step_dev(self.params, self.grads, self.exp_avg, self.exp_avg_sq, self._adam)
        self.eng.repack(self._pc, self._pf)

    def _capture(self, body, row, world=1, group=None, after_collective=None):
        """body() once eagerly, then body, the all-reduce (world > 1) followed by after_collective(), Adam with its regulariser
        on `row` and the re-pack captured into a CUDA graph.  Returns the graph, what the captured body returned (its buffers
        must outlive the graph) and the renderer's buffer epoch."""
        def tail():
            if world > 1:
                dist.all_reduce(self.grads, group=group)
                if after_collective is not None:
                    after_collective()
            self._adam_repack(row)
        return _capture(self._own_engine, self.eng, self.grads, body, tail)

    def gradients(self, ray_origins, ray_directions, target, expressions, latent_index, background=None, world=1, n_total=None,
                  noise=None, events=None, group=None):
        """Forward, loss and backward of this rank's rays ([n,3] CUDA tensors) into the flat gradient bucket; world > 1: the rays
        are one of `world` equal shards of a batch of n_total rays and the bucket is SUM-all-reduced (one collective), after
        which every rank holds the whole batch's gradient.  Returns the device tensor [mse_coarse, mse_fine] of THIS shard's
        share (sum over ranks = batch loss).  `events`: optional (before_collective, after_collective) CUDA events.  A trainer
        that learns its background raises ValueError (so do step, capture and step_graph)."""
        self._single_image("gradients")
        self._own_engine()
        n = ray_origins.shape[0]
        n_total = n * world if n_total is None else n_total
        if noise is None:
            noise = self._draw_noise(n)
        g = self._g_rgb.get(n)
        if g is None:
            g = self._g_rgb[n] = (torch.empty((n, 3), device=self.dev), torch.empty((n, 3), device=self.dev))
        glat = self.grads[self.lat_off + 32 * latent_index:self.lat_off + 32 * latent_index + 32]
        self._forward_backward(expressions, self.latent_codes[latent_index], None, ray_origins, ray_directions, background,
                               _engine._f32c(target, self.dev), n_total, noise, g, glat)
        if events is not None:
            events[0].record()
        if world > 1:
            dist.all_reduce(self.grads, group=group)  # ONE collective over the flat bucket (sum: the loss is pre-divided by n_total)
        if events is not None:
            events[1].record()
        self._reg_row = latent_index
        return self.loss[:2]

    def update(self):
        """Adam over the bucket (+ the latent regulariser's gradient on the last frame's row, + zero_grad) on the trainer's device
        state, then the re-pack."""
        self._adam_repack(self._reg_row)
        self._stepped()

    def _check_epoch(self, g):
        _check_epoch(self.eng, g)

    # ---- the whole iteration as ONE CUDA graph (launch-bound at small per-rank batches: ~20 kernels of 3-800 us)
    def capture(self, n, has_background=True, world=1, n_total=None, group=None):
        """Capture gradients() + update() for batches of exactly n rays on this rank into a CUDA graph.  Everything that changes
        from step to step lives in device memory: the inputs (static buffers filled by step_graph), the latent row index, and the
        optimizer's step counter / learning rate (the trainer's one nfb_adam_step_dev state, which its eager steps share).  The
        noise is drawn inside the graph (torch's graph-safe Philox state), in the reference's order.  With world > 1 the NCCL all-reduce of the flat bucket is part of the graph."""
        self._single_image("capture")
        dev = self.dev
        n_total = n * world if n_total is None else n_total
        z = lambda *shape, dt=torch.float32: torch.zeros(shape, device=dev, dtype=dt)  # noqa: E731
        sb = dict(ro=z(n, 3), rd=z(n, 3), tgt=z(n, 3), bg=z(n, 3) if has_background else None, expr=z(76), idx=z(1, dt=torch.int64),
                  lat=z(32), glat=z(32), g0=z(n, 3), g1=z(n, 3))
        sb["rd"][:, 2] = -1.0  # a valid ray for the warm-up
        sb["adam"] = self._adam     # the optimizer state the graph advances: the trainer's one state, not a copy
        table_grads = self._latent_grads()

        def forward_backward():
            sb["lat"].copy_(self.latent_codes.index_select(0, sb["idx"])[0])
            out = self._forward_backward(sb["expr"], sb["lat"], None, sb["ro"], sb["rd"], sb["bg"], sb["tgt"], n_total,
                                         self._draw_noise(n), (sb["g0"], sb["g1"]), sb["glat"])
            table_grads.index_add_(0, sb["idx"], sb["glat"][None])
            return out

        self._graph = dict(self._capture(forward_backward, sb["idx"], world, group), sb=sb, n=n)
        return self

    def step_graph(self, ray_origins, ray_directions, target, expressions, latent_index, background=None):
        """One optimizer step by replaying the captured graph (capture() first): copies the step's inputs into the static buffers —
        on the current stream, so the caller may keep them on the device or in pinned host memory — and replays.  Raises
        RuntimeError, before it copies or launches anything, when a call on this device has re-allocated the renderer buffers the
        graph points at since capture (nfb_buffer_epoch): capture again."""
        self._single_image("step_graph")
        g = self._graph
        self._check_epoch(g)
        sb = g["sb"]
        if ray_origins.shape[0] != g["n"]:
            raise ValueError(f"the graph was captured for {g['n']} rays per step")
        self._own_engine()
        sb["ro"].copy_(ray_origins, non_blocking=True)
        sb["rd"].copy_(ray_directions, non_blocking=True)
        sb["tgt"].copy_(target, non_blocking=True)
        if sb["bg"] is not None:
            sb["bg"].copy_(background, non_blocking=True)
        sb["expr"].copy_(expressions.reshape(-1), non_blocking=True)
        sb["idx"].fill_(int(latent_index))
        g["graph"].replay()
        self._stepped()
        return self.loss[:2]

    def step(self, *args, **kwargs):
        """One optimizer step: gradients(...) then update().  Returns gradients()'s loss tensor."""
        self._single_image("step")
        loss = self.gradients(*args, **kwargs)
        self.update()
        return loss

    # ---- steps over rays of several training images (DESIGN.md 8c): sample, gather, fold, forward, loss, backward, latent rows,
    # Adam and re-pack from K image indices alone.  world > 1: every rank samples the whole batch of N = K * n rays on the same
    # draws and renders its slice [rank * N / world, (rank + 1) * N / world); one SUM all-reduce of the bucket joins the slices.
    def _images_buffers(self, data, k, n):
        """Per-step buffers of a K-image step (cached per shape: the chunked backward re-reads rays and frame indices); with a
        learned background also the pixels, the per-ray background gradient and (supervised) the background term's gradients."""
        extra = dict(glat=(k, 32), zero_lat=(k, 32))
        if self.background is not None:
            extra.update(pixel_rc=((k * n, 2), torch.int32), g_bg=(k * n, 3))
            if self.background_loss > 0.0:
                extra.update(g_bgl=(k * n, 3), g_wl=(k * n,))
        return _image_buffers(self._image_bufs, self.dev, data, k, n, self.shortfall, **extra)

    def _images_data(self, data):
        """What the sampler reads: with a learned background, a copy of the caller's set whose background is the bucket's rows
        (read in place, so every step and every replay gathers the current estimate); otherwise the caller's set."""
        return data.with_background(self.background) if self.background is not None else data

    def _images_sample(self, data, sb, n, draws, max_rounds):
        self.eng.sample_images(data, sb["img"], n, draws, max_rounds, self.latent_codes, sb)

    def _images_gradients(self, sb, k, n, world=1, rank=0):
        """Forward, loss and backward of this rank's slice of the sampled batch into the flat bucket, then the latent-table rows.
        K = 1 takes the single-frame kernels (its regulariser stays in Adam, as in step()); K >= 2 one multi-frame forward and
        backward over all K frames (a frame without rays in the slice gets exactly zero d latent).  The noise is drawn for the
        whole batch and sliced, and the loss is divided by the whole batch's N = K * n rays, so the slices' buckets sum to the
        single-process gradient.  The K >= 2 regulariser is added here only when world == 1 (else _images_regulariser, after
        the collective, adds it once).  A learned background: the supervised term (background_loss > 0) after the MSE, the
        per-ray background gradient from the backward, and the slice's background rows before the latent rows."""
        N = k * n
        per = N // world
        sl = slice(rank * per, (rank + 1) * per)
        noise = self._draw_noise(N)
        if world > 1 and noise is not None:
            noise = {key: (v[sl] if v is not None else None) for key, v in noise.items()}
        if k == 1:
            expr, lat, fi, glat = sb["expressions"][0], sb["latents"][0], None, sb["glat"][0]
        else:
            expr, lat, fi, glat = sb["expressions"], sb["latents"], sb["frame_index"][sl], sb["glat"]
        bg = sb["background"][sl] if sb["background"] is not None else None
        learn, supervised = self.background is not None, self.background_loss > 0.0
        g = (sb["g0"][sl], sb["g1"][sl]) + ((sb["g_bgl"][sl], sb["g_wl"][sl]) if supervised else ())
        out = self._forward_backward(expr, lat, fi, sb["ray_origins"][sl], sb["ray_directions"][sl], bg, sb["target"][sl], N, noise,
                                     g, glat, grad_background=sb["g_bg"][sl] if learn else None)
        if learn:
            self.eng.background_rows_grad(sb["pixel_rc"][sl], self.background.shape[0], self.background.shape[1], sb["g_bg"][sl],
                                          sb["g_bgl"][sl] if supervised else None, self._bg_grads)
        self.eng.latent_rows_grad(sb["glat"], sb["img"], self.latent_codes, self._latent_grads(),
                                  self.latent_reg / k if k >= 2 and world == 1 else 0.0)
        return out

    def _images_regulariser(self, sb, k):
        """K >= 2 after the collective: the regulariser terms (latent_reg / K) * l / ||l|| added once, in ascending k, onto the
        summed latent rows (nfb_latent_rows_grad with zero frame gradients: adding +0.0 leaves a row as it is)."""
        if k >= 2:
            self.eng.latent_rows_grad(sb["zero_lat"], sb["img"], self.latent_codes, self._latent_grads(), self.latent_reg / k)

    def _check_images(self, data, k, n, world, group=None, rank=None):
        """Argument checks of a K-image step, all before any launch or collective; returns this rank's index.  world > 1 needs
        the collective: without an initialised torch.distributed process group and without an explicit rank the step cannot
        run data-parallel (NotImplementedError, as for any world > 1 step before data-parallel steps existed)."""
        if world < 1:
            raise ValueError(f"world = {world}: a step runs on at least one rank")
        if world > 1:
            if rank is None:
                if not (dist.is_available() and dist.is_initialized()):
                    raise NotImplementedError("steps over several images with world > 1 run over a torch.distributed process "
                                              "group: initialise one (or pass rank=) first")
                rank = dist.get_rank(group)
            rank = int(rank)
            if not 0 <= rank < world:
                raise ValueError(f"rank {rank} is outside [0, {world})")
        if not 1 <= k <= 64:
            raise ValueError("1 <= K <= 64 images per step")
        if not 1 <= n <= 2048 or n > data.H * data.W:
            raise ValueError("1 <= n_per_image <= 2048 rays per image (and no more than the frame's pixels)")
        if data.n_images > self.latent_codes.shape[0]:
            raise ValueError("the latent table has fewer rows than the training set has images")
        if (k * n) % world:
            raise ValueError(f"a batch of K * n_per_image = {k * n} rays does not split evenly over world = {world} ranks")
        if self.background is not None:
            if data.background is not None:
                raise ValueError("this trainer learns the background: the training set must not carry one of its own")
            if tuple(self.background.shape[:2]) != (data.H, data.W):
                raise ValueError(f"the learned background is {tuple(self.background.shape[:2])} but the training set's frames are "
                                 f"{(data.H, data.W)}")
        return 0 if world == 1 else rank

    def step_images(self, data, image_index, n_per_image, draws=None, max_rounds=32, world=1, group=None, rank=None):
        """One optimizer step on n_per_image rays of each of the K images image_index (host ints, repeats allowed; image i
        conditions on expressions[i] and latent row i).  data: ray_sampler.TrainImages.  draws: float64 CUDA [K * max_rounds * n]
        (image k consumes slice k as RandomState.rand inside np.random.choice); None: torch.rand on the device.  The loss is
        mse(rgb_c, t) + mse(rgb_f, t) + (latent_reg / K) * sum_k ||latent[image_index[k]]|| over all K * n rays.  K = 1 is step()
        on the sampled rays, bit for bit.  Raises RuntimeError, before any gradient is formed, when an image's selection came
        up short of n distinct pixels within max_rounds rounds.
        world > 1 (rank: dist.get_rank(group), or the explicit `rank`): data-parallel over `world` ranks, K * n must divide by
        world (ValueError otherwise); without an initialised process group and without `rank` it raises NotImplementedError, as
        every world > 1 step did before data-parallel steps existed.  Every rank samples the whole batch and renders its slice
        of K * n / world rays; one SUM all-reduce of the bucket over `group` follows, then (K >= 2) the regulariser, once.  Every rank must pass the same
        image_index and draws (with draws=None, seed torch alike on every rank): the argument checks and the short-selection
        error then raise on all ranks together, before the collective.
        Launches (within the memory budget; +1 the first time the sampler's scratch grows): K = 1: 16 = sample 1, set_frame 1,
        forward 1, loss 1, backward 7, latent rows 1, Adam 2, re-pack 2; K >= 2: 19 = sample 1, set_frames 1, forward 1, loss 1,
        backward 10, latent rows 1, Adam 2, re-pack 2 (Adam: schedule and update on the trainer's device state, as in every step,
        eager or captured).  world > 1 adds the all-reduce, and at K >= 2 one latent-rows launch after it (20).  Returns the
        device tensor [mse_coarse, mse_fine] (world > 1: this rank's share; the shares sum to the batch loss).
        A learned background (background= at construction; DESIGN.md 8e): the sampler gathers the background rays from the
        bucket's rows, the backward also forms the per-ray background gradient (+1 launch) and nfb_background_rows_grad adds this
        rank's rays onto the rows before the latent rows (+1): 18 launches at K = 1 and 21 at K >= 2.  background_loss > 0 adds
        the supervised term weight * mean(w_last * ||bg - target||^2) after the MSE (+1: 19 and 22), its w_last gradient
        feeding the backward; its share of the loss is in self.loss[2].  The argument checks also raise ValueError when `data`
        carries a background of its own or its frames are not the learned background's H x W."""
        k, n = len(image_index), int(n_per_image)
        rank = self._check_images(data, k, n, world, group, rank)
        if any(not 0 <= int(i) < data.n_images for i in image_index):
            raise ValueError("image index out of range")
        if draws is not None and draws.numel() < k * max_rounds * n:
            raise ValueError("draws must hold K * max_rounds * n_per_image values")
        data = self._images_data(data)
        sb = self._images_buffers(data, k, n)
        sb["img"].copy_(torch.tensor([int(i) for i in image_index], dtype=torch.int32))
        if draws is None:
            draws = torch.rand(k * max_rounds * n, dtype=torch.float64, device=self.dev)
        self._own_engine()
        self._images_sample(data, sb, n, draws, max_rounds)
        found = sb["state"][:, 0].cpu()
        if bool((found < n).any()):
            short = [(int(image_index[j]), int(found[j])) for j in range(k) if int(found[j]) < n]
            raise RuntimeError(f"ray sampler: {max_rounds} rounds of draws found fewer than {n} distinct pixels for (image, found) "
                               f"{short}; raise max_rounds")
        self._images_gradients(sb, k, n, world, rank)
        if world > 1:
            dist.all_reduce(self.grads, group=group)  # ONE collective over the flat bucket
            self._images_regulariser(sb, k)
        # K = 1: the regulariser in Adam on the image's row, as in step(); K >= 2: none (nfb_latent_rows_grad added it)
        self._reg_row = int(image_index[0]) if k == 1 else -1
        self.update()
        return self.loss[:2]

    def capture_images(self, data, k, n_per_image, has_background=True, max_rounds=32, device_draws=True, world=1, group=None,
                       rank=None):
        """Capture a whole K-image step into a CUDA graph: sampler (draws from torch.rand(float64) inside the graph, or with
        device_draws=False from a static buffer step_images_graph fills), fold, noise, forward, loss, backward, latent rows,
        [world > 1: the all-reduce of the bucket, then at K >= 2 the regulariser], Adam with its device-side schedule, re-pack.
        Only the K image indices change between replays.  world, group and rank as in step_images; with device_draws=True every
        rank must seed torch alike, so that the ranks sample the same batch.  An incomplete selection does not stop the graph:
        the image's missing slots repeat its first pixels and self.shortfall[k] counts them (include/nfb.h,
        nfb_sample_rays_images).  Launches per replay: 16 at K = 1, 19 at K >= 2 (world > 1: + the all-reduce, and 20 at K >= 2);
        a learned background adds step_images' 2, and its supervised term 1 more.  has_background is ignored then.
        The graph holds the renderer's device buffers as sized at capture, and they only grow: a later call on the same device,
        by any trainer, that needs more room (more images or rays per step, more frames, a larger render with gradients)
        re-allocates them.  step_images_graph then raises RuntimeError instead of replaying (nfb_buffer_epoch): capture again."""
        n = int(n_per_image)
        rank = self._check_images(data, k, n, world, group, rank)
        if self.background is None and has_background != (data.background is not None):
            raise ValueError("has_background must say whether the training set has a background")
        dev = self.dev
        data = self._images_data(data)
        sb = dict(self._images_buffers(data, k, n))  # own copies of the per-step buffers: eager steps must not write into them
        for name, t in list(sb.items()):
            if t is not None and name != "shortfall":
                sb[name] = torch.zeros_like(t)
        sb["draws"] = None if device_draws else torch.zeros(k * max_rounds * n, device=dev, dtype=torch.float64)

        def body():
            draws = torch.rand(k * max_rounds * n, dtype=torch.float64, device=dev) if device_draws else sb["draws"]
            self._images_sample(data, sb, n, draws, max_rounds)
            return self._images_gradients(sb, k, n, world, rank), draws

        sb["img"].copy_(torch.arange(k, dtype=torch.int32) % data.n_images)
        if not device_draws:
            sb["draws"].uniform_()
        before = self.shortfall.clone()
        # K = 1: the regulariser in Adam on the image's row; K >= 2: none (nfb_latent_rows_grad adds it)
        g = self._capture(body, sb["img"] if k == 1 else -1, world, group, after_collective=lambda: self._images_regulariser(sb, k))
        self.shortfall.copy_(before)  # the warm-up's selections are not a step's
        self._igraph = dict(g, sb=sb, k=k, n=n, max_rounds=max_rounds)
        return self

    def step_images_graph(self, image_index, draws=None):
        """One optimizer step by replaying the graph of capture_images: copies the K image indices (host ints, or an int32 CUDA /
        pinned tensor: no host sync) and, when captured with device_draws=False, the draws, then replays.  Raises RuntimeError, as
        step_graph does, when the renderer buffers the graph points at were re-allocated since capture."""
        g = self._igraph
        self._check_epoch(g)
        sb = g["sb"]
        if len(image_index) != g["k"]:
            raise ValueError(f"the graph was captured for {g['k']} images per step")
        idx = image_index if torch.is_tensor(image_index) else torch.tensor([int(i) for i in image_index], dtype=torch.int32)
        sb["img"].copy_(idx, non_blocking=True)
        if sb["draws"] is not None:
            if draws is None:
                raise ValueError("the graph was captured with device_draws=False: pass the draws")
            sb["draws"].copy_(draws.reshape(-1)[:sb["draws"].numel()], non_blocking=True)
        self._own_engine()
        g["graph"].replay()
        self._stepped()
        return self.loss[:2]
