"""Host-side engine: owns NfbHandle objects, keeps the packed weight streams in sync with the caller's
FP32 nn.Parameters, and launches the fused render kernel on torch's current CUDA stream.

torch is used here only for device memory, streams and (in the trainer) torch.distributed."""
import ctypes as C
import os
import weakref

import torch

from . import _capi as capi

PARAM_ORDER = ([f"layers_xyz.{i}.{k}" for i in range(6) for k in ("weight", "bias")]
               + ["fc_feat.weight", "fc_feat.bias", "fc_alpha.weight", "fc_alpha.bias"]
               + [f"layers_dir.{i}.{k}" for i in range(4) for k in ("weight", "bias")]
               + ["fc_rgb.weight", "fc_rgb.bias"])
# Members of NfbInputGrads (include/nfb.h): the input gradients Renderer.backward can return.
INPUT_GRADS = ("ray_origins", "ray_directions", "dir_z", "background", "expression")

_precision = os.environ.get("NFB_PRECISION", "fast")


# precision name -> NfbSampling.precision (include/nfb.h NFB_PREC_*)
PRECISIONS = {"fast": capi.NFB_PREC_FAST, "exact": capi.NFB_PREC_EXACT, "exact_grad": capi.NFB_PREC_EXACT_GRAD}


def set_precision(mode: str):
    """'fast' = FP16 operands / FP32 accumulate; 'exact' = 3-pass FP16 hi/lo split of the forward; 'exact_grad' = exact's forward
    and a hi/lo backward (see include/nfb.h)."""
    global _precision
    if mode not in PRECISIONS:
        raise ValueError("precision must be 'fast', 'exact' or 'exact_grad'")
    _precision = mode


def get_precision() -> str:
    return _precision


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _f32c(t, device):
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


OUTPUTS = ("rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last")  # members of NfbOutputs


def _ptrs(tensors):
    """The C array of 26 pointers (PARAM_ORDER) the library takes for one network's parameters or gradients; None entries are
    null, and None gives a null array."""
    return (C.c_void_p * 26)(*[(t.data_ptr() if t is not None else None) for t in tensors]) if tensors is not None else None


def _outputs(out, has_fine):
    """NfbOutputs pointing at the seven tensors of `out` (the fine ones null without a fine network)."""
    return capi.NfbOutputs(*[(out[k].data_ptr() if has_fine or not k.endswith("_fine") else None) for k in OUTPUTS])


def _out_grads(out_grads, device, keep):
    """NfbOutGrads from 7 tensors or None in OUTPUTS order; the FP32 copies handed to the library are appended to `keep`."""
    og = capi.NfbOutGrads()
    for field, g in zip(OUTPUTS, out_grads):
        if g is not None:
            g = _f32c(g, device)
            keep.append(g)
            setattr(og, field, g.data_ptr())
    return og


class Renderer:
    """One NfbHandle on one CUDA device plus the bookkeeping that decides when weights must be re-packed."""

    def __init__(self, device: torch.device):
        if device.type != "cuda":
            raise RuntimeError("the nfb render path runs on CUDA (sm_90a) only; there is no CPU fallback")
        self.device = device
        idx = device.index if device.index is not None else torch.cuda.current_device()
        dims = capi.NfbModelDims(10, 4, 1, 0, 76, 32)
        h = C.c_void_p()
        capi.check(capi.lib.nfb_create(C.byref(dims), idx, C.byref(h)), "create")
        self._h = h
        self._lin = {}
        self._plist = {}
        self.packed_owner = None   # the FusedTrainer whose weights the packed streams hold (None: whatever sync_weights packed last)
        self._versions = [None, None]
        self._keep = [None, None]  # contiguous FP32 copies handed to the pack kernels
        self.train_token = 0       # bumped by every training forward: the handle keeps ONE saved state
        self.train_rays = 0        # rays of that forward
        self.n_frames = 0          # frames of the last set_frames
        self.train_frames = None   # frames of the last training forward when it was a multi-frame one
        weakref.finalize(self, capi.lib.nfb_destroy, h)

    def _params(self, model):
        """The model's 26 parameters in PARAM_ORDER; the walk over named_parameters() is cached per module object."""
        cached = self._plist.get(id(model))
        if cached is None or cached[0]() is not model:
            sd = dict(model.named_parameters())
            cached = self._plist[id(model)] = (weakref.ref(model), [sd[k] for k in PARAM_ORDER])
        return cached[1]

    def _fingerprint(self, model):
        """(identity, storage, in-place version) of every parameter.  Writes that bypass autograd's version counter
        (`p.data.copy_()`, external kernels) are invisible here: call invalidate() after them."""
        return (id(model),) + tuple((p.data_ptr(), p._version) for p in self._params(model))

    def invalidate(self):
        """Force a re-pack of both networks at the next render (after parameter writes torch cannot see)."""
        self._versions = [None, None]

    def mark_synced(self, model_coarse, model_fine):
        """The packed streams already hold these models' current values (the fused optimizer step re-packed them)."""
        self._versions[0] = self._fingerprint(model_coarse)
        if model_fine is not None:
            self._versions[1] = self._fingerprint(model_fine)

    def sync_weights(self, model_coarse, model_fine):
        for which, model in ((capi.NFB_NET_COARSE, model_coarse), (capi.NFB_NET_FINE, model_fine)):
            if model is None:
                continue
            fp = self._fingerprint(model)
            if fp == self._versions[which]:
                continue
            tensors = [_f32c(t, self.device) for t in self._params(model)]
            capi.check(capi.lib.nfb_load_weights(self._h, which, _ptrs(tensors), _stream()), "load_weights")
            self.packed_owner = None
            self._keep[which] = tensors
            self._versions[which] = fp

    def linspace(self, n):
        """torch.linspace(0, 1, n) evaluated by ATen's CPU kernel (whose vectorised halves are not the scalar
        formula of nfb_host_linspace) and cached on the device, so depths match the CPU reference bit for bit."""
        t = self._lin.get(n)
        if t is None:
            t = self._lin[n] = torch.linspace(0.0, 1.0, n, dtype=torch.float32).to(self.device)
        return t

    def _sampling(self, num_coarse, num_fine, precision, white_bkgd, perturb=False, noise_std=0.0):
        prec = precision or _precision
        if prec not in PRECISIONS:  # a misspelt mode must not quietly train in another one
            raise ValueError(f"precision must be 'fast', 'exact' or 'exact_grad', not {prec!r}")
        return capi.NfbSampling(num_coarse, num_fine, int(bool(perturb)), float(noise_std), int(bool(white_bkgd)), 0,
                                PRECISIONS[prec], self.linspace(num_coarse).data_ptr(),
                                self.linspace(num_fine).data_ptr() if num_fine > 0 else None)

    def set_frame(self, expressions, latent_code):
        e = _f32c(expressions, self.device).reshape(-1)
        l = _f32c(latent_code, self.device).reshape(-1)
        if e.numel() != 76 or l.numel() != 32:
            raise ValueError("expressions must have 76 and latent_code 32 elements")
        capi.check(capi.lib.nfb_set_frame(self._h, _ptr(e), _ptr(l), _stream()), "set_frame")
        self._frame = (e, l)

    def set_frames(self, expressions, latent_codes):
        """nfb_set_frames: expressions [F,76], latent_codes [F,32] -> the frame table a `frame_index` render reads."""
        e = _f32c(expressions, self.device).reshape(-1, 76)
        l = _f32c(latent_codes, self.device).reshape(-1, 32)
        if e.shape[0] != l.shape[0] or e.shape[0] < 1:
            raise ValueError("expressions [F,76] and latent_codes [F,32] must have the same F >= 1")
        capi.check(capi.lib.nfb_set_frames(self._h, _ptr(e), _ptr(l), e.shape[0], _stream()), "set_frames")
        self._frames = (e, l)
        self.n_frames = e.shape[0]

    def kernel_info(self, precision="fast"):
        """Which render kernel an evaluation call runs (bench.py): one kernel, both precision modes."""
        return dict(name="nfb::render_kernel", block_size=384)

    def launch_count(self) -> int:
        n = C.c_longlong()
        capi.check(capi.lib.nfb_launch_count(self._h, C.byref(n)))
        return n.value

    def buffer_epoch(self) -> int:
        """nfb_buffer_epoch: changes whenever the handle frees or refills a buffer a captured training step points at."""
        n = C.c_longlong()
        capi.check(capi.lib.nfb_buffer_epoch(self._h, C.byref(n)))
        return n.value

    def render(self, ro, rd, near, far, num_coarse, num_fine, perturb=False, noise_std=0.0, white_bkgd=False,
               background=None, dir_z=None, noise=None, precision=None, debug=False, act_step=None, train=False, frame_index=None):
        """ro, rd: [N,3] CUDA FP32.  noise: dict with t_rand, n_c, u, n_f (any may be None).  Returns a dict
        with the seven outputs (+ per-sample dumps when debug).  train=True: nfb_render_forward_train (the handle keeps
        the state `backward` consumes).  frame_index: [N] int32-convertible CUDA tensor -> a multi-frame call over the frames of
        set_frames (nfb_render_forward_frames[_train]; no debug dumps)."""
        dev = self.device
        ro, rd = _f32c(ro, dev), _f32c(rd, dev)
        n = ro.shape[0]
        has_fine = num_fine > 0
        out = {k: torch.empty((n, 3) if k.startswith("rgb") else (n,), device=dev, dtype=torch.float32)
               for k in OUTPUTS if has_fine or not k.endswith("_fine")}
        rays = capi.NfbRays()
        rays.o, rays.d, rays.n_rays = ro.data_ptr(), rd.data_ptr(), n
        rays.near_, rays.far_ = float(near), float(far)
        keep = [ro, rd]
        if background is not None:
            bg = _f32c(background, dev).reshape(n, 3)
            rays.background = bg.data_ptr()
            keep.append(bg)
        if dir_z is not None:
            dz = _f32c(dir_z, dev).reshape(n)
            rays.dir_z = dz.data_ptr()
            keep.append(dz)
        sm = self._sampling(num_coarse, num_fine, precision, white_bkgd, perturb, noise_std)
        nz = capi.NfbNoise()
        if noise:
            for field, key in (("t_rand", "t_rand"), ("sigma_noise_c", "n_c"), ("u", "u"), ("sigma_noise_f", "n_f")):
                t = noise.get(key)
                if t is not None:
                    t = _f32c(t, dev)
                    keep.append(t)
                    setattr(nz, field, t.data_ptr())
        o = _outputs(out, has_fine)
        dbg = None
        if debug or act_step is not None:
            dbg = self._debug_dumps(out, n, num_coarse, num_fine)
            if act_step is not None:
                out["act"] = torch.zeros((128, 256), device=dev)
                dbg.act_dump, dbg.act_step = out["act"].data_ptr(), int(act_step)
        if frame_index is not None:
            if dbg is not None:
                raise ValueError("a multi-frame render takes no debug dumps")
            fi = frame_index.detach().to(device=dev, dtype=torch.int32).reshape(n).contiguous()
            keep.append(fi)
        if train:
            self.train_token += 1
            self.train_rays = n
            self.train_frames = self.n_frames if frame_index is not None else None
        nzp = C.byref(nz) if noise else None
        if frame_index is not None:
            fn = capi.lib.nfb_render_forward_frames_train if train else capi.lib.nfb_render_forward_frames
            capi.check(fn(self._h, C.byref(rays), _ptr(fi), C.byref(sm), nzp, C.byref(o), _stream()), "render_forward_frames")
        elif train:
            capi.check(capi.lib.nfb_render_forward_train(self._h, C.byref(rays), C.byref(sm), nzp, C.byref(o), _stream()),
                       "render_forward_train")
        else:
            capi.check(capi.lib.nfb_render_forward(self._h, C.byref(rays), C.byref(sm), nzp, C.byref(o),
                                                   C.byref(dbg) if dbg is not None else None, _stream()), "render_forward")
        out["_keep"] = keep  # inputs must outlive the asynchronous launch
        return out

    def _debug_dumps(self, out, n, num_coarse, num_fine):
        """NfbDebug with the per-sample dumps (depths and MLP outputs of both passes) allocated into `out`."""
        dev = self.device
        out["z_coarse"] = torch.zeros((n, num_coarse), device=dev)
        out["raw_coarse"] = torch.zeros((n, num_coarse, 4), device=dev)
        dbg = capi.NfbDebug(out["z_coarse"].data_ptr(), out["raw_coarse"].data_ptr(), None, None, None, 0)
        if num_fine > 0:
            s = num_coarse + num_fine
            out["z_fine"] = torch.zeros((n, s), device=dev)
            out["raw_fine"] = torch.zeros((n, s, 4), device=dev)
            dbg.z_fine, dbg.raw_fine = out["z_fine"].data_ptr(), out["raw_fine"].data_ptr()
        return dbg

    def loss_mse_grad(self, rgb_c, rgb_f, target, n_total, grad_c, grad_f, loss):
        """nfb_loss_mse_grad: d mse / d rgb into grad_c / grad_f ([n,3] CUDA buffers), loss[0:2] += this shard's share."""
        n = rgb_c.shape[0]
        capi.check(capi.lib.nfb_loss_mse_grad(self._h, _ptr(rgb_c), _ptr(rgb_f), _ptr(target), n, int(n_total), _ptr(grad_c),
                                              _ptr(grad_f), _ptr(loss), _stream()), "loss_mse_grad")

    def adam_step(self, params, grads, exp_avg, exp_avg_sq, lr, step, betas=(0.9, 0.999), eps=1e-8, grad_scale=1.0,
                  reg_offset=-1, reg_weight=0.0):
        """nfb_adam_step over flat FP32 CUDA buffers (in place; grads are zeroed)."""
        hp = capi.NfbAdam(float(lr), float(betas[0]), float(betas[1]), float(eps), int(step), float(grad_scale), int(reg_offset),
                          float(reg_weight))
        capi.check(capi.lib.nfb_adam_step(self._h, _ptr(params), _ptr(grads), _ptr(exp_avg), _ptr(exp_avg_sq), params.numel(),
                                          C.byref(hp), _stream()), "adam_step")

    def adam_step_dev(self, params, grads, exp_avg, exp_avg_sq, dev_state):
        """nfb_adam_step_dev: like adam_step with step counter / LR schedule / regularised row in the device struct `dev_state`
        (a uint8 CUDA tensor holding an NfbAdamDev) — capturable in a CUDA graph."""
        capi.check(capi.lib.nfb_adam_step_dev(self._h, _ptr(params), _ptr(grads), _ptr(exp_avg), _ptr(exp_avg_sq), params.numel(),
                                              _ptr(dev_state), _stream()), "adam_step_dev")

    def repack(self, params_c, params_f):
        """nfb_repack: both networks' FP32 parameter tensors (lists in PARAM_ORDER) -> kernel-layout streams, one launch."""
        capi.check(capi.lib.nfb_repack(self._h, _ptrs(params_c), _ptrs(params_f), _stream()), "repack")

    def backward_into(self, out_grads, params_c, params_f, grads_c, grads_f, grad_latent, frames=False, grad_expressions=None,
                      grad_ray_origins=None, grad_ray_directions=None, grad_background=None):
        """nfb_render_backward writing straight into caller-owned gradient tensors (views of a flat bucket): params_* / grads_*
        are lists of 26 contiguous FP32 CUDA tensors in PARAM_ORDER (grads of layers_dir.3.* may be None; grads_c and grads_f
        both None: input-only mode).  frames=True: nfb_render_backward_frames after a multi-frame training forward, per-frame
        d latent into grad_latent [F,32], and into caller-owned buffers too d expression [F,76] (grad_expressions) and the per-ray
        ray gradients [N,3] (grad_ray_origins, grad_ray_directions), each when given.  grad_background: the per-ray background
        gradient [N,3] (NfbInputGrads.background; the single-frame call is then nfb_render_backward_ex)."""
        keep = []
        args = (self._h, C.byref(_out_grads(out_grads, self.device, keep)), _ptrs(params_c), _ptrs(params_f), _ptrs(grads_c),
                _ptrs(grads_f), _ptr(grad_latent))
        ig = None
        if grad_ray_origins is not None or grad_ray_directions is not None or grad_background is not None:
            ig = capi.NfbInputGrads(ray_origins=_ptr(grad_ray_origins), ray_directions=_ptr(grad_ray_directions),
                                    background=_ptr(grad_background))
        if frames:
            capi.check(capi.lib.nfb_render_backward_frames(*args, _ptr(grad_expressions) if grad_expressions is not None else None,
                                                           C.byref(ig) if ig is not None else None, _stream()), "render_backward_frames")
        elif ig is not None:
            capi.check(capi.lib.nfb_render_backward_ex(*args, C.byref(ig), _stream()), "render_backward")
        else:
            capi.check(capi.lib.nfb_render_backward(*args, _stream()), "render_backward")
        self._bwd_keep = keep

    def sample_images(self, data, image_index, n, draws, max_rounds, latent_table, out):
        """nfb_sample_rays_images: data = ray_sampler.TrainImages, image_index = int32 CUDA [K], draws = float64 CUDA
        [K * max_rounds * n], latent_table = [n_images,32] CUDA; out = dict of CUDA tensors named like NfbImageBatch's members
        (missing keys: not written)."""
        b = capi.NfbImageBatch()
        for name, _ in capi.NfbImageBatch._fields_:
            t = out.get(name)
            if t is not None:
                setattr(b, name, t.data_ptr())
        capi.check(capi.lib.nfb_sample_rays_images(self._h, C.byref(data.desc), _ptr(image_index), image_index.numel(), int(n),
                                                   _ptr(draws), int(max_rounds), _ptr(latent_table), C.byref(b), _stream()),
                   "sample_rays_images")

    def latent_rows_grad(self, grad_latents, image_index, table, table_grads, reg_weight):
        """nfb_latent_rows_grad: table_grads[image_index[k]] += grad_latents[k] in ascending k, then the regulariser terms
        reg_weight * l / ||l|| in ascending k (all CUDA tensors; image_index int32 [K])."""
        capi.check(capi.lib.nfb_latent_rows_grad(self._h, _ptr(grad_latents), _ptr(image_index), image_index.numel(), _ptr(table),
                                                 table.shape[0], _ptr(table_grads), float(reg_weight), _stream()), "latent_rows_grad")

    def fit_rows_grad(self, data, image_index, n, pixel_rc, grad_ray_origins, grad_ray_directions, pose_grads, grad_expressions,
                      expression_grads):
        """nfb_fit_rows_grad: pose_grads[image_index[k]] ([n_images,12]) += slot k's pose gradient from the per-ray ray gradients at
        pixel_rc, and expression_grads[image_index[k]] ([n_images,76]) += grad_expressions[k], in ascending k (CUDA tensors; any
        pair may be None; data = ray_sampler.TrainImages)."""
        capi.check(capi.lib.nfb_fit_rows_grad(self._h, C.byref(data.desc), _ptr(image_index), image_index.numel(), int(n), _ptr(pixel_rc),
                                              _ptr(grad_ray_origins), _ptr(grad_ray_directions), _ptr(pose_grads), _ptr(grad_expressions),
                                              _ptr(expression_grads), _stream()), "fit_rows_grad")

    def background_rows_grad(self, pixel_rc, height, width, grad_bg_render, grad_bg_loss, table_grads):
        """nfb_background_rows_grad: table_grads ([H,W,3] or its flat view) += each ray's background gradient (grad_bg_render
        [+ grad_bg_loss], [n,3]) at its pixel_rc ([n,2] int32), in ascending ray order (CUDA tensors; grad_bg_loss may be None)."""
        capi.check(capi.lib.nfb_background_rows_grad(self._h, _ptr(pixel_rc), pixel_rc.shape[0], int(height), int(width),
                                                     _ptr(grad_bg_render), _ptr(grad_bg_loss), _ptr(table_grads), _stream()),
                   "background_rows_grad")

    def loss_background_grad(self, bg_rays, target, w_last, n_total, weight, grad_bg_rays, grad_w_last, loss):
        """nfb_loss_background_grad: weight * mean(w_last * ||bg - target||^2) over n_total rays; writes grad_bg_rays [n,3] and
        grad_w_last [n], loss[0] += this shard's share (CUDA tensors)."""
        capi.check(capi.lib.nfb_loss_background_grad(self._h, _ptr(bg_rays), _ptr(target), _ptr(w_last), bg_rays.shape[0],
                                                     int(n_total), float(weight), _ptr(grad_bg_rays), _ptr(grad_w_last), _ptr(loss),
                                                     _stream()), "loss_background_grad")

    def backward(self, out_grads, params_c, params_f, want_latent=True, want_params=True, inputs=None, frames=False):
        """nfb_render_backward_ex for the last training forward.  out_grads: 7 CUDA tensors or None (rgb_c, disp_c, acc_c,
        rgb_f, disp_f, acc_f, w_last); params_*: the 26 FP32 parameter tensors in PARAM_ORDER (params_f None without a
        fine network).  Returns (grads_c, grads_f, grad_latent) — lists aligned with PARAM_ORDER, None for layers_dir.3.*.
        inputs: names of the input gradients wanted, out of INPUT_GRADS ("ray_origins", "ray_directions", "dir_z", "background",
        "expression"); then a 4th element, a dict name -> tensor, is returned.  want_params=False: input-only backward (no
        parameter gradient is formed; grads_c / grads_f are None).  frames=True: nfb_render_backward_frames after a multi-frame
        forward; grad_latent is then [F,32], and "expression" in `inputs` yields [F,76]."""
        dev = self.device
        if frames and self.train_frames is None:
            raise RuntimeError("backward(frames=True) needs a multi-frame training forward (render(..., train=True, "
                               "frame_index=...)); the last training forward was a single-frame one")
        keep = []
        og = _out_grads(out_grads, dev, keep)

        def pack(params):
            if params is None:
                return None, None
            ps = [_f32c(t, dev) for t in params]
            keep.extend(ps)
            return ps, [None if k.startswith("layers_dir.3") else torch.empty_like(p) for k, p in zip(PARAM_ORDER, ps)]

        pc, grads_c = pack(params_c)
        pf, grads_f = pack(params_f)
        if not want_params:
            grads_c = grads_f = None
        n, nfr = self.train_rays, self.train_frames
        shapes = dict(ray_origins=(n, 3), ray_directions=(n, 3), dir_z=(n,), background=(n, 3),
                      expression=(nfr, 76) if frames else (76,))
        ing = {name: torch.empty(shapes[name], device=dev, dtype=torch.float32) for name in (inputs or ())}
        # the single-frame backward takes a null NfbInputGrads when no input gradient is asked for; the multi-frame one always
        # takes the struct, and returns d expression [F,76] through its own argument instead
        ig = capi.NfbInputGrads() if frames or inputs is not None else None
        for name, t in ing.items():
            if not (frames and name == "expression"):
                setattr(ig, name, t.data_ptr())
        glat = torch.empty((nfr, 32) if frames else 32, device=dev, dtype=torch.float32) if want_latent else None
        args = (self._h, C.byref(og), _ptrs(pc), _ptrs(pf), _ptrs(grads_c), _ptrs(grads_f), _ptr(glat))
        if frames:
            capi.check(capi.lib.nfb_render_backward_frames(*args, _ptr(ing.get("expression")), C.byref(ig), _stream()),
                       "render_backward_frames")
        else:
            capi.check(capi.lib.nfb_render_backward_ex(*args, C.byref(ig) if ig is not None else None, _stream()), "render_backward")
        self._bwd_keep = keep
        return (grads_c, grads_f, glat, ing) if inputs is not None else (grads_c, grads_f, glat)

    def train_debug(self):
        d = capi.NfbTrainDebug()
        capi.check(capi.lib.nfb_train_debug(self._h, C.byref(d)), "train_debug")
        return d

    def weights_debug(self, net):
        """nfb_debug_weights: device pointers and sizes of network `net`'s packed weight buffers (an NfbWeightDebug)."""
        d = capi.NfbWeightDebug()
        capi.check(capi.lib.nfb_debug_weights(self._h, int(net), C.byref(d)), "debug_weights")
        return d

    def render_camera(self, pose, intrinsics, height, width, row_begin, rows, near, far, num_coarse, num_fine,
                      background=None, out=None, precision=None, white_bkgd=False, prof=None, debug=False):
        """Deterministic render of image rows [row_begin, row_begin+rows) with in-kernel ray generation
        (no o/d tensors in HBM).  pose: 3x4 / 4x4 CPU tensor; background: [rows*width,3] CUDA tensor or None.
        `out`: optional preallocated [11, rows*width] CUDA buffer; returns the dict of output views (+ the per-sample
        dumps of `render` when debug)."""
        dev = self.device
        n = rows * width
        if out is None:
            out = torch.empty((11, n), device=dev, dtype=torch.float32)
        flat = out.view(-1)
        views = dict(rgb_coarse=flat[0:3 * n].view(n, 3), disp_coarse=flat[3 * n:4 * n], acc_coarse=flat[4 * n:5 * n],
                     rgb_fine=flat[5 * n:8 * n].view(n, 3), disp_fine=flat[8 * n:9 * n], acc_fine=flat[9 * n:10 * n],
                     w_last=flat[10 * n:11 * n])
        rays = capi.NfbRays()
        rays.n_rays = n
        p = pose.detach().cpu().float().reshape(-1)
        rows34 = p[:12] if p.numel() in (12, 16) else None
        for i in range(12):
            rays.pose[i] = float(rows34[i])
        for i in range(4):
            rays.intrinsics[i] = float(intrinsics[i])
        rays.height, rays.width, rays.row_begin = height, width, row_begin
        rays.near_, rays.far_ = float(near), float(far)
        if background is not None:
            rays.background = background.data_ptr()
        sm = self._sampling(num_coarse, num_fine, precision, white_bkgd)
        o = _outputs(views, num_fine > 0)
        dbg = self._debug_dumps(views, n, num_coarse, num_fine) if debug else None
        if prof is not None:  # int64[64] CUDA tensor of phase-cycle counters
            if dbg is None:
                dbg = capi.NfbDebug()
            dbg.prof = prof.data_ptr()
        capi.check(capi.lib.nfb_render_forward(self._h, C.byref(rays), C.byref(sm), None, C.byref(o),
                                               C.byref(dbg) if dbg is not None else None, _stream()), "render_forward")
        views["_buf"] = out
        return views

    def render_frame_host(self, pose, intrinsics, height, width, row_begin, rows, near, far, expr_host, latent_host,
                          bg_host, num_coarse, num_fine, out_host, precision=None, white_bkgd=False):
        """Host-buffer end-to-end call (bench e2e leg).  All tensors are CPU (ideally pinned) FP32."""
        sm = self._sampling(num_coarse, num_fine, precision, white_bkgd)
        pose_a = (C.c_float * 12)(*[float(v) for v in pose.reshape(-1)[:12]])
        intr_a = (C.c_double * 4)(*[float(v) for v in intrinsics])
        capi.check(capi.lib.nfb_render_frame_host(self._h, pose_a, intr_a, height, width, row_begin, rows, float(near),
                                                  float(far), _ptr(expr_host), _ptr(latent_host), _ptr(bg_host),
                                                  C.byref(sm), _ptr(out_host), _stream()), "render_frame_host")


_renderers = {}


def renderer_for(device: torch.device) -> Renderer:
    if device.type != "cuda":
        raise RuntimeError("the nfb render path runs on CUDA (sm_90a) only; there is no CPU fallback")
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    r = _renderers.get(key)
    if r is None:
        r = _renderers[key] = Renderer(torch.device("cuda", key[1]))
    return r
