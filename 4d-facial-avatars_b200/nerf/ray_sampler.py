"""The per-iteration ray selection of train_transformed_rays.py:230-239 (importance maps) and :303-331 (np.random.choice +
gathers) on the device (SURVEY.md §8f rank 3): nfb_sample_rays returns the indices numpy would return for the same uniform
draws, bit for bit, and gathers ray origins / directions, target and background colours of the selected pixels in the same launch."""
import copy
import ctypes as C

import numpy as np
import torch

from . import _capi as capi
from . import _engine


def importance_map(height, width, bbox, p=0.9):
    """The reference's per-image probability map (:232-238), evaluated with numpy exactly as the script does, reduced to what the
    device sampler needs: the two values of the normalised map and the box.  Returns (NfbRayMap, flat float64 map)."""
    probs = np.zeros((height, width))
    probs.fill(1 - p)
    probs[bbox[0]:bbox[1], bbox[2]:bbox[3]] = p
    probs = (1 / probs.sum()) * probs
    b = [int(max(0, min(bbox[0], height))), int(max(0, min(bbox[1], height))), int(max(0, min(bbox[2], width))), int(max(0, min(bbox[3], width)))]
    inside = b[1] > b[0] and b[3] > b[2]
    q_in = float(probs[b[0], b[2]]) if inside else float(probs[0, 0])
    outside = np.ones((height, width), dtype=bool)
    if inside:
        outside[b[0]:b[1], b[2]:b[3]] = False
    q_out = float(probs[outside][0]) if outside.any() else q_in
    if not inside:
        b = [0, 0, 0, 0]
    m = capi.NfbRayMap(int(height), int(width), (C.c_int32 * 4)(*b), q_out, q_in)
    return m, probs.reshape(-1)


class RaySampler:
    def __init__(self, height, width, bboxs, p=0.9, size=2048, device=None):
        self.H, self.W, self.size = int(height), int(width), int(size)
        self.dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.eng = _engine.renderer_for(self.dev)
        self.maps = [importance_map(self.H, self.W, [int(v) for v in bb], p)[0] for bb in bboxs]
        self._state = torch.zeros(3, dtype=torch.int32, device=self.dev)

    def sample(self, img_idx, draws=None, pose=None, intrinsics=None, image=None, background=None, max_rounds=8, numpy_lockstep=False):
        """Select `size` distinct pixels of training image img_idx.  draws: float64 CUDA tensor consumed like RandomState.rand inside
        np.random.choice (None: torch.rand on the device; numpy_lockstep=True: np.random.rand on the host, round by round, so the
        global numpy stream advances exactly as the reference's call would).  Returns a dict with `indices` (int64, numpy's order)
        and, when their inputs are given, ray_origins / ray_directions (pose + intrinsics), target (image), background, pixel_rc."""
        dev, n = self.dev, self.size
        idx = torch.empty(n, dtype=torch.int64, device=dev)
        out = dict(indices=idx, pixel_rc=torch.empty((n, 2), dtype=torch.int32, device=dev))
        g = capi.NfbRayGather()
        g.pixel_rc = out["pixel_rc"].data_ptr()
        keep = []
        if pose is not None:
            p34 = pose.detach().cpu().float().reshape(-1)[:12]
            for i in range(12):
                g.pose[i] = float(p34[i])
            for i in range(4):
                g.intrinsics[i] = float(intrinsics[i])
            out["ray_origins"], out["ray_directions"] = torch.empty((n, 3), device=dev), torch.empty((n, 3), device=dev)
            g.ray_origins, g.ray_directions = out["ray_origins"].data_ptr(), out["ray_directions"].data_ptr()
        for name, src, field_in, field_out in (("target", image, "image", "target"), ("background", background, "background", "background_out")):
            if src is not None:
                t = _engine._f32c(src, dev).reshape(self.H, self.W, 3)
                keep.append(t)
                out[name] = torch.empty((n, 3), device=dev)
                setattr(g, field_in, t.data_ptr())
                setattr(g, field_out, out[name].data_ptr())
        self._state.zero_()
        call = lambda d, rounds: capi.check(capi.lib.nfb_sample_rays(  # noqa: E731
            self.eng._h, C.byref(self.maps[img_idx]), C.c_void_p(d.data_ptr()), n, rounds, C.c_void_p(idx.data_ptr()),
            C.c_void_p(self._state.data_ptr()), C.byref(g), _engine._stream()), "sample_rays")
        if numpy_lockstep:
            buf = torch.empty(max_rounds * n, dtype=torch.float64, device=dev)
            used = found = rounds = 0
            while found < n and rounds < max_rounds:
                x = np.random.rand(n - found)  # the draw RandomState.choice makes at this point
                buf[used:used + x.size] = torch.from_numpy(x).to(dev)
                call(buf, 1)
                found, used = int(self._state[0]), used + x.size
                rounds += 1
        else:
            if draws is None:
                draws = torch.rand(max_rounds * n, dtype=torch.float64, device=dev)
            call(draws, max_rounds)
        out["_keep"] = keep + [draws] if draws is not None else keep
        out["state"] = self._state
        return out


class TrainImages:
    """The training set as nfb_sample_rays_images reads it (NfbTrainImages), built once: the importance map of every image
    (importance_map above), poses [N,12], expressions [N,76] on the device, and the images [N,H,W,3] FP32 — kept where they are
    when on the device, otherwise pinned in host memory, from which the sampler reads only the selected pixels.  background:
    optional [H,W,3], one for the whole set."""

    def __init__(self, images, poses, expressions, bboxs, intrinsics, background=None, p=0.9, device=None):
        self.dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        n, H, W = images.shape[0], images.shape[1], images.shape[2]
        if images.shape[3] != 3 or len(bboxs) != n or poses.shape[0] != n or expressions.shape[0] != n:
            raise ValueError("images [N,H,W,3], poses [N,...], expressions [N,76] and N boxes")
        self.n_images, self.H, self.W = int(n), int(H), int(W)
        maps = (capi.NfbRayMap * n)(*[importance_map(H, W, [int(v) for v in bb], p)[0] for bb in bboxs])
        self.maps = torch.frombuffer(bytearray(bytes(maps)), dtype=torch.uint8).to(self.dev)
        self.poses = poses.detach().to(device=self.dev, dtype=torch.float32).reshape(n, -1)[:, :12].contiguous()
        self.expressions = _engine._f32c(expressions, self.dev).reshape(n, 76)
        self.images = self._keep_in_place(images)
        self.background = self._keep_in_place(background.reshape(H, W, 3)) if background is not None else None
        self.intrinsics = [float(v) for v in intrinsics]
        self.desc = capi.NfbTrainImages(self.maps.data_ptr(), self.poses.data_ptr(), self.expressions.data_ptr(),
                                        self.images.data_ptr(), self.background.data_ptr() if self.background is not None else None,
                                        self.n_images, self.H, self.W, 0, (C.c_double * 4)(*self.intrinsics))

    def alias_tables(self, poses, expressions):
        """Point the descriptor's pose and expression tables at caller-owned rows instead of this object's copies: poses [N,12] and
        expressions [N,76], contiguous FP32 tensors on this device, read in place by every later sampler call (and by every
        replay of a graph captured over one), so that writes into them change the rays and conditioning rows drawn next.  The
        caller keeps them alive while this object is used.  (The fitter's parameter tables are such rows.)"""
        for name, t, w in (("poses", poses, 12), ("expressions", expressions, 76)):
            if (t.dtype != torch.float32 or t.device != self.dev or tuple(t.shape) != (self.n_images, w) or not t.is_contiguous()):
                raise ValueError(f"{name} must be a contiguous FP32 [{self.n_images},{w}] tensor on {self.dev}")
        self.poses, self.expressions = poses, expressions
        self.desc.poses, self.desc.expressions = poses.data_ptr(), expressions.data_ptr()

    def with_background(self, background):
        """A copy of this set whose sampler reads `background` ([H,W,3] contiguous FP32 on this device) in place: every later
        sampler call, and every replay of a graph captured over one, gathers what the table holds then (a trainer's learned
        background is such a table).  The copy shares every other table with this object, which is left unchanged.  The caller
        keeps `background` alive while the copy is used."""
        if (background.dtype != torch.float32 or background.device != self.dev or tuple(background.shape) != (self.H, self.W, 3)
                or not background.is_contiguous()):
            raise ValueError(f"the background must be a contiguous FP32 [{self.H},{self.W},3] tensor on {self.dev}")
        view = copy.copy(self)
        view.background = background
        view.desc = capi.NfbTrainImages.from_buffer_copy(self.desc)
        view.desc.background = background.data_ptr()
        return view

    def _keep_in_place(self, t):
        if t.is_cuda:
            return t.detach().to(device=self.dev, dtype=torch.float32).contiguous()
        t = t.detach().to(dtype=torch.float32).contiguous()
        return t if t.is_pinned() else t.pin_memory()


def frame_products(rgb, disparity, w_last, intrinsics, want_disparity=False, like_torch_cpu=False):
    """cast_to_image / torch_normal_map(clean=True) / cast_to_disparity_image of eval_transformed_rays.py (:84-119, :184-198) on
    the device, one launch: [H,W,3] rgb, [H,W] disparity and last-sample weights -> uint8 tensors (rgb, normals [(H-1),(W-1),3],
    optionally the disparity image).  like_torch_cpu: round like torch's CPU back end instead of its CUDA back end (include/nfb.h: NFB_PRODUCTS_LIKE_TORCH_CPU)."""
    dev = rgb.device
    eng = _engine.renderer_for(dev)
    H, W = disparity.shape
    rgb, disparity = _engine._f32c(rgb, dev), _engine._f32c(disparity, dev)
    w_last = _engine._f32c(w_last, dev) if w_last is not None else None
    out_rgb = torch.empty((H, W, 3), dtype=torch.uint8, device=dev)
    out_n = torch.empty((H - 1, W - 1, 3), dtype=torch.uint8, device=dev)
    out_d = torch.empty((H, W), dtype=torch.uint8, device=dev) if want_disparity else None
    intr = (C.c_double * 4)(*[float(v) for v in intrinsics])
    capi.check(capi.lib.nfb_frame_products(eng._h, _engine._ptr(rgb), _engine._ptr(disparity), _engine._ptr(w_last), intr, H, W,
                                           _engine._ptr(out_rgb), _engine._ptr(out_n), _engine._ptr(out_d), 1 if like_torch_cpu else 0,
                                           _engine._stream()),
               "frame_products")
    return out_rgb, out_n, out_d
