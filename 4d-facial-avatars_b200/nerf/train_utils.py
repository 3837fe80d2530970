"""Render driver with the reference's call surface (nerf/train_utils.py:36-290), backed by the fused sm_90a
kernel.  What stays on the host: argument plumbing, the reference's chunk-ordered noise draws, output reshaping."""
import torch

from . import _engine


def _mode_opts(options, mode):
    o = getattr(options.nerf, mode)
    return dict(num_coarse=int(o.num_coarse), num_fine=int(getattr(o, "num_fine", 0)), perturb=bool(o.perturb),
                lindisp=bool(getattr(o, "lindisp", False)), noise_std=float(getattr(o, "radiance_field_noise_std", 0.0)),
                white_bkgd=bool(getattr(o, "white_background", False)), chunksize=int(o.chunksize))


def _check_ndc(options):
    if options.dataset.no_ndc is False:
        raise NotImplementedError("NDC rays are not implemented (every shipped config sets no_ndc: True)")


def _check_models(model_coarse, model_fine):
    for m in (model_coarse, model_fine):
        if m is not None and not (hasattr(m, "fused_supported") and m.fused_supported()):
            raise NotImplementedError("the fused render path implements ConditionalBlendshapePaperNeRFModel with the "
                                      "shipped encoder sizes (xyz 10 + input, dir 4 without input, 76 + 32 conditioning)")


def _draw_noise(n, opts, device, has_fine):
    """Per-chunk draws in the reference's order: rand[N,Nc] (train_utils.py:75), randn[N,Nc]
    (volume_rendering_utils.py:44), rand[N,Nf] (nerf_helpers.py:363), randn[N,Nc+Nf]."""
    nc, nf = opts["num_coarse"], opts["num_fine"]
    out = dict(t_rand=None, n_c=None, u=None, n_f=None)
    kw = dict(dtype=torch.float32, device=device)
    if opts["perturb"]:
        out["t_rand"] = torch.rand((n, nc), **kw)
    if opts["noise_std"] > 0.0:
        out["n_c"] = torch.randn((n, nc), **kw)
    if has_fine:
        if opts["perturb"]:
            out["u"] = torch.rand((n, nf), **kw)
        if opts["noise_std"] > 0.0:
            out["n_f"] = torch.randn((n, nc + nf), **kw)
    return out


# Set by nerf/parallel.py: data_parallel while it calls run_one_iter_of_nerf on one shard (begin, count) of a call that has
# n_full rays in the single-process program.  The noise is then drawn for ALL n_full rays in the reference's chunk order and
# sliced, so (a) every rank consumes the RNG stream exactly like the single-process run (the streams stay in lock-step for the
# script's own np.random / torch draws) and (b) the shards see independent noise — the same noise the unsharded run would.
_shard_ctx = None


def _cat_noise(chunks):
    return {k: (torch.cat([c[k] for c in chunks], dim=0) if chunks[0][k] is not None else None) for k in chunks[0]}


def _chunk_noise(n, opts, device, has_fine, shard=None):
    """The noise of a call of n rays, drawn chunk by chunk in the reference's order; None when the reference draws none.
    shard = (begin, count, n_full) (see _shard_ctx): the draws are made for all n_full rays and rays [begin, begin + count)
    kept."""
    if not (opts["perturb"] or opts["noise_std"] > 0.0):
        return None
    begin, count, n_full = shard if shard is not None else (0, n, n)
    assert count == n
    chunk = opts["chunksize"]
    full = _cat_noise([_draw_noise(min(chunk, n_full - st), opts, device, has_fine) for st in range(0, n_full, chunk)])
    if shard is None:
        return full
    return {k: (v[begin:begin + count].contiguous() if v is not None else None) for k, v in full.items()}


def _render(rays, near, far, model_coarse, model_fine, opts, expressions, background_prior, latent_code, dir_z, noise,
            frame_index=None):
    """rays [N,8] = (o, d, near, far) on a CUDA device -> the 7-tuple of predict_and_render_radiance.  frame_index [N]: ray i is
    conditioned on expressions[frame_index[i]] ([F,76]) and latent_code[frame_index[i]] ([F,32])."""
    _check_models(model_coarse, model_fine)
    if opts["lindisp"]:
        raise NotImplementedError("lindisp sampling is not implemented (every shipped config sets it to False)")
    if expressions is None or latent_code is None:
        raise NotImplementedError("the paper model is conditioned on expressions and latent_code; both are required")
    has_fine = model_fine is not None and opts["num_fine"] > 0
    eng = _engine.renderer_for(rays.device)
    eng.sync_weights(model_coarse, model_fine if has_fine else None)
    needs_grad = torch.is_grad_enabled() and (
        any(p.requires_grad for p in model_coarse.parameters())
        or (has_fine and any(p.requires_grad for p in model_fine.parameters()))
        or any(t is not None and t.requires_grad for t in (latent_code, rays, expressions, background_prior, dir_z)))
    args = dict(near=float(near), far=float(far), num_coarse=opts["num_coarse"], num_fine=opts["num_fine"] if has_fine else 0,
                perturb=opts["perturb"], noise_std=opts["noise_std"], white_bkgd=opts["white_bkgd"],
                background=background_prior, dir_z=dir_z, noise=noise)
    if needs_grad:
        from ._autograd import render_with_grad
        return render_with_grad(eng, rays, model_coarse, model_fine if has_fine else None, expressions, latent_code, args,
                                frame_index)
    if frame_index is None:
        eng.set_frame(expressions, latent_code)
    else:
        eng.set_frames(expressions, latent_code)
    out = eng.render(rays[:, :3], rays[:, 3:6], frame_index=frame_index, **args)
    return (out["rgb_coarse"], out["disp_coarse"], out["acc_coarse"], out.get("rgb_fine"), out.get("disp_fine"),
            out.get("acc_fine"), out["w_last"])


def predict_and_render_radiance(ray_batch, model_coarse, model_fine, options, mode="train", encode_position_fn=None,
                                encode_direction_fn=None, expressions=None, background_prior=None, latent_code=None,
                                ray_dirs_fake=None):
    """One ray chunk [N,8] -> (rgb_c, disp_c, acc_c, rgb_f, disp_f, acc_f, weights_fine[:, -1])
    (train_utils.py:36-162).  The encode_*_fn arguments are accepted and ignored: encoding is fused."""
    opts = _mode_opts(options, mode)
    n = ray_batch.shape[0]
    has_fine = model_fine is not None and opts["num_fine"] > 0
    noise = _draw_noise(n, opts, ray_batch.device, has_fine)
    dir_z = None
    if ray_dirs_fake:  # ablation: the direction encoder sees chunk 0 of the fake bundle (train_utils.py:81-82)
        fake = ray_dirs_fake[0]
        if fake.shape[0] != n:
            raise RuntimeError(f"shape mismatch: ray chunk has {n} rays, ablation chunk 0 has {fake.shape[0]}")
        dir_z = fake[:, 5]
    return _render(ray_batch, options.dataset.near, options.dataset.far, model_coarse, model_fine, opts, expressions, background_prior, latent_code, dir_z,
                   noise if (opts["perturb"] or opts["noise_std"] > 0.0) else None)


def run_one_iter_of_nerf(height, width, focal_length, model_coarse, model_fine, ray_origins, ray_directions, options,
                         mode="train", encode_position_fn=None, encode_direction_fn=None, expressions=None,
                         background_prior=None, latent_code=None, ray_directions_ablation=None):
    """Drop-in for train_utils.py:165-290.  Returns the same tuple (7 outputs; 6 in validation mode without a
    fine network), shaped like the reference's.  All rays of the call go through ONE kernel launch; the
    reference's `chunksize` only controls the order of the noise draws (and the ablation quirk)."""
    _check_ndc(options)
    opts = _mode_opts(options, mode)
    has_fine = bool(model_fine) and opts["num_fine"] > 0
    shape3, shape1 = ray_directions.shape, ray_directions.shape[:-1]
    ro = ray_origins.reshape(-1, 3)
    rd = ray_directions.reshape(-1, 3)
    n = rd.shape[0]
    near = options.dataset.near * torch.ones_like(rd[..., :1])
    far = options.dataset.far * torch.ones_like(rd[..., :1])
    rays = torch.cat((ro, rd, near, far), dim=-1)
    chunk = opts["chunksize"]
    dir_z = None
    if torch.is_tensor(ray_directions_ablation):
        # every chunk sees chunk 0 of the ablation bundle (train_utils.py:81-82).  Under data_parallel the bundle is the WHOLE
        # call's and the chunks are the single-process program's; this shard keeps its slice.
        n_all = _shard_ctx[2] if _shard_ctx is not None else n
        fake0 = ray_directions_ablation.reshape(-1, 3)[:chunk]
        parts = []
        for st in range(0, n_all, chunk):
            m = min(chunk, n_all - st)
            if fake0.shape[0] != m:
                raise RuntimeError(f"shape mismatch: ray chunk has {m} rays, ablation chunk 0 has {fake0.shape[0]}")
            parts.append(fake0[:, 2])
        dir_z = torch.cat(parts, dim=0)
        if _shard_ctx is not None:
            dir_z = dir_z[_shard_ctx[0]:_shard_ctx[0] + _shard_ctx[1]].contiguous()
    noise = _chunk_noise(n, opts, rays.device, has_fine, _shard_ctx)
    bg = background_prior.reshape(-1, 3) if background_prior is not None else None
    outs = list(_render(rays, options.dataset.near, options.dataset.far, model_coarse, model_fine if has_fine else None, opts, expressions, bg, latent_code, dir_z, noise))
    if mode == "validation":
        shapes = [shape3, shape1, shape1]
        if model_fine:
            shapes = shapes + shapes + [shape1]
            return tuple(o.view(s) if o is not None else None for o, s in zip(outs, shapes))
        return tuple([o.view(s) for o, s in zip(outs, shapes)] + [None, None, None])
    return tuple(outs)


def render_frames(ray_origins, ray_directions, frame_index, expressions, latent_codes, model_coarse, model_fine, options, mode="train",
                  background_prior=None):
    """Render rays of several frames in ONE kernel launch, each ray conditioned on its own frame: ray i uses expressions[frame_index[i]]
    ([F,76]) and latent_codes[frame_index[i]] ([F,32]).  Options as run_one_iter_of_nerf handles them (near/far from
    options.dataset, the noise of the whole call drawn in the reference's chunk order).  Returns the 7-tuple of
    run_one_iter_of_nerf's training mode for the flattened rays.  Differentiable with respect to the parameters, every frame's
    expression and latent (pass `latent_table[ids]` to route the gradients back into a table), the rays and the background: a
    loss over several frames is one forward and one backward (the renderer keeps one saved training state).  frame_index outside
    [0, F) gives NaN outputs for those rays only.  Up to 1024 frames per call."""
    _check_ndc(options)
    opts = _mode_opts(options, mode)
    has_fine = bool(model_fine) and opts["num_fine"] > 0
    ro = ray_origins.reshape(-1, 3)
    rd = ray_directions.reshape(-1, 3)
    n = rd.shape[0]
    fi = frame_index.reshape(-1)
    if fi.shape[0] != n:
        raise ValueError(f"frame_index has {fi.shape[0]} entries for {n} rays")
    if expressions.dim() != 2 or latent_codes.dim() != 2 or expressions.shape[0] != latent_codes.shape[0]:
        raise ValueError("expressions [F,76] and latent_codes [F,32] must share F")
    near, far = options.dataset.near, options.dataset.far
    rays = torch.cat((ro, rd, near * torch.ones_like(rd[..., :1]), far * torch.ones_like(rd[..., :1])), dim=-1)
    noise = _chunk_noise(n, opts, rays.device, has_fine, _shard_ctx)
    bg = background_prior.reshape(-1, 3) if background_prior is not None else None
    return _render(rays, near, far, model_coarse, model_fine, opts, expressions, bg, latent_codes, None, noise, frame_index=fi)


render_frames.multi_frame = True  # nerf.parallel.data_parallel shards it by rays, with the signature above


class GaussianSmoothing(torch.nn.Module):
    """Depth-wise Gaussian blur (nerf/train_utils.py:379-442); only reachable in the reference when two
    hard-coded flags are edited.  Kept so `from nerf import GaussianSmoothing` works."""

    def __init__(self, channels, kernel_size, sigma, dim=2):
        super().__init__()
        if dim != 2:
            raise NotImplementedError("only 2-D smoothing is provided")
        k = int(kernel_size)
        ax = torch.arange(k, dtype=torch.float32) - (k - 1) / 2.0
        g = torch.exp(-(ax ** 2) / (2.0 * float(sigma) ** 2))
        kern = torch.outer(g, g)
        kern = kern / kern.sum()
        self.register_buffer("weight", kern.view(1, 1, k, k).repeat(channels, 1, 1, 1))
        self.groups = channels

    def forward(self, x):
        return torch.nn.functional.conv2d(x, self.weight, groups=self.groups)
