"""Data-parallel helpers for the render path (SURVEY.md §8e).  Rays are independent, so there is no collective
inside the path: evaluation shards contiguous pixel rows across ranks and all-gathers the output tiles; training
shards the ray batch and all-reduces one flat FP32 gradient bucket.  One process per GPU, torch.distributed
(NCCL on GPUs; the same code runs on gloo/CPU tensors in the tests)."""
import torch
import torch.distributed as dist

from . import train_utils


def shard_rows(height: int, world: int, rank: int):
    """Contiguous row block [begin, begin+rows) of rank `rank`; the first height % world ranks get one extra row."""
    base, extra = divmod(height, world)
    rows = base + (1 if rank < extra else 0)
    begin = rank * base + min(rank, extra)
    return begin, rows


def gather_rows(local: torch.Tensor, height: int, group=None) -> torch.Tensor:
    """All-gather per-rank row blocks [rows_r, W, C] (ragged when height % world != 0) into [height, W, C]."""
    world = dist.get_world_size(group)
    if world == 1:
        return local
    shapes = [shard_rows(height, world, r)[1] for r in range(world)]
    max_rows = max(shapes)
    pad = local
    if local.shape[0] < max_rows:
        pad = torch.cat((local, local.new_zeros((max_rows - local.shape[0],) + tuple(local.shape[1:]))), dim=0)
    out = local.new_empty((world * max_rows,) + tuple(local.shape[1:]))
    dist.all_gather_into_tensor(out, pad.contiguous(), group=group)
    parts = [out[r * max_rows:r * max_rows + shapes[r]] for r in range(world)]
    return torch.cat(parts, dim=0)


def render_frame_sharded(render_rows, height: int, group=None) -> torch.Tensor:
    """render_rows(row_begin, rows) -> [rows, W, C] on this rank; returns the assembled [height, W, C] on every rank."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    begin, rows = shard_rows(height, world, rank)
    local = render_rows(begin, rows)
    return gather_rows(local, height, group) if world > 1 else local


def shard_batch(n: int, world: int, rank: int):
    """Equal contiguous shards of a ray batch (n must divide evenly so that mean-of-means == global mean)."""
    if n % world:
        raise ValueError(f"ray batch of {n} does not split evenly over {world} ranks")
    per = n // world
    return rank * per, per


def allreduce_gradients(params, group=None, average=True):
    """One all-reduce over a single flat FP32 bucket holding every existing .grad (parameters whose grad is None,
    e.g. layers_dir.3, are skipped on every rank alike)."""
    grads = [p.grad for p in params if p.grad is not None]
    if not grads or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return 0
    flat = torch.cat([g.reshape(-1).float() for g in grads])
    dist.all_reduce(flat, group=group)
    if average:
        flat /= dist.get_world_size(group)
    off = 0
    for g in grads:
        n = g.numel()
        g.copy_(flat[off:off + n].view_as(g))
        off += n
    return flat.numel()


class _ScaleGrad(torch.autograd.Function):
    """Identity whose gradient is multiplied by `factor` (see data_parallel: local rows count `world` times under an
    AVERAGING gradient all-reduce, so that terms every rank computes identically — the latent regulariser — stay right)."""

    @staticmethod
    def forward(ctx, x, factor):
        ctx.factor = factor
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g * ctx.factor, None


def _gather_cat(local: torch.Tensor, group=None):
    """All-gather equal-sized shards along dim 0 (values only, no gradient)."""
    world = dist.get_world_size(group)
    out = local.new_empty((world * local.shape[0],) + tuple(local.shape[1:]))
    dist.all_gather_into_tensor(out, local.detach().contiguous(), group=group)
    return out


def _gather_train(outs, begin, count, world, group=None):
    """A training shard's outputs (rows [begin, begin + count) of the call) -> the whole call's: the other shards' rows
    all-gathered without gradient, the local rows through _ScaleGrad(world)."""
    full = []
    for o in outs:
        if o is None:
            full.append(None)
            continue
        g = _gather_cat(o, group)
        local = _ScaleGrad.apply(o, float(world)) if o.requires_grad else o
        full.append(torch.cat((g[:begin], local, g[begin + count:]), dim=0))
    return tuple(full)


def data_parallel(run_fn, group=None):
    """Wrap a function with the signature of run_one_iter_of_nerf (train_utils.py:165-181) so that an UNMODIFIED caller
    (train_transformed_rays.py:336-352, eval_transformed_rays.py:449-467) runs it data-parallel, one process per GPU:

    * mode == "validation": the [H, W, 3] ray bundle (and background / ablation directions) is split into contiguous row
      blocks (shard_rows), each rank renders its block, and every output is all-gathered back to [H, W, ...].
    * mode == "train": the [N, 3] ray batch is split evenly (shard_batch); every rank renders its shard and receives the
      other shards' outputs by all-gather, so the caller's loss over the FULL batch is unchanged.  Only the local rows carry
      gradient, scaled by the world size, so that an averaging all-reduce of the parameter gradients
      (allreduce_gradients(average=True), e.g. from an optimizer pre-step hook) yields exactly the single-process gradient —
      including loss terms that do not depend on the rays (the latent-code regulariser), which every rank computes alike.

    Noise: every rank draws the noise of the WHOLE call in the reference's order and keeps its shard's slice
    (train_utils._shard_ctx), so a seeded multi-rank run renders exactly what the seeded single-process run renders and the
    ranks' RNG streams stay in lock-step for the caller's own draws (ray selection).

    Multi-frame calls (a run_fn with the signature of nerf.render_frames, marked `multi_frame`): see _data_parallel_frames."""
    if getattr(run_fn, "multi_frame", False):
        return _data_parallel_frames(run_fn, group)
    def wrapped(height, width, focal_length, model_coarse, model_fine, ray_origins, ray_directions, options, mode="train",
                encode_position_fn=None, encode_direction_fn=None, expressions=None, background_prior=None, latent_code=None,
                ray_directions_ablation=None):
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        if world == 1:
            return run_fn(height, width, focal_length, model_coarse, model_fine, ray_origins, ray_directions, options, mode,
                          encode_position_fn, encode_direction_fn, expressions, background_prior, latent_code, ray_directions_ablation)
        if torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in (
                ray_origins, ray_directions, expressions, background_prior, ray_directions_ablation)):
            raise NotImplementedError("data_parallel differentiates the parameters and the latent code only: gradients with "
                                      "respect to rays, expressions, background or ablation directions would need all-reduces "
                                      "it does not do (run the fit in one process)")
        rank = dist.get_rank(group)
        if mode == "validation":
            H, W = ray_directions.shape[0], ray_directions.shape[1]
            begin, rows = shard_rows(H, world, rank)
            sl = slice(begin, begin + rows)
            bg = background_prior.reshape(H, W, 3)[sl].reshape(-1, 3) if background_prior is not None else None
            abl = ray_directions_ablation  # the whole bundle: train_utils slices it by the single-process chunk rule (_shard_ctx)
            train_utils._shard_ctx = (begin * W, rows * W, H * W)
            try:
                outs = run_fn(rows, width, focal_length, model_coarse, model_fine, ray_origins[sl], ray_directions[sl], options, mode,
                              encode_position_fn, encode_direction_fn, expressions, bg, latent_code, abl)
            finally:
                train_utils._shard_ctx = None
            return tuple(gather_rows(o.contiguous(), H, group) if o is not None else None for o in outs)
        n = ray_directions.shape[0]
        begin, per = shard_batch(n, world, rank)
        sl = slice(begin, begin + per)
        bg = background_prior[sl] if background_prior is not None else None
        abl = ray_directions_ablation
        train_utils._shard_ctx = (begin, per, n)
        try:
            outs = run_fn(height, width, focal_length, model_coarse, model_fine, ray_origins[sl], ray_directions[sl], options, mode,
                          encode_position_fn, encode_direction_fn, expressions, bg, latent_code, abl)
        finally:
            train_utils._shard_ctx = None
        return _gather_train(outs, begin, per, world, group)
    return wrapped


def _data_parallel_frames(run_fn, group=None):
    """data_parallel for nerf.render_frames: the flattened rays are split into contiguous shards, evenly in training mode
    (shard_batch) and by shard_rows' rule in validation mode, and frame_index and the background are sliced with them; every
    rank gets all F frames' expressions and latent codes.  The outputs are all-gathered as in data_parallel, and in training
    mode the local rows carry the gradient, scaled by the world size, so that per-frame latent gradients reach a latent table
    (`latent_table[ids]`) through the same averaging all-reduce as the parameters'.  The noise of the whole call is drawn on
    every rank and sliced (train_utils._shard_ctx)."""
    def wrapped(ray_origins, ray_directions, frame_index, expressions, latent_codes, model_coarse, model_fine, options, mode="train",
                background_prior=None):
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        if world == 1:
            return run_fn(ray_origins, ray_directions, frame_index, expressions, latent_codes, model_coarse, model_fine, options, mode,
                          background_prior)
        if torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in (
                ray_origins, ray_directions, expressions, background_prior)):
            raise NotImplementedError("data_parallel differentiates the parameters and the latent codes only: gradients with "
                                      "respect to rays, expressions or background would need all-reduces it does not do "
                                      "(run the fit in one process)")
        rank = dist.get_rank(group)
        ro, rd, fi = ray_origins.reshape(-1, 3), ray_directions.reshape(-1, 3), frame_index.reshape(-1)
        n = rd.shape[0]
        if fi.shape[0] != n:
            raise ValueError(f"frame_index has {fi.shape[0]} entries for {n} rays")
        begin, count = shard_rows(n, world, rank) if mode == "validation" else shard_batch(n, world, rank)
        sl = slice(begin, begin + count)
        bg = background_prior.reshape(-1, 3)[sl] if background_prior is not None else None
        train_utils._shard_ctx = (begin, count, n)
        try:
            outs = run_fn(ro[sl], rd[sl], fi[sl], expressions, latent_codes, model_coarse, model_fine, options, mode, bg)
        finally:
            train_utils._shard_ctx = None
        if mode == "validation":
            return tuple(gather_rows(o.contiguous(), n, group) if o is not None else None for o in outs)
        return _gather_train(outs, begin, count, world, group)
    return wrapped
