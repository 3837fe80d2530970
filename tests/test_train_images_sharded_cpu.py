"""Data-parallel steps over several images and multi-frame calls, host logic without a GPU:
  * FusedTrainer's K-image argument checks for world > 1 (an uneven split, a rank outside the world, no process group and no
    explicit rank), all before any launch;
  * nerf.parallel.data_parallel(render_frames) on CPU (gloo, world_size 2) around a small differentiable stand-in with
    render_frames' signature: the slices of rays, frame_index and background each rank is handed, the noise context
    (train_utils._shard_ctx), the gathered outputs, the world-size gradient factor of the local rows (after an averaging
    all-reduce the parameter and per-frame latent gradients are the single-process ones), and the refusal of input gradients."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Data:
    H = W = 8
    n_images = 2


def test_sharded_step_argument_checks(built_lib):
    from nerf import fused_train
    tr = fused_train.FusedTrainer.__new__(fused_train.FusedTrainer)
    tr.latent_codes = torch.zeros(2, 32)
    with pytest.raises(ValueError, match="1 <= K <= 64"):
        tr._check_images(_Data(), 65, 16, 1)
    with pytest.raises(ValueError, match="1 <= K <= 64"):
        tr._check_images(_Data(), 65, 16, 2, rank=1)
    with pytest.raises(ValueError, match="does not split evenly"):
        tr._check_images(_Data(), 3, 7, 2, rank=0)          # 21 rays over 2 ranks
    with pytest.raises(ValueError, match="at least one rank"):
        tr._check_images(_Data(), 2, 16, 0)
    with pytest.raises(ValueError, match="outside"):
        tr._check_images(_Data(), 2, 16, 4, rank=4)
    with pytest.raises(ValueError, match="outside"):
        tr._check_images(_Data(), 2, 16, 4, rank=-1)
    # world > 1 with neither a process group nor an explicit rank: there is no collective to run the step over
    assert not torch.distributed.is_initialized()
    with pytest.raises(NotImplementedError, match="process group"):
        tr._check_images(_Data(), 2, 16, 2)
    assert tr._check_images(_Data(), 3, 8, 3, rank=2) == 2   # 24 rays over 3 ranks; slices straddle frames
    assert tr._check_images(_Data(), 1, 16, 1) == 0          # world 1 needs no process group


# A stand-in for nerf.render_frames: ray i is conditioned on latent_codes[frame_index[i]]; records what it was handed.
_CALLS = []


def _fake_frames(ray_origins, ray_directions, frame_index, expressions, latent_codes, model_coarse, model_fine, options,
                 mode="train", background_prior=None):
    from nerf import train_utils
    _CALLS.append(dict(ro=ray_origins.clone(), rd=ray_directions.clone(), fi=frame_index.clone(), expr=expressions,
                       lat=latent_codes, bg=None if background_prior is None else background_prior.clone(),
                       ctx=train_utils._shard_ctx, mode=mode))
    ro, rd = ray_origins.reshape(-1, 3), ray_directions.reshape(-1, 3)
    x = torch.cat((ro, rd, latent_codes[frame_index.long()]), dim=-1)
    hc, hf = torch.tanh(model_coarse(x)), torch.tanh(model_fine(x))
    if background_prior is not None:
        hc = hc + 0.1 * torch.cat((background_prior, background_prior[:, :2]), dim=-1)
    return hc[:, :3], hc[:, 3], hc[:, 4], hf[:, :3], hf[:, 3], hf[:, 4], hf[:, 4] * 0.5


_fake_frames.multi_frame = True


def _models():
    torch.manual_seed(0)
    return torch.nn.Linear(6 + 4, 5), torch.nn.Linear(6 + 4, 5)


def _worker(rank, world, port, q):
    sys.path.insert(0, os.path.join(ROOT, "4d-facial-avatars_b200"))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from nerf import parallel, train_utils
    run = parallel.data_parallel(_fake_frames)
    g = torch.Generator().manual_seed(1)
    mc, mf = _models()
    F = 3
    table = torch.randn(5, 4, generator=g).requires_grad_(True)
    ids = torch.tensor([4, 0, 2])
    expr = torch.randn(F, 76, generator=g)
    res = {}
    # ---- validation: 7 rays over 2 ranks (4 + 3, shard_rows' rule), gathered
    n = 7
    ro, rd, bg = torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g), torch.rand(n, 3, generator=g)
    fi = torch.randint(0, F, (n,), generator=g, dtype=torch.int32)
    with torch.no_grad():
        _CALLS.clear()
        got = run(ro, rd, fi, expr, table[ids], mc, mf, None, mode="validation", background_prior=bg)
        c = _CALLS[-1]
        ref = _fake_frames(ro, rd, fi, expr, table[ids], mc, mf, None, mode="validation", background_prior=bg)
    begin, rows = parallel.shard_rows(n, world, rank)
    sl = slice(begin, begin + rows)
    res["val_slices"] = (torch.equal(c["ro"], ro[sl]) and torch.equal(c["rd"], rd[sl]) and torch.equal(c["fi"], fi[sl])
                         and torch.equal(c["bg"], bg[sl]) and c["expr"].shape == (F, 76) and c["lat"].shape == (F, 4)
                         and c["ctx"] == (begin, rows, n) and c["mode"] == "validation")
    res["val_gather"] = all(a.shape == b.shape and torch.allclose(a, b) for a, b in zip(got, ref))
    # ---- train: 16 rays (8 per rank), the loss over the whole batch as a single-process caller writes it
    n = 16
    ro, rd, bg = torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g), torch.rand(n, 3, generator=g)
    fi = torch.randint(0, F, (n,), generator=g, dtype=torch.int32)
    tgt = torch.rand(n, 3, generator=g)
    params = list(mc.parameters()) + list(mf.parameters()) + [table]

    def loss_of(outs):
        return ((outs[0] - tgt) ** 2).mean() + ((outs[3] - tgt) ** 2).mean() + 0.005 * sum(table[i].norm() for i in ids)
    loss_ref = loss_of(_fake_frames(ro, rd, fi, expr, table[ids], mc, mf, None, background_prior=bg))
    g_ref = torch.autograd.grad(loss_ref, params)
    _CALLS.clear()
    outs = run(ro, rd, fi, expr, table[ids], mc, mf, None, mode="train", background_prior=bg)
    c = _CALLS[-1]
    begin, per = parallel.shard_batch(n, world, rank)
    sl = slice(begin, begin + per)
    res["train_slices"] = (torch.equal(c["ro"], ro[sl]) and torch.equal(c["fi"], fi[sl]) and torch.equal(c["bg"], bg[sl])
                           and c["ctx"] == (begin, per, n) and train_utils._shard_ctx is None)
    # the local rows carry world x their gradient, the gathered rows none
    gl = torch.autograd.grad(outs[0].sum(), mc.bias, retain_graph=True)[0]
    lone = torch.autograd.grad(_fake_frames(ro[sl], rd[sl], fi[sl], expr, table[ids], mc, mf, None, background_prior=bg[sl])[0].sum(),
                               mc.bias)[0]
    res["scale"] = torch.allclose(gl, world * lone)
    loss = loss_of(outs)
    loss.backward()
    parallel.allreduce_gradients(params, average=True)
    res["train_loss"] = abs(float(loss) - float(loss_ref)) < 1e-6 and all(o.shape[0] == n for o in outs)
    res["train_grads"] = all(torch.allclose(p.grad, r, atol=1e-6, rtol=1e-5) for p, r in zip(params, g_ref))
    q.put((rank, res))
    dist.destroy_process_group()


def test_data_parallel_render_frames_gloo():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33600 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=180) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, checks in res:
        assert all(checks.values()), (rank, checks)


@pytest.mark.parametrize("which", ["ray_origins", "ray_directions", "expressions", "background_prior"])
def test_data_parallel_render_frames_refuses_input_gradients(monkeypatch, which):
    from nerf import parallel
    monkeypatch.setattr(parallel.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(parallel.dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(parallel.dist, "get_rank", lambda group=None: 0)
    called = []

    def stub(*a, **k):
        called.append(1)
    stub.multi_frame = True
    n = 8
    kw = dict(ray_origins=torch.zeros(n, 3), ray_directions=torch.ones(n, 3), expressions=torch.zeros(2, 76),
              background_prior=torch.zeros(n, 3))
    kw[which].requires_grad_(True)
    with pytest.raises(NotImplementedError, match="data_parallel"):
        parallel.data_parallel(stub)(kw["ray_origins"], kw["ray_directions"], torch.zeros(n, dtype=torch.int32), kw["expressions"],
                                     torch.zeros(2, 32, requires_grad=True), None, None, None, mode="train",
                                     background_prior=kw["background_prior"])
    assert not called
