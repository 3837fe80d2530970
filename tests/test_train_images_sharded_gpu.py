"""Data-parallel steps over several images (FusedTrainer.step_images / capture_images with world > 1) on ONE GPU: one process
plays W ranks and does each rank's work in turn, as test_sharded_fp64_gpu.py does, so the SUM all-reduce becomes the sum of
the ranks' buckets in rank order.  Each rank runs the trainer's own K-image step body (_images_gradients(world, rank), what
step_images runs before its collective) from identical draws and seeds; the single process is the same body with world = 1.
  (a) bit for bit   every rank's sampled batch (rays, targets, background, frame indices, conditioning rows, state, shortfall)
                    is the single process's; its forward outputs are the matching rows of the single-process K * n-ray forward;
                    grad_rgb is 2 (rgb - t) * fp32(1 / fp32(3 N)) with N = K * n; a frame without rays in the rank's slice has
                    exactly zero d latent; each rank's loss share is within gamma(3 N_r + 32) of float64 (C1's bound).
  (b) float64       (slices of 256 rays or more, with a background) each rank's bucket against float64 torch_reference.render_at_depths per frame
                    on the slice's rays, at the slice's depths and grad_rgb, at test_sharded_fp64_gpu.py's C2 bounds; latent rows
                    fed by fewer than 256 rays at the single-ray bound PROBE_TOL.  The FP32 rank-order sum within
                    gamma(W) sum_r |bucket_r| of the float64 sum, which is within C3's gate (TOL) of the float64 batch gradient.
                    Without a background the fine fc_alpha.bias gradient (one scalar) of a 384-ray fast-mode slice was measured
                    0.87 of itself from float64 on an H100: the sigma gradients of rays that end on nothing cancel in that sum,
                    so the gate measures the slice's conditioning there, not the split; that case keeps the other checks.
  (c) regulariser   after the collective, the latent rows are the summed rows plus (latent_reg / K) l / ||l|| in ascending k, bit
                    for bit the documented FP32 order of nfb_latent_rows_grad (K >= 2); at K = 1 the rows are the summed rows
                    and Adam adds the term.  No rank's bucket carries it before the collective.
  (d) Adam          step_images(world = W, rank = W - 1) with dist.all_reduce replaced by the rank-order sum: the bucket it hands
                    the collective is rank W - 1's bit for bit, its parameters equal the internal path's (sum, regulariser,
                    update()) bit for bit and float64 Adam on the summed bucket with the term added once within 1e-6.
  (e) graph         capture_images(world = W, rank = r) replays equal eager step_images(world = W, rank = r) bit for bit over
                    10 steps, with dist.all_reduce replaced by a capturable stand-in (the bucket doubled: two ranks holding the
                    same bucket), so the collective, the regulariser after it and Adam sit in the same order in both.
  (f) chunked       over NFB_TRAIN_MEM_MB the ranks' backwards run in chunks over sliced views: outputs and grad_rgb bit for
                    bit, the summed bucket within the chunked path's 3e-3 of the in-budget single process's.
  (g) errors        an uneven split, a rank outside the world, K or n out of range raise ValueError before any library launch
                    and before the collective.
Real collectives (NCCL) are test_multigpu_images.py's."""
import math
import types

import pytest
import torch

import nerface_oracle as O
from test_backward_fp64_gpu import PROBE_TOL, TOL, check, reference
from test_backward_gpu import dev_tensor
from test_train_images_gpu import latent_rows_fp32, make_model

pytestmark = pytest.mark.gpu

NC, NF, ROUNDS, REG, SEED = 64, 64, 32, 0.005, 91
NAMES = ("rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last")
BATCH_NAMES = ("ray_origins", "ray_directions", "target", "background", "frame_index", "expressions", "latents", "state", "shortfall")
U = 2.0 ** -24
N_IMAGES = 6


def gamma(k):
    return k * U / (1.0 - k * U)


def tol_of(prec, rays):
    """C2's bounds (test_sharded_fp64_gpu.shard_tol: TOL, twice its max for 256-ray shards), the single-ray bound below 256 rays."""
    base = "exact" if prec == "exact_grad" else prec
    if rays < 256:
        return PROBE_TOL[base]
    return TOL[base] if rays >= 512 else (2.0 * TOL[base][0], TOL[base][1])


@pytest.fixture(scope="module")
def env(built_lib):
    import nerf
    from nerf import _engine, fused_train, ray_sampler
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    e = types.SimpleNamespace(nerf=nerf, fused_train=fused_train, ray_sampler=ray_sampler, dev=dev, eng=_engine.renderer_for(dev))
    e.lat0 = torch.randn(N_IMAGES, 32, generator=torch.Generator().manual_seed(3)) * 0.1
    e.data = {bg: dataset(e, bg) for bg in (True, False)}
    return e


def dataset(e, bg):
    H = W = 64
    frs = [O.synthetic_frame(40 + i, H, W) for i in range(N_IMAGES)]
    g = torch.Generator().manual_seed(140)
    images = torch.rand(N_IMAGES, H, W, 3, generator=g).to(e.dev)
    poses = torch.stack([f["pose"][:3, :4].reshape(-1) for f in frs])
    exprs = torch.stack([f["expr"] for f in frs])
    bboxs = [(4 + 2 * i, 60, 2 + i, 62 - i) for i in range(N_IMAGES)]
    return e.ray_sampler.TrainImages(images, poses, exprs, bboxs, frs[0]["intrinsics"], background=frs[0]["bg"] if bg else None,
                                     device=e.dev)


def trainer(e, prec, perturb=True):
    return e.fused_train.FusedTrainer(make_model(e.nerf, O.random_init_params(100), e.dev), make_model(e.nerf, O.random_init_params(101), e.dev),
                                      n_latent=N_IMAGES, num_coarse=NC, num_fine=NF, perturb=perturb, noise_std=0.1 if perturb else 0.0,
                                      latent_reg=REG, latent_codes=e.lat0, precision=prec)


def run_rank(e, data, ids, n, draws, prec, world, rank, depths=True):
    """One rank's step body up to its collective; copies of everything the next rank's run overwrites (the sample depths only
    with `depths`: a chunked step keeps one chunk's)."""
    tr = trainer(e, prec)
    tr._own_engine()
    k = len(ids)
    sb = tr._images_buffers(data, k, n)
    sb["img"].copy_(torch.tensor(ids, dtype=torch.int32))
    tr._images_sample(data, sb, n, draws, ROUNDS)
    torch.manual_seed(SEED)
    l0 = e.eng.launch_count()
    out = tr._images_gradients(sb, k, n, world, rank)
    torch.cuda.synchronize()
    per = k * n // world
    d = tr.eng.train_debug() if depths else None
    return types.SimpleNamespace(
        tr=tr, lo=rank * per, hi=(rank + 1) * per, per=per, launches=e.eng.launch_count() - l0,
        sb={name: t.clone() for name, t in sb.items() if t is not None}, out={name: out[name].clone() for name in NAMES},
        bucket=tr.grads.clone(), loss=tr.loss[:2].clone(),
        z_c=dev_tensor(d.z_coarse, (per, NC)).clone() if depths else None,
        z_f=dev_tensor(d.z_fine, (per, NC + NF)).clone() if depths else None)


def split_bucket(tr, flat):
    """(coarse grads, fine grads) in PARAM_ORDER (None for layers_dir.3) and the latent table's [rows, 32] view of a bucket."""
    views, off = [], 0
    for v in tr._views:
        views.append(flat[off:off + v.numel()].view(v.shape))
        off += v.numel()
    skip = [g is None for g in tr._gc]
    gc = [None if s else t for s, t in zip(skip, views[:26])]
    gf = [None if s else t for s, t in zip(skip, views[26:])]
    return gc, gf, flat[tr.lat_off:].view(-1, 32)


def reference_rank(e, r, ids, noise):
    """float64 gradients of rank r's slice: per frame on the slice's rays of that frame, parameters summed over frames, each
    frame's latent gradient on its image's row; and the rays feeding each row."""
    sb, sl = r.sb, slice(r.lo, r.hi)
    fi = sb["frame_index"][sl]
    gc = gf = None
    table = torch.zeros(N_IMAGES, 32, dtype=torch.float64, device=e.dev)
    rays = [0] * N_IMAGES
    for f in range(len(ids)):
        idx = torch.nonzero(fi == f).flatten()
        if len(idx) == 0:
            continue
        rows = idx + r.lo
        pick = lambda t: None if t is None else t[rows].contiguous()  # noqa: E731
        c = types.SimpleNamespace(n=len(idx), nc=NC, nf=NF, noise_std=0.1, white=False, dz=None, mc=r.tr.mc, mf=r.tr.mf,
                                  noise={key: pick(v) for key, v in noise.items() if v is not None}, bg=pick(sb.get("background")),
                                  expr=sb["expressions"][f], latent=sb["latents"][f], ro=pick(sb["ray_origins"]),
                                  rd=pick(sb["ray_directions"]))
        gouts = [sb["g0"][rows], None, None, sb["g1"][rows], None, None, None]
        R = reference(e, c, r.z_c[idx], r.z_f[idx], gouts)
        add = lambda a, b: b if a is None else [None if x is None else x + y for x, y in zip(a, b)]  # noqa: E731
        gc, gf = add(gc, R.gc), add(gf, R.gf)
        table[ids[f]] += R.glat.reshape(32)
        rays[ids[f]] += len(idx)
    return types.SimpleNamespace(gc=gc, gf=gf, table=table, rays=rays)


def pairs(tr, flat, R):
    gc, gf, table = split_bucket(tr, flat)
    from nerf._engine import PARAM_ORDER
    params = [(f"{net}/{k}", g, rr) for net, gs, rs in (("coarse", gc, R.gc), ("fine", gf, R.gf))
              for k, g, rr in zip(PARAM_ORDER, gs, rs) if g is not None]
    used = [i for i in range(N_IMAGES) if R.rays[i]]
    rows = {i: (f"latent row {i}", table[i], R.table[i]) for i in used}
    return params, rows


def adam64(p0, g64):
    b1, b2, eps, lr = 0.9, 0.999, 1e-8, 5e-4
    m, v = (1 - b1) * g64, (1 - b2) * g64 * g64
    return p0 - lr / (1 - b1) * m / (v.sqrt() / math.sqrt(1 - b2) + eps)


def reg64(e, ids):
    """The regulariser's float64 gradient, added once: (latent_reg / K) l / ||l|| per step image (latent_reg l / ||l|| at K = 1)."""
    out = torch.zeros(N_IMAGES, 32, dtype=torch.float64, device=e.dev)
    w = REG / len(ids)
    for i in ids:
        lat = e.lat0[i].double().to(e.dev)
        if float(lat.norm()) > 0:
            out[i] += w * lat / lat.norm()
    return out


# (W, K, n, precision, background): slices inside one frame, straddling frames, one frame per rank, 64 frames, single rays
CASES = {
    "W2_K1_2048_fast": (2, 1, 2048, "fast", True),
    "W4_K2_512_exact": (4, 2, 512, "exact", True),
    "W4_K3_512_fast_nobg": (4, 3, 512, "fast", False),
    "W8_K8_256_exact_grad": (8, 8, 256, "exact_grad", True),
    "W8_K64_32_exact": (8, 64, 32, "exact", True),
    "W3_K3_100_fast": (3, 3, 100, "fast", True),
    "W2_K2_1_exact": (2, 2, 1, "exact", False),
    "W3_K1_3_fast": (3, 1, 3, "fast", True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_sharded_step_against_single_process_and_float64(env, case, monkeypatch):
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    W, k, n, prec, bg = CASES[case]
    e, data = env, env.data[bg]
    g = torch.Generator().manual_seed(17 + k)
    ids = [int(i) for i in torch.randint(0, N_IMAGES, (k,), generator=g)]
    if k >= 2:
        ids[1] = ids[0]  # a repeated image: two frames on one latent row
    N = k * n
    draws = torch.rand(k * ROUNDS * n, dtype=torch.float64, generator=g).to(e.dev)
    single = run_rank(e, data, ids, n, draws, prec, 1, 0)
    assert (single.sb["state"][:, 0] == n).all()
    ranks = [run_rank(e, data, ids, n, draws, prec, W, r) for r in range(W)]
    f32 = lambda v: torch.tensor(v, dtype=torch.float32)  # noqa: E731
    inv = (f32(1.0) / (f32(3.0) * f32(float(N)))).to(e.dev)
    worst = {}

    # ---- (a) bit for bit
    for r in ranks:
        tag = (case, r.lo)
        for name in BATCH_NAMES:
            if name in single.sb:
                assert torch.equal(r.sb[name], single.sb[name]), (tag, name)
        sl = slice(r.lo, r.hi)
        for name in NAMES:
            assert torch.equal(r.out[name], single.out[name][sl]), (tag, name)
        tgt = r.sb["target"][sl]
        for p, name in ((0, "rgb_coarse"), (1, "rgb_fine")):
            gr = r.sb["g0" if p == 0 else "g1"][sl]
            assert torch.equal(gr, (2.0 * (r.out[name] - tgt)) * inv), (tag, name)
            share64 = float(((r.out[name].double() - tgt.double()) ** 2).sum()) / (3.0 * N)
            assert abs(float(r.loss[p]) - share64) <= gamma(3 * r.per + 32) * share64, (tag, p)
        if k >= 2:
            present = set(r.sb["frame_index"][sl].tolist())
            for f in range(k):
                if f not in present:
                    assert torch.count_nonzero(r.sb["glat"][f]) == 0, (tag, f)
    assert torch.equal(ranks[0].tr.shortfall, single.tr.shortfall)

    # ---- (b) float64
    torch.manual_seed(SEED)
    noise = single.tr._draw_noise(N)
    f64 = ranks[0].per >= 256 and bg
    refs = []
    if f64:
        for r in ranks:
            R = reference_rank(e, r, ids, noise)
            refs.append(R)
            params, rows = pairs(r.tr, r.bucket, R)
            worst[f"rank {r.lo // r.per} params"] = check(f"{case} rank {r.lo // r.per} params", params, tol_of(prec, r.per), quiet=True)
            for i, row in rows.items():
                check(f"{case} rank {r.lo // r.per} row {i}", [row], tol_of(prec, R.rays[i]), quiet=True)
    sum32 = ranks[0].bucket.clone()
    for r in ranks[1:]:
        sum32 = sum32 + r.bucket
    sum64 = sum((r.bucket.double() for r in ranks[1:]), ranks[0].bucket.double().clone())
    absum = sum((r.bucket.double().abs() for r in ranks[1:]), ranks[0].bucket.double().abs())
    assert bool(((sum32.double() - sum64).abs() <= gamma(W) * absum).all()), case
    if f64:
        add = lambda xs: None if xs[0] is None else sum(xs[1:], xs[0].clone())  # noqa: E731
        R_all = types.SimpleNamespace(gc=[add([R.gc[i] for R in refs]) for i in range(26)],
                                      gf=[add([R.gf[i] for R in refs]) for i in range(26)],
                                      table=sum((R.table for R in refs[1:]), refs[0].table.clone()),
                                      rays=[sum(R.rays[i] for R in refs) for i in range(N_IMAGES)])
        params, rows = pairs(single.tr, sum64, R_all)
        worst["sum params"] = check(f"{case} rank-order sum", params, tol_of(prec, N))
        for i, row in rows.items():
            check(f"{case} sum row {i}", [row], tol_of(prec, R_all.rays[i]), quiet=True)

    # ---- (c) the regulariser, once, after the collective
    t = trainer(e, prec)
    sbt = t._images_buffers(data, k, n)
    sbt["img"].copy_(torch.tensor(ids, dtype=torch.int32))
    t.grads.copy_(sum32)
    t._images_regulariser(sbt, k)
    torch.cuda.synchronize()
    rows32 = sum32[t.lat_off:].view(-1, 32).cpu()
    want = latent_rows_fp32(torch.zeros(k, 32), ids, e.lat0, rows32, REG / k) if k >= 2 else rows32
    assert torch.equal(t.grads[t.lat_off:].view(-1, 32).cpu(), want), case
    assert torch.equal(t.grads[:t.lat_off], sum32[:t.lat_off])

    # ---- (d) Adam through the public eager step, the collective standing in as the rank-order sum
    seen = []

    def all_reduce(tensor, group=None):
        seen.append(tensor.clone())
        tensor.copy_(sum32)
    monkeypatch.setattr(torch.distributed, "all_reduce", all_reduce)
    pub = trainer(e, prec)
    torch.manual_seed(SEED)
    loss = pub.step_images(data, ids, n, draws=draws, max_rounds=ROUNDS, world=W, rank=W - 1).clone()
    torch.cuda.synchronize()
    assert len(seen) == 1 and torch.equal(seen[0], ranks[-1].bucket) and torch.equal(loss, ranks[-1].loss), case
    t._reg_row = ids[0] if k == 1 else -1
    t.update()
    torch.cuda.synchronize()
    assert torch.equal(t.params, pub.params) and torch.equal(t.exp_avg_sq, pub.exp_avg_sq), case
    p0 = trainer(e, prec).params.double()
    g64 = sum32.double()
    g64[t.lat_off:] += reg64(e, ids).reshape(-1)
    worst["adam"] = float((pub.params.double() - adam64(p0, g64)).abs().max())
    assert worst["adam"] <= 1e-6, (case, worst["adam"])
    print(f"{case}: " + ", ".join(f"{key} {v}" for key, v in worst.items()))


@pytest.mark.parametrize("W,k,n", [(4, 4, 64), (2, 1, 128), (3, 2, 48)])
def test_captured_sharded_step_equals_the_eager_one(env, W, k, n, monkeypatch):
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    monkeypatch.setattr(torch.distributed, "all_reduce", lambda tensor, group=None: tensor.add_(tensor))
    e, data = env, env.data[True]
    g = torch.Generator(device=e.dev).manual_seed(13 + k)
    for rank in sorted({0, W - 1}):
        te, tg = trainer(e, "fast", perturb=False), trainer(e, "fast", perturb=False)
        tg.capture_images(data, k, n, max_rounds=ROUNDS, device_draws=False, world=W, rank=rank)
        for i in range(10):
            draws = torch.rand(k * ROUNDS * n, dtype=torch.float64, device=e.dev, generator=g)
            ids = [(3 * i + j) % N_IMAGES for j in range(k)]
            la = te.step_images(data, ids, n, draws=draws, max_rounds=ROUNDS, world=W, rank=rank).clone()
            lb = tg.step_images_graph(torch.tensor(ids, dtype=torch.int32, device=e.dev), draws=draws).clone()
            torch.cuda.synchronize()
            assert torch.equal(la, lb), (W, k, rank, i)
            for name in ("params", "exp_avg", "exp_avg_sq"):
                assert torch.equal(getattr(te, name), getattr(tg, name)), (W, k, rank, i, name)
        assert te.iter == tg.iter == 10


def test_chunked_sharded_backward(env, monkeypatch):
    """K = 4 x 128 rays over 2 ranks at NFB_TRAIN_MEM_MB=48: each rank's 256 rays render and differentiate in chunks."""
    e, data = env, env.data[True]
    ids, n, W = [0, 2, 1, 2], 128, 2
    draws = torch.rand(4 * ROUNDS * n, dtype=torch.float64, generator=torch.Generator().manual_seed(5)).to(e.dev)
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    single = run_rank(e, data, ids, n, draws, "fast", 1, 0)
    in_budget = run_rank(e, data, ids, n, draws, "fast", W, 0)
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")
    ranks = [run_rank(e, data, ids, n, draws, "fast", W, r, depths=False) for r in range(W)]
    assert ranks[0].launches > in_budget.launches + 10  # the chunked path ran
    inv = (torch.tensor(1.0) / (torch.tensor(3.0) * torch.tensor(float(4 * n)))).to(e.dev)
    for r in ranks:
        sl = slice(r.lo, r.hi)
        for name in NAMES:
            assert torch.equal(r.out[name], single.out[name][sl]), (r.lo, name)
        assert torch.equal(r.sb["g0"][sl], (2.0 * (r.out["rgb_coarse"] - r.sb["target"][sl])) * inv)
    total = ranks[0].bucket + ranks[1].bucket
    gs, _, _ = split_bucket(single.tr, single.bucket)
    gt, _, _ = split_bucket(single.tr, total)
    for a, b in zip(gs, gt):
        if a is not None:
            assert float((a - b).abs().max()) <= 3e-3 * max(float(a.abs().max()), 1e-12)
    rows = single.bucket[single.tr.lat_off:].view(-1, 32)
    rows_t = total[single.tr.lat_off:].view(-1, 32)
    reg = reg64(e, ids).float()  # the single process's rows carry the regulariser; the ranks' add it after the collective
    assert float((rows - reg - rows_t).abs().max()) <= 3e-3 * float(rows.abs().max())


def test_errors_before_any_launch_or_collective(env, monkeypatch):
    e, data = env, env.data[True]
    calls = []
    monkeypatch.setattr(torch.distributed, "all_reduce", lambda *a, **kw: calls.append(1))
    tr = trainer(e, "fast")
    torch.cuda.synchronize()
    l0 = e.eng.launch_count()
    bad = [dict(image_index=[0, 1, 2], n=7, world=2, rank=0),      # 21 rays over 2 ranks
           dict(image_index=[0, 1], n=16, world=2, rank=2),        # rank outside the world
           dict(image_index=[0, 1], n=16, world=2, rank=-1),
           dict(image_index=[0] * 65, n=16, world=5, rank=0),      # K > 64
           dict(image_index=[0, 1], n=4096, world=2, rank=0),      # n > 2048
           dict(image_index=[0, 9], n=16, world=2, rank=0)]        # image outside the set
    for a in bad:
        with pytest.raises(ValueError):
            tr.step_images(data, a["image_index"], a["n"], world=a["world"], rank=a["rank"])
        if a["image_index"] != [0, 9]:
            with pytest.raises(ValueError):
                tr.capture_images(data, len(a["image_index"]), a["n"], world=a["world"], rank=a["rank"])
    with pytest.raises(ValueError):
        tr.step_images(data, [0, 1], 16, draws=torch.zeros(10, dtype=torch.float64, device=e.dev), world=2, rank=0)
    torch.cuda.synchronize()
    assert e.eng.launch_count() == l0 and not calls and tr.iter == 0 and float(tr.grads.abs().max()) == 0.0
