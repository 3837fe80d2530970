"""The multi-GPU split (DESIGN §0 row e, §7) on ONE GPU: one process plays N ranks on one device and does each rank's work in
turn, and the collectives become what they compute — a concatenation of row shards in rank order (evaluation), a sum of flat
gradient buckets (training).  Each stage is fed the kernel's own output of the stage before it and is compared with a plain
reference: the unsharded call bit for bit where the split must not change a bit, float64 where FP32 sums are reordered.
  (A) row shards      render_camera(row_begin, rows) per shard of parallel.shard_rows, concatenated: all 7 outputs bitwise the
                      full-frame call (also through render_frame_host, and against render() on the shard's explicit O.ray_bundle
                      rays).  Odd W puts shard boundaries inside a 2-ray unit; a one-row shard of the 97-wide frame launches
                      fewer units than SMs (the launch's own small-grid path).
  (B) drop-in eval    data_parallel's validation body re-enacted per rank (_shard_ctx, seeded like every real rank), chunksize
                      straddling the shards: bitwise the unsharded seeded call, also with ray_directions_ablation.
  (C) training batch  FusedTrainer.gradients(world=1, n_total=n) per shard with the noise drawn once and sliced:
      C1 loss gradient  grad_rgb bitwise 2 * (rgb - t) * fp32(1 / fp32(3 n_total)); each shard's loss share within
                        gamma(3 n_shard + 32) of float64 (3 n_shard FMAs in at most that many sequential steps, 5 butterfly
                        levels, 32 warp partials, the rounded 1 / (3 n_total) and the product: all terms are positive, so the
                        bound is relative to the share); the sum of shares within the sum of those bounds of the float64 batch loss.
      C2 shard backward all 48 parameter gradients and the latent gradient against float64 torch_reference.render_at_depths at the
                        shard's depths, fed its own grad_rgb, per tensor at TOL (max, L2) of test_backward_fp64_gpu.py (twice its
                        max bound for 256-ray shards, see below).
      C3 all-reduce     the float64 sum of the buckets against the float64 gradient of the whole batch at TOL; the FP32 rank-order
                        sum within gamma(N) sum_r |bucket_r| of the float64 sum, element by element.
      C4 control        one unsharded 2048-ray gradients() call: its depths and grad_rgb are the shards' concatenated bit for bit
                        (so C3's reference is also its reference), and it meets the same gate.
      C5 regulariser    no shard's latent row carries reg_weight l / |l|: its error against the float64 backward alone must stay
                        below half the term's largest entry; update() of two fresh trainers given the summed bucket: bitwise the same
                        parameters, within 1e-6 of float64 Adam with the term added once (test_adam_kernel_matches_torch_adam).
      C6 drop-in train  run_one_iter_of_nerf(mode="train") under _shard_ctx: shard outputs bitwise the unsharded seeded call's
                        rows; the wrapper's loss (others detached, local rows through parallel._ScaleGrad(world), averaged after
                        summing) gives parameter and latent gradients within C3's gate, regulariser included.
  A shard whose target is its own render gets exactly zero output gradients, an exactly zero bucket and loss scale 1.

Real collectives (NCCL refuses two ranks on one device) are test_multigpu.py's; NCCL's summation order for N > 2 is not rank
order, so no bits are asserted against a real collective here.

Measured on an H100 80GB HBM3 at a 700 W power limit (CUDA 12.9), worst over all cases; the file takes about 25 s:
  (A), (B), C1 grad_rgb, C4 depths / grad_rgb, C6 outputs, Adam across two trainers: bitwise in every case.
  C1 loss share      0.0039 of its bound (N = 8, fast); the sum of shares within its bound in every case.
  C2 shard backward  shards of 1000 rays or more: exact max 1.4e-3, L2 8.0e-4 (N = 2); fast max 2.5e-2, L2 8.7e-3 (the 1000-ray
                     shard) -> TOL.  512-ray shards: exact 2.2e-3 / 6.0e-4, fast 1.1e-2 / 6.6e-3.  256-ray shards (N = 8): exact
                     max 4.7e-3, L2 1.4e-3; fast max 4.0e-2 (coarse layers_dir.2.bias of shard 1), L2 1.3e-2 -> twice TOL's max bound
                     for them (shard_tol).  A bias gradient summed over fewer rays cancels more: exact mode's worst 256-ray shard,
                     on the same tensor, is five times its whole-batch error too, so this is the shard's conditioning.
  C3 summed buckets  exact max 9.6e-4, L2 6.1e-4; fast max 3.2e-3, L2 1.6e-3, for every N and the unequal split.
  C4 control         exact max 9.6e-4, L2 6.0e-4; fast max 3.1e-3, L2 1.6e-3: the sharded sum is as accurate as one call.
  C5 regulariser     a shard's latent-row error is at most 7.9e-6 of the regulariser's largest entry; Adam within 4.7e-9 of
                     float64 (gate 1e-6).
  C6 drop-in train   as C3: exact max 9.6e-4, L2 6.1e-4; fast max 3.2e-3, L2 1.6e-3.
Planted defects, each built once and not kept:
  launch_loss_grad dividing by n_rays instead of n_total: C1's bitwise grad_rgb check, in all 8 training-batch cases (the
      unsharded control, where the two agree, is unaffected).
  in-kernel ray generation taking a ray's pixel row from its unit's first ray instead of its own index: (A) bitwise at 97x97
      with 2-ray units (64c128f), both precisions, from N = 2; even widths and 1-ray units are unaffected, as they must be.
  the _shard_ctx noise slice counted from the start of the chunk the shard begins in: (B) bitwise in all 4 cases, and C6's
      bitwise shard outputs at N = 2, 4, 8.
  the regulariser added in gradients() as well as in Adam: C5's latent-row check (error / regulariser = 1.0) in all 8 cases.
"""
import math
import types

import pytest
import torch

import nerface_oracle as O
import torch_reference as TR
from test_backward_fp64_gpu import TOL, check, grad_pairs, reference
from test_backward_gpu import dev_tensor

pytestmark = pytest.mark.gpu

NEAR, FAR = 0.2, 0.8
NAMES = ("rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine", "w_last")
PRECS = ["exact", "fast"]
U = 2.0 ** -24
NC, NF, BATCH, LAT_ROW, REG = 64, 64, 2048, 2, 0.005   # the production training batch


def gamma(k):
    return k * U / (1.0 - k * U)


@pytest.fixture(scope="module")
def S(built_lib):
    import nerf
    from nerf import _engine, fused_train, parallel, train_utils
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    s = types.SimpleNamespace(nerf=nerf, fused_train=fused_train, parallel=parallel, train_utils=train_utils,
                              dev=torch.device("cuda", 0))
    s.eng = _engine.renderer_for(s.dev)
    s.sms = torch.cuda.get_device_properties(0).multi_processor_count
    s.cache = {}
    return s


def fresh_model(S, seed, stress=False, edit=None):
    """A new module (FusedTrainer turns its parameters into views of the trainer's bucket, so no two users share one)."""
    m = S.nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                          include_input_xyz=True, include_input_dir=False)
    p = O.random_init_params(seed, stress)
    if edit is not None:
        edit(p)
    m.load_state_dict(p)
    return m.to(S.dev)


def shards(S, H, N):
    return [S.parallel.shard_rows(H, N, r) for r in range(N)]


# ================================================================================================================ (A)
GEOMS = {"64c128f": (64, 128, 2), "128c256f": (128, 256, 1)}   # (coarse, fine, rays per unit)
FRAMES = {"128x128": (128, 128), "97x97": (97, 97), "129x64": (129, 64)}
SPLITS_A = [2, 3, 4, 5, 8, "H"]
OPTS_A = {"bg": dict(bg=True, white=False), "white": dict(bg=False, white=True), "none": dict(bg=False, white=False)}


def frame_setup(S, H, W, geom):
    fr = O.synthetic_frame(31, H, W)
    if geom not in S.cache:
        S.cache[geom] = (fresh_model(S, 100, True), fresh_model(S, 101, True))
    mc, mf = S.cache[geom]
    S.eng.sync_weights(mc, mf)
    S.eng.set_frame(fr["expr"].to(S.dev), fr["latent"].to(S.dev))
    return fr, fr["bg"].reshape(-1, 3).to(S.dev).contiguous()


def render_rows(S, fr, H, W, begin, rows, nc, nf, bg, white, prec):
    return S.eng.render_camera(fr["pose"], fr["intrinsics"], H, W, begin, rows, NEAR, FAR, nc, nf,
                               background=bg[begin * W:(begin + rows) * W].contiguous() if bg is not None else None,
                               precision=prec, white_bkgd=white)


def assert_concat_equal(full, parts, tag):
    for k in NAMES:
        cat = torch.cat([p[k] for p in parts], dim=0)
        assert cat.shape == full[k].shape and torch.equal(cat, full[k]), (tag, k)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("frame", list(FRAMES))
def test_row_shards_bit_identical(S, frame, geom, prec):
    """Every split N in 2, 3, 4, 5, 8 and H (one row per shard), with a background image, on white without one, and with
    neither: the shards' outputs, concatenated in rank order, are the full-frame call's bit for bit."""
    H, W = FRAMES[frame]
    nc, nf, R = GEOMS[geom]
    fr, bg_all = frame_setup(S, H, W, geom)
    if frame == "97x97":
        assert W % 2 == 1 and math.ceil(W / R) < S.sms  # a one-row shard: fewer units than SMs
    for opt, o in OPTS_A.items():
        bg = bg_all if o["bg"] else None
        full = render_rows(S, fr, H, W, 0, H, nc, nf, bg, o["white"], prec)
        for N in SPLITS_A:
            N = H if N == "H" else N
            parts = [render_rows(S, fr, H, W, b, r, nc, nf, bg, o["white"], prec) for b, r in shards(S, H, N)]
            torch.cuda.synchronize()
            assert_concat_equal(full, parts, (frame, geom, prec, opt, N))
        assert bool(torch.isfinite(full["_buf"]).all())


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("geom", list(GEOMS))
def test_row_shards_bit_identical_512(S, geom, prec):
    H = W = 512
    nc, nf, _ = GEOMS[geom]
    fr, bg = frame_setup(S, H, W, geom)
    full = render_rows(S, fr, H, W, 0, H, nc, nf, bg, False, prec)
    parts = [render_rows(S, fr, H, W, b, r, nc, nf, bg, False, prec) for b, r in shards(S, H, 8)]
    torch.cuda.synchronize()
    assert_concat_equal(full, parts, (512, geom, prec))


def unpack(buf, n):
    f = buf.view(-1)
    return dict(rgb_coarse=f[0:3 * n].view(n, 3), disp_coarse=f[3 * n:4 * n], acc_coarse=f[4 * n:5 * n], rgb_fine=f[5 * n:8 * n].view(n, 3),
                disp_fine=f[8 * n:9 * n], acc_fine=f[9 * n:10 * n], w_last=f[10 * n:11 * n])


@pytest.mark.parametrize("prec", PRECS)
def test_ragged_shards_host_entry_and_explicit_rays(S, prec):
    """129x64 over 5 ranks (26, 26, 26, 26, 25 rows): every shard through render_frame_host (the bench e2e leg) gives the full
    frame's bytes, and every shard equals render() on the explicit O.ray_bundle rays of its pixels, bit for bit."""
    H, W = 129, 64
    nc, nf, _ = GEOMS["64c128f"]
    fr, bg = frame_setup(S, H, W, "64c128f")
    full = render_rows(S, fr, H, W, 0, H, nc, nf, bg, False, prec)
    torch.cuda.synchronize()
    fbuf = {k: full[k].cpu() for k in NAMES}
    ro, rd = O.ray_bundle(H, W, fr["intrinsics"], fr["pose"])
    expr_h, lat_h = fr["expr"].contiguous().pin_memory(), fr["latent"].contiguous().pin_memory()
    bg_h = fr["bg"].reshape(-1, 3).contiguous()
    for b, r in shards(S, H, 5):
        n = r * W
        out_h = torch.empty(11 * n).pin_memory()
        S.eng.render_frame_host(fr["pose"], fr["intrinsics"], H, W, b, r, NEAR, FAR, expr_h, lat_h,
                                bg_h[b * W:(b + r) * W].contiguous().pin_memory(), nc, nf, out_h, precision=prec)
        for k, v in unpack(out_h, n).items():  # render_camera's packed [11, n] layout
            assert torch.equal(v, fbuf[k][b * W:(b + r) * W]), (b, r, k)
        S.eng.set_frame(fr["expr"].to(S.dev), fr["latent"].to(S.dev))
        ex = S.eng.render(ro[b:b + r].reshape(-1, 3).to(S.dev), rd[b:b + r].reshape(-1, 3).to(S.dev), NEAR, FAR, nc, nf,
                          background=bg[b * W:(b + r) * W], precision=prec)
        torch.cuda.synchronize()
        for k in NAMES:
            assert torch.equal(ex[k], full[k][b * W:(b + r) * W]), (b, r, k)


# ================================================================================================================ (B)
def eval_cfg(S, chunk):
    """The shipped YAML's validation block: perturb: True (stochastic evaluation), 64 + 64 samples."""
    blk = dict(num_coarse=64, num_fine=64, perturb=True, lindisp=False, radiance_field_noise_std=0.0, white_background=False,
               chunksize=chunk)
    return S.nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, validation=blk, train=blk), dataset=dict(no_ndc=True, near=NEAR, far=FAR)))


def run_sharded(S, run, N, seed, ro, rd, bg, ctx_of, **kw):
    """Rank r's call of the drop-in wrapper's body, for r in rank order: seeded as every rank is, _shard_ctx set, the rank's
    rows / rays and background."""
    outs = []
    for r in range(N):
        begin, cnt, ctx = ctx_of(r)
        torch.manual_seed(seed)
        S.train_utils._shard_ctx = ctx
        try:
            outs.append(run(begin, cnt, ro, rd, bg, **kw))
        finally:
            S.train_utils._shard_ctx = None
    return outs


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("ablation", [False, True], ids=["plain", "ablation"])
def test_stochastic_validation_sharded_by_shard_ctx(S, ablation, prec):
    """37 x 29 (1073 rays) in chunks of 100, or with the ablation bundle (every chunk must be as long as chunk 0, so the chunks
    divide the frame) 36 x 29 in chunks of 36: no shard boundary falls on a chunk boundary, so the single-process chunks whose
    noise each shard slices straddle the shards."""
    H, W, chunk = (36, 29, 36) if ablation else (37, 29, 100)
    nerf = S.nerf
    fr = O.synthetic_frame(33, H, W)
    mc, mf = fresh_model(S, 100), fresh_model(S, 101)
    cfg = eval_cfg(S, chunk)
    ro, rd = nerf.get_ray_bundle(H, W, fr["intrinsics"], fr["pose"].to(S.dev))
    bg = fr["bg"].reshape(-1, 3).to(S.dev)
    fr2 = O.synthetic_frame(34, H, W)
    abl = nerf.get_ray_bundle(H, W, fr2["intrinsics"], fr2["pose"].to(S.dev))[1] if ablation else None
    kw = dict(expressions=fr["expr"].to(S.dev), latent_code=fr["latent"].to(S.dev), ray_directions_ablation=abl)
    nerf.set_precision(prec)
    try:
        with torch.no_grad():
            torch.manual_seed(9)
            full = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro, rd, cfg, mode="validation", background_prior=bg, **kw)

            def run(begin, rows, ro, rd, bg, **kw):
                sl = slice(begin, begin + rows)
                return nerf.run_one_iter_of_nerf(rows, W, fr["intrinsics"], mc, mf, ro[sl], rd[sl], cfg, mode="validation",
                                                 background_prior=bg.reshape(H, W, 3)[sl].reshape(-1, 3), **kw)
            for N in (2, 3, 5):
                parts = shards(S, H, N)
                assert all((b * W) % chunk for b, _ in parts[1:])  # every shard starts inside a chunk
                if ablation:
                    assert (H * W) % chunk == 0
                else:
                    assert (H * W) % chunk and all((r * W) % chunk for _, r in parts)
                outs = run_sharded(S, run, N, 9, ro, rd, bg, lambda r: (*parts[r], (parts[r][0] * W, parts[r][1] * W, H * W)), **kw)
                for i, nme in enumerate(NAMES):
                    cat = torch.cat([o[i] for o in outs], dim=0)
                    assert cat.shape == full[i].shape and torch.equal(cat, full[i]), (N, nme)
            torch.manual_seed(10)
            other = nerf.run_one_iter_of_nerf(H, W, fr["intrinsics"], mc, mf, ro, rd, cfg, mode="validation", background_prior=bg, **kw)
            assert not torch.equal(other[3], full[3])  # the noise reaches the outputs: another seed renders other pixels
    finally:
        nerf.set_precision("fast")
        assert S.train_utils._shard_ctx is None


# ================================================================================================================ (C)
def batch(S):
    """2048 rays of a 64 x 64 frame, targets, the frame's expression and a latent table with a nonzero row LAT_ROW."""
    if "batch" not in S.cache:
        fr = O.synthetic_frame(35, 64, 64)
        ro, rd = O.ray_bundle(64, 64, fr["intrinsics"], fr["pose"])
        g = torch.Generator().manual_seed(36)
        sel = torch.randperm(64 * 64, generator=g)[:BATCH]
        S.cache["batch"] = types.SimpleNamespace(
            ro=ro.reshape(-1, 3)[sel].to(S.dev).contiguous(), rd=rd.reshape(-1, 3)[sel].to(S.dev).contiguous(),
            bg=fr["bg"].reshape(-1, 3)[sel].to(S.dev).contiguous(), tgt=torch.rand(BATCH, 3, generator=g).to(S.dev),
            expr=fr["expr"].to(S.dev), table=(torch.randn(4, 32, generator=g) * 0.1).to(S.dev), intr=fr["intrinsics"])
    return S.cache["batch"]


def trainer(S, prec, b, mc=None, mf=None, perturb=True):
    mc = mc if mc is not None else fresh_model(S, 100)
    mf = mf if mf is not None else fresh_model(S, 101)
    return S.fused_train.FusedTrainer(mc, mf, n_latent=4, num_coarse=NC, num_fine=NF, perturb=perturb, noise_std=0.1, near=NEAR,
                                      far=FAR, latent_reg=REG, latent_codes=b.table, precision=prec)


def draw_batch_noise(tr, seed=77):
    torch.manual_seed(seed)
    return tr._draw_noise(BATCH)


def run_shard(S, tr, b, lo, hi, noise, target=None):
    """FusedTrainer.gradients on rays [lo, hi) of the batch (world=1, n_total = the batch): copies of everything the next
    call overwrites — bucket, loss share, grad_rgb, depths, loss scale — and the shard's colours (the same render again)."""
    sl = slice(lo, hi)
    nz = {k: (v[sl].contiguous() if v is not None else None) for k, v in noise.items()}
    tgt = b.tgt[sl] if target is None else target
    tr.grads.zero_()
    loss = tr.gradients(b.ro[sl], b.rd[sl], tgt, b.expr, LAT_ROW, background=b.bg[sl], world=1, n_total=BATCH, noise=nz)
    torch.cuda.synchronize()
    n = hi - lo
    d = tr.eng.train_debug()
    sh = types.SimpleNamespace(lo=lo, hi=hi, n=n, noise=nz, tgt=tgt, bucket=tr.grads.clone(), loss=loss.clone(),
                               g=[t.clone() for t in tr._g_rgb[n]], scale=dev_tensor(d.scale, (2,)).clone(),
                               z_c=dev_tensor(d.z_coarse, (n, NC)).clone(), z_f=dev_tensor(d.z_fine, (n, NC + NF)).clone())
    out = tr.eng.render(b.ro[sl], b.rd[sl], NEAR, FAR, NC, NF, perturb=tr.opts["perturb"], noise_std=0.1, background=b.bg[sl],
                        noise=nz, precision=tr.opts["precision"], train=True)
    torch.cuda.synchronize()
    sh.rgb = (out["rgb_coarse"].clone(), out["rgb_fine"].clone())
    tr.grads.zero_()
    return sh


def split_bucket(tr, flat):
    """(coarse grads, fine grads, latent row) views of a bucket, None for the unused layers_dir.3; and a mask of the entries
    no gradient may reach (layers_dir.3, the padding, the other latent rows)."""
    views, off = [], 0
    for v in tr._views:
        views.append(flat[off:off + v.numel()].view(v.shape))
        off += v.numel()
    skip = [k.startswith("layers_dir.3") for k in TR.PARAM_ORDER]
    gc = [None if s else t for s, t in zip(skip, views[:26])]
    gf = [None if s else t for s, t in zip(skip, views[26:])]
    lat = flat[tr.lat_off + 32 * LAT_ROW:tr.lat_off + 32 * LAT_ROW + 32]
    unused = torch.zeros(flat.numel(), dtype=torch.bool, device=flat.device)
    off = 0
    for i, v in enumerate(tr._views):
        if skip[i % 26]:
            unused[off:off + v.numel()] = True
        off += v.numel()
    unused[off:] = True
    unused[tr.lat_off + 32 * LAT_ROW:tr.lat_off + 32 * LAT_ROW + 32] = False
    return (gc, gf, lat), unused


def shard_case(tr, b, sh):
    """The shard as test_backward_fp64_gpu.reference takes a case."""
    return types.SimpleNamespace(n=sh.n, nc=NC, nf=NF, noise_std=0.1, noise={k: v for k, v in sh.noise.items() if v is not None},
                                 white=False, bg=b.bg[sh.lo:sh.hi], dz=None, mc=tr.mc, mf=tr.mf, expr=b.expr,
                                 latent=tr.latent_codes[LAT_ROW].detach().clone(), ro=b.ro[sh.lo:sh.hi], rd=b.rd[sh.lo:sh.hi])


def ref_sum(refs):
    """Parameter / latent gradients are linear in the output gradients: the float64 gradient of the whole batch is the sum of
    the shards' float64 gradients."""
    add = lambda xs: None if xs[0] is None else sum(xs[1:], xs[0].clone())  # noqa: E731
    return types.SimpleNamespace(gc=[add([r.gc[i] for r in refs]) for i in range(26)],
                                 gf=[add([r.gf[i] for r in refs]) for i in range(26)], glat=add([r.glat for r in refs]))


def shard_tol(prec, n):
    """TOL for shards of 512 rays or more; twice its max bound for the 256-ray shards of N = 8 (module docstring)."""
    return TOL[prec] if n >= 512 else (2.0 * TOL[prec][0], TOL[prec][1])


def stage_loss(tag, sh):
    """C1: grad_rgb bitwise the FP32 expression in the kernel's order; the loss share against float64."""
    f32 = lambda v: torch.tensor(v, dtype=torch.float32)  # noqa: E731
    inv = (f32(1.0) / (f32(3.0) * f32(float(BATCH)))).to(sh.tgt.device)
    worst = 0.0
    for p, (rgb, g) in enumerate(zip(sh.rgb, sh.g)):
        want = (2.0 * (rgb - sh.tgt)) * inv
        assert torch.equal(g, want), (tag, p, float((g - want).abs().max()))
        ref = float(((rgb.double() - sh.tgt.double()) ** 2).sum()) / (3.0 * BATCH)
        bound = gamma(3 * sh.n + 32) * ref
        err = abs(float(sh.loss[p]) - ref)
        assert err <= bound, (tag, p, err, bound)
        worst = max(worst, err / bound)
    return worst


SPLITS_C = {"2": [1024] * 2, "4": [512] * 4, "8": [256] * 8, "1000+1048": [1000, 1048]}


def control(S, prec):
    """C4: the whole batch in one gradients() call, from the same state and noise."""
    key = ("control", prec)
    if key not in S.cache:
        b = batch(S)
        tr = trainer(S, prec, b)
        noise = draw_batch_noise(tr)
        sh = run_shard(S, tr, b, 0, BATCH, noise)
        S.cache[key] = (tr, noise, sh)
    return S.cache[key]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("split", list(SPLITS_C))
def test_sharded_training_batch_against_float64(S, split, prec):
    """The production batch split over N = 2, 4, 8 equal shards or 1000 + 1048 rays, stages C1 to C6 of the module docstring."""
    b = batch(S)
    ctl_tr, noise, ctl = control(S, prec)
    tr = trainer(S, prec, b)
    bounds = [0] + list(torch.cumsum(torch.tensor(SPLITS_C[split]), 0).tolist())
    assert bounds[-1] == BATCH
    shs = [run_shard(S, tr, b, lo, hi, noise) for lo, hi in zip(bounds[:-1], bounds[1:])]
    N = len(shs)
    worst = {}

    # ---- C1: the loss gradient and the loss shares
    worst["C1 share / bound"] = max(stage_loss(f"{split} {prec} shard {r}", sh) for r, sh in enumerate(shs))
    for p in (0, 1):
        shares64 = [float(((sh.rgb[p].double() - sh.tgt.double()) ** 2).sum()) / (3.0 * BATCH) for sh in shs]
        got = sum(float(sh.loss[p]) for sh in shs)
        bound = sum(gamma(3 * sh.n + 32) * r for sh, r in zip(shs, shares64))
        assert abs(got - sum(shares64)) <= bound, (p, got, sum(shares64), bound)

    # ---- C4 (part): the unsharded call saw the same depths and output gradients, bit for bit
    for sh in shs:
        sl = slice(sh.lo, sh.hi)
        assert torch.equal(sh.z_c, ctl.z_c[sl]) and torch.equal(sh.z_f, ctl.z_f[sl]), (split, sh.lo)
        assert all(torch.equal(a, c[sl]) for a, c in zip(sh.g, ctl.g)), (split, sh.lo)

    # ---- C2: every shard's backward against float64 at its own depths and grad_rgb
    refs = []
    lat = tr.latent_codes[LAT_ROW].detach().double()
    reg64 = REG * lat / lat.norm()
    for r, sh in enumerate(shs):
        gouts = [sh.g[0], None, None, sh.g[1], None, None, None]
        R = reference(S, shard_case(tr, b, sh), sh.z_c, sh.z_f, gouts)
        refs.append(R)
        kg, unused = split_bucket(tr, sh.bucket)
        assert float(sh.bucket[unused].abs().max()) == 0.0, (split, r)
        # C5 (part): the latent row is the backward's alone: its error is far below the regulariser's gradient
        lat_err = float((kg[2].double() - R.glat).abs().max()) / float(reg64.abs().max())
        worst["C5 latent err / reg"] = max(worst.get("C5 latent err / reg", 0.0), lat_err)
        assert lat_err < 0.5, (split, r, lat_err)
        em, el = check(f"C2 {split} {prec} shard {r}", grad_pairs(kg, R), shard_tol(prec, sh.n))
        worst["C2"] = max(worst.get("C2", (0, 0)), (em, el))

    # ---- C3: the emulated SUM all-reduce
    R_all = ref_sum(refs)
    sum64 = sum((sh.bucket.double() for sh in shs[1:]), shs[0].bucket.double().clone())
    sum32 = shs[0].bucket.clone()
    for sh in shs[1:]:
        sum32 = sum32 + sh.bucket
    absum = sum((sh.bucket.double().abs() for sh in shs[1:]), shs[0].bucket.double().abs())
    assert bool(((sum32.double() - sum64).abs() <= gamma(N) * absum).all()), split
    kg64, _ = split_bucket(tr, sum64)
    worst["C3"] = check(f"C3 {split} {prec} sum of {N}", grad_pairs(kg64, R_all), TOL[prec])

    # ---- C4: the unsharded control against the same float64 gradient
    kgc, unused = split_bucket(ctl_tr, ctl.bucket)
    assert float(ctl.bucket[unused].abs().max()) == 0.0
    worst["C4"] = check(f"C4 unsharded {prec}", grad_pairs(kgc, R_all), TOL[prec])

    # ---- C5: Adam on the summed bucket adds the regulariser once
    tas = [trainer(S, prec, b) for _ in range(2)]
    for t in tas:
        t.grads.copy_(sum32)
        t._reg_row = LAT_ROW
        t.update()
    torch.cuda.synchronize()
    assert torch.equal(tas[0].params, tas[1].params)
    p0 = trainer(S, prec, b).params.double()
    g64 = sum32.double().clone()
    row = slice(tr.lat_off + 32 * LAT_ROW, tr.lat_off + 32 * LAT_ROW + 32)
    g64[row] += REG * p0[row] / p0[row].norm()
    b1, b2, eps, lr = 0.9, 0.999, 1e-8, 5e-4
    m, v = (1 - b1) * g64, (1 - b2) * g64 * g64
    want = p0 - lr / (1 - b1) * m / (v.sqrt() / math.sqrt(1 - b2) + eps)
    worst["C5 adam"] = float((tas[0].params.double() - want).abs().max())
    assert worst["C5 adam"] <= 1e-6, worst["C5 adam"]

    # ---- C6: the drop-in train shard (equal shards only: data_parallel's shard_batch)
    if len(set(SPLITS_C[split])) == 1:
        worst["C6"] = dropin_train(S, prec, b, N, R_all, reg64)
    print(f"{split} {prec}: " + ", ".join(f"{k} {v}" for k, v in worst.items()))


def dropin_train(S, prec, b, N, R_all, reg64):
    nerf, parallel = S.nerf, S.parallel
    blk = dict(num_coarse=NC, num_fine=NF, perturb=True, lindisp=False, radiance_field_noise_std=0.1, white_background=False,
               chunksize=BATCH)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk), dataset=dict(no_ndc=True, near=NEAR, far=FAR)))
    mc, mf = fresh_model(S, 100), fresh_model(S, 101)
    table = b.table.clone().requires_grad_(True)
    params = list(mc.parameters()) + list(mf.parameters())
    nerf.set_precision(prec)
    try:
        def call(sl):
            return nerf.run_one_iter_of_nerf(64, 64, b.intr, mc, mf, b.ro[sl], b.rd[sl], cfg, mode="train", expressions=b.expr,
                                             background_prior=b.bg[sl], latent_code=table[LAT_ROW])
        torch.manual_seed(77)
        full = [o.detach() for o in call(slice(0, BATCH))]
        per = BATCH // N
        outs = []
        for r in range(N):  # every rank's forward, seeded alike: its outputs are the unsharded call's rows
            begin, cnt = parallel.shard_batch(BATCH, N, r)
            torch.manual_seed(77)
            S.train_utils._shard_ctx = (begin, cnt, BATCH)
            try:
                o = call(slice(begin, begin + cnt))
            finally:
                S.train_utils._shard_ctx = None
            outs.append([t.detach() for t in o])
            for i, nme in enumerate(NAMES):
                assert torch.equal(outs[r][i], full[i][begin:begin + cnt]), (N, r, nme)
        acc = None
        for r in range(N):  # rank r's loss as the wrapper assembles it, its backward, the sum over ranks
            begin, cnt = parallel.shard_batch(BATCH, N, r)
            torch.manual_seed(77)
            S.train_utils._shard_ctx = (begin, cnt, BATCH)
            try:
                o = call(slice(begin, begin + cnt))
            finally:
                S.train_utils._shard_ctx = None
            rows = []
            for i in (0, 3):
                whole = torch.cat([outs[q][i] for q in range(N)], dim=0)
                rows.append(torch.cat((whole[:begin], parallel._ScaleGrad.apply(o[i], float(N)), whole[begin + per:]), dim=0))
            loss = torch.nn.functional.mse_loss(rows[0], b.tgt) + torch.nn.functional.mse_loss(rows[1], b.tgt) \
                + torch.norm(table[LAT_ROW]) * 0.0005 * 10
            loss.backward()
            g = [p.grad.double().clone() if p.grad is not None else None for p in params] + [table.grad[LAT_ROW].double().clone()]
            acc = g if acc is None else [None if a is None else a + c for a, c in zip(acc, g)]
            for p in params:
                p.grad = None
            table.grad = None
    finally:
        nerf.set_precision("fast")
    avg = [None if a is None else a / N for a in acc]
    names = [n for n, _ in mc.named_parameters()]
    gc = [avg[names.index(k)] for k in TR.PARAM_ORDER]
    gf = [avg[26 + names.index(k)] for k in TR.PARAM_ORDER]
    R = types.SimpleNamespace(gc=R_all.gc, gf=R_all.gf, glat=R_all.glat + reg64)
    return check(f"C6 drop-in {N} ranks {prec}", grad_pairs((gc, gf, avg[-1]), R), TOL[prec])


@pytest.mark.parametrize("prec", PRECS)
def test_shard_with_its_own_render_as_target(S, prec):
    """Two 1024-ray shards; the second's target is its own rendered colour.  The target is one image for both passes, so coarse
    and fine must render the same colours: both networks are the same opaque one (fc_alpha.bias + 3e4), and the fine pass's
    first sample is the coarse pass's.  Without perturbation that sample's interval is at least half a coarse spacing, so its
    alpha is exactly 1 and both passes return its colour.  That shard gets exactly zero output gradients, an exactly zero
    bucket and loss scale 1; the first shard, with random targets, does not."""
    b = batch(S)

    def opaque(p):
        p["fc_alpha.bias"] += 3e4
    tr = trainer(S, prec, b, fresh_model(S, 100, edit=opaque), fresh_model(S, 100, edit=opaque), perturb=False)
    noise = draw_batch_noise(tr)
    half = BATCH // 2
    sl = slice(half, BATCH)
    nz = {k: (v[sl].contiguous() if v is not None else None) for k, v in noise.items()}
    tr.eng.set_frame(b.expr, tr.latent_codes[LAT_ROW])
    out = tr.eng.render(b.ro[sl], b.rd[sl], NEAR, FAR, NC, NF, perturb=False, noise_std=0.1, background=b.bg[sl], noise=nz,
                        precision=prec)
    torch.cuda.synchronize()
    target = out["rgb_fine"].clone()
    assert torch.equal(out["rgb_coarse"], target)
    first = run_shard(S, tr, b, 0, half, noise)
    assert float(first.scale[0]) != 1.0 and float(first.bucket.abs().max()) > 0.0
    sh = run_shard(S, tr, b, half, BATCH, noise, target=target)
    assert torch.equal(sh.rgb[0], target) and torch.equal(sh.rgb[1], target)  # the same noise renders the same bits
    assert all(float(g.abs().max()) == 0.0 for g in sh.g)
    assert float(sh.loss.abs().max()) == 0.0
    assert float(sh.bucket.abs().max()) == 0.0 and bool(torch.isfinite(sh.bucket).all())
    assert float(sh.scale[0]) == 1.0 and float(sh.scale[1]) == 1.0
