"""The packed weight buffers every kernel reads (csrc/nfb_pack.cu: fold_feat_kernel, repack_kernel; read back through
nfb_debug_weights) against the numpy restatement of tests/weight_pack_reference.py and against float64, each case once through
nfb_load_weights (one network per call) and once through nfb_repack (both networks in one call):
  (1) every byte    0xFF (an FP16 / FP32 NaN) written into every byte of all ten buffers of both networks, then the load: x1,
                    x3, bwd, bias_static, w0c, w3c and wd0b_t equal the restatement bit for bit (so every byte is written), w6
                    / b6 rows 129..143 are +0, and bias_frame after nfb_set_frame equals bias_static outside the rows of steps 0
                    and 3.  The restatement takes the fold's FP32 result from the kernel (its rounding is checked in (3)); a
                    position whose expected value is NaN must hold a NaN that is not the poison (the payload of a NaN is the
                    converter's: numpy and the device produce different ones).  Parameters: random-init, opaque-stress, and
                    adversarial ones planted in every tensor — FP16 rounding ties, values in and below FP16's subnormal range
                    (1e-6, 2^-24, 2^-25, 3 2^-25), +-65504, 65519.996 (still 65504) and 65520 (inf), -0.0 — and a non-finite
                    set (NaN, +-inf: hi = inf, lo = NaN, and a NaN or inf anywhere in the fold's inputs makes its outputs so).
  (2) exact split   every x3 (hi, lo) pair with both halves finite satisfies |hi + lo - w| <= max(2^-22 |w|, 2^-25) (the 2^-25
                    floor: lo below FP16's normal range); a half is non-finite exactly where w is non-finite or |w| >= 65520.
  (3) fold          w6 / b6 rows 0..128 against the float64 fold of the FP32 parameters (compensated sums of the exact
                    products): |got - ref| <= 1/2 ulp32 + gamma64(66) sum |a b| for W6 (four float64 chains of 64 terms and
                    their combination), gamma64(257) sum for b6; one case has a row of layers_dir.0 orthogonal to a column of
                    fc_feat up to one ulp, and fc_alpha to another, where the bound's absolute term is all there is.
  (4) transitions   nfb_load_weights of each network == nfb_repack of both, byte for byte; a repeated nfb_repack changes
                    nothing; nfb_repack(params_fine = NULL) leaves network 1's buffers bit for bit as they were.
  (5) training      after each of 3 eager FusedTrainer.step, 3 step_graph replays and 3 step_images_graph replays (K = 2), and
                    with two trainers alternating on the device's one renderer, both networks' buffers equal the restatement
                    of the trainer's bucket at that moment (the graphs' re-pack reads parameter pointers fixed at capture).

Measured on an H100 80GB HBM3 at a 700 W power limit (CUDA 12.9): every buffer bit for bit in every case; the split's
relative error at most 1.0 (a weight below 2^-25 whose lo rounds to 0) with median 5.1e-7 on random-init and 2.4e-7 on
opaque-stress weights, never above the bound; W6 / b6 equal to the FP32 rounding of the float64 fold in every element of
every case, the cancelling rows included.  The file takes about 20 s.

Planted defects, each built once on a scratch copy of csrc/nfb_pack.cu, with the checks that caught them here:
  swizzle XOR on n & 3 (forward and backward units):  (1) x1 differs, every case; (2); (4); (5).
  lo written as fp16(w):                              (1) x3 differs, every case; (2) the split bound; (4); (5).
  step 3's conditioning-column offset off by one:     (1) x1 differs in step 3's hidden atoms, every case; (2); (4); (5).
  padding rows of the forward units left unwritten:   (1) x1 rows 129..143 of step 6 / 3..15 of step 9 hold the poison;
                                                      (2) non-finite halves where w is +0; (4).  (5) passes: fresh device
                                                      memory happened to be zero.
  W6 accumulated in FP32:                             (3) at 2e4 - 5e4 times the fold bound, every case; (4); (5).
What the existing stage-by-stage suites saw: test_render_fp64_gpu.py caught the swizzle (44 of 64 tests), lo (22, exact mode
only) and the column offset (44), and missed the unwritten padding and the FP32 fold; test_param_backward_fp64_gpu.py
caught the swizzle (24 of 29), lo (1, exact mode) and the FP32 fold (15, its dX-chain stage streams the fold), and missed
the column offset and the unwritten padding.  The unwritten padding passed both: the activations it multiplies are 0.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import nerface_oracle as O
import weight_pack_reference as R
from test_backward_gpu import dev_tensor

pytestmark = pytest.mark.gpu

U64 = 2.0 ** -53
POISON16, POISON32 = 0xFFFF, 0xFFFFFFFF
FLOAT_BUFS = dict(w6=144 * 256, b6=144, bias_static=R.BIAS_FLOATS, bias_frame=R.BIAS_FLOATS, w0c=256 * 108, w3c=256 * 108,
                  wd0b_t=24 * 128)


def gamma64(n):
    return n * U64 / (1 - n * U64)


@pytest.fixture(scope="module")
def env(built_lib):
    import nerf
    from nerf import _capi, _engine
    dev = torch.device("cuda", 0)
    return nerf, _capi, _engine, dev, R.Layout(_capi.lib)


@pytest.fixture(scope="module")
def eng(env):
    _, _, _engine, dev, _ = env
    return _engine.Renderer(dev)  # its own handle: nothing else packs into it


def views(eng, net):
    """Integer views of network net's ten buffers (int16 for the FP16 streams, int32 for the FP32 ones): read and poison."""
    d = eng.weights_debug(net)
    assert (d.x1_bytes, d.x3_bytes, d.bwd_bytes, d.bias_floats) == (R.X1_BYTES, 2 * R.X1_BYTES, R.BWD_BYTES, R.BIAS_FLOATS)
    out = {k: dev_tensor(getattr(d, k), (getattr(d, k + "_bytes") // 2,), "<i2") for k in ("x1", "x3", "bwd")}
    out.update({k: dev_tensor(getattr(d, k), (n,), "<i4") for k, n in FLOAT_BUFS.items()})
    return out


def read(eng, net):
    torch.cuda.synchronize()
    v = views(eng, net)
    return {k: t.cpu().numpy().view(np.uint16 if t.dtype == torch.int16 else np.uint32) for k, t in v.items()}


def poison(eng):
    for net in (0, 1):
        for t in views(eng, net).values():
            t.fill_(-1)
    torch.cuda.synchronize()


def dev_params(p, dev):
    return [torch.as_tensor(a).to(dev).contiguous() for a in p]


def load(env, eng, pc, pf, how):
    """Pack FP32 tensors (lists in PARAM_ORDER) through nfb_load_weights per network ("load") or one nfb_repack ("repack")."""
    _, capi, _engine, dev, _ = env
    tc = dev_params(pc, dev)
    tf = dev_params(pf, dev) if pf is not None else None
    if how == "load":
        for which, ts in ((0, tc), (1, tf)):
            if ts is not None:
                arr = (C.c_void_p * 26)(*[t.data_ptr() for t in ts])
                capi.check(capi.lib.nfb_load_weights(eng._h, which, arr, _engine._stream()), "load_weights")
    else:
        eng.repack(tc, tf)
    torch.cuda.synchronize()


# ---- parameters
SPECIALS = np.array([1 + 2 ** -11, 1 + 3 * 2 ** -11, -(1 + 2 ** -11), 0.0625 * (1 + 2 ** -11), 0.0625 * (1 - 2 ** -12),
                     2049.0 * 2 ** -14, 1e-6, -1e-6, 2 ** -24, 2 ** -25, -(2 ** -25), 3 * 2 ** -25, 2 ** -26, 6e-8, 2 ** -14,
                     2 ** -14 * (1 - 2 ** -11), 65504.0, -65504.0, 65519.996, 65520.0, -70000.0, -0.0], np.float32)
NONFINITE = np.array([np.nan, np.inf, -np.inf], np.float32)


def plant(p, vals, seed, per_tensor):
    """Overwrite `per_tensor` spread-out elements of every tensor with vals (cycled from a per-tensor offset), and the
    boundary columns 62, 63, 170 of layers_xyz.0 / .3 (and 171, 426 of .3) in a few rows."""
    rng = np.random.default_rng(seed)
    out = [a.copy() for a in p]
    for t, a in enumerate(out):
        f = a.reshape(-1)
        pos = rng.choice(f.size, size=min(per_tensor, f.size), replace=False)
        f[pos] = vals[(np.arange(pos.size) + 7 * t) % vals.size]
    for t, cols in ((0, (62, 63, 170)), (6, (62, 63, 170, 171, 426))):
        for i, c in enumerate(cols):
            out[t][(5 * i + t) % 256, c] = vals[(3 * i + t) % vals.size]
    return out


def cancel(p):
    """Row 5 of layers_dir.0[:, :256] orthogonal to column 9 of fc_feat, and fc_alpha to column 200, up to one ulp:
    left[2i] = v[2i+1], left[2i+1] = -v[2i] cancels pairwise; one element moved by an ulp leaves a residue ~ 1e-9 of sum |a b|."""
    out = [a.copy() for a in p]
    for row, col in ((out[16][5], 9), (out[14][0], 200)):
        v = out[12][:, col]
        row[0:256:2], row[1:256:2] = v[1::2], -v[0::2]
        row[7] = np.nextafter(row[7], np.float32(np.inf))
    return out


def params(case, seed):
    if case == "stress":
        return R.flat_params(O.random_init_params(seed, True))
    p = R.flat_params(O.random_init_params(seed))
    if case == "adversarial":
        return plant(p, SPECIALS, seed, 97)
    if case == "nonfinite":
        return plant(p, np.concatenate([SPECIALS, NONFINITE]), seed, 9)
    if case == "cancel":
        return cancel(p)
    return p


# ---- checks
def same_bits(got, exp, name, poison_bits):
    """got (uint view) == exp bit for bit, except where exp is NaN: there got must be a NaN other than the poison."""
    fl = np.float16 if got.dtype == np.uint16 else np.float32
    exp = np.asarray(exp).view(got.dtype)
    nan_e = np.isnan(exp.view(fl))
    bad = (got != exp) & ~nan_e
    bad |= nan_e & (~np.isnan(got.view(fl)) | (got == poison_bits))
    assert not bad.any(), f"{name}: {int(bad.sum())} of {got.size} differ, first at {np.flatnonzero(bad)[:8]}"


def check_fold(got, p, label):
    """w6 / b6 against the float64 fold; rows 129..143 exactly +0.  Returns the number of W6 elements that are not the FP32
    rounding of the float64 value."""
    w6 = got["w6"].view(np.float32).reshape(144, 256)
    b6 = got["b6"].view(np.float32)
    assert (got["w6"].reshape(144, 256)[129:] == 0).all() and (got["b6"][129:] == 0).all(), f"{label}: fold padding rows"
    ref_w, ref_b, abs_w, abs_b = R.fold64(p)
    off = 0
    for g, ref, absum, gam in ((w6[:129], ref_w[:129], abs_w[:129], gamma64(66)), (b6[:129], ref_b[:129], abs_b[:129], gamma64(257))):
        with np.errstate(over="ignore", invalid="ignore"):
            r32 = ref.astype(np.float32)
            fin = np.isfinite(r32)
            assert np.array_equal(np.isfinite(g), fin), f"{label}: fold non-finite pattern"
            assert np.array_equal(g[np.isinf(r32)], r32[np.isinf(r32)]), f"{label}: fold infinities"
            gf, rf = g[fin].astype(np.float64), ref[fin]
            ulp = np.spacing(np.maximum(np.abs(g[fin]), np.abs(r32[fin])).astype(np.float32)).astype(np.float64)
            bound = 0.5 * ulp + gam * absum[fin]
            err = np.abs(gf - rf)
        worst = float((err / bound).max()) if err.size else 0.0
        assert worst <= 1.0, f"{label}: fold error {worst:.3g} of its bound"
        off += int((g[fin] != r32[fin]).sum())
    return off


def check_net(env, got, p, label):
    """Every buffer of one network against the restatement of p (fold from the kernel, checked by check_fold)."""
    layout = env[4]
    off = check_fold(got, p, label)
    exp = R.expected(p, got["w6"].view(np.float32).reshape(144, 256), got["b6"].view(np.float32), layout)
    for k in ("x1", "x3", "bwd"):
        same_bits(got[k], exp[k], f"{label} {k}", POISON16)
    for k in ("bias_static", "w0c", "w3c", "wd0b_t"):
        same_bits(got[k], exp[k].ravel(), f"{label} {k}", POISON32)
    return off


def check_split(env, got, p, label):
    """(2): the x3 pairs against the FP32 weights; returns (max, median) relative error over nonzero finite weights."""
    layout = env[4]
    vals = R.values(p, got["w6"].view(np.float32).reshape(144, 256))
    src = layout.x3[layout.x3_hi_slot]
    w = vals[np.where(src < 0, len(vals) - 1, src)].astype(np.float64)
    hi = got["x3"][layout.x3_hi_slot].view(np.float16).astype(np.float64)
    lo = got["x3"][layout.x3_lo_slot].view(np.float16).astype(np.float64)
    fin = np.isfinite(hi) & np.isfinite(lo)
    assert np.array_equal(~fin, ~np.isfinite(w) | (np.abs(w) >= 65520)), f"{label}: non-finite halves"
    err = np.abs(hi[fin] + lo[fin] - w[fin])
    wf = np.abs(w[fin])
    assert (err <= np.maximum(2.0 ** -22 * wf, 2.0 ** -25)).all(), f"{label}: split bound, worst abs {err.max():.3g}"
    nz = wf > 0
    rel = err[nz] / wf[nz]
    return float(rel.max()), float(np.median(rel))


def check_frame(got, p, expr, latent, label):
    """bias_frame: bias_static bit for bit outside rows 0..255 and 768..1023; those rows within gamma32(109) of float64."""
    bf, bs = got["bias_frame"], got["bias_static"]
    keep = np.ones(R.BIAS_FLOATS, bool)
    keep[0:256] = keep[768:1024] = False
    assert np.array_equal(bf[keep], bs[keep]), f"{label}: bias_frame outside the folded rows"
    ref, absum = R.frame_rows64(p, bs.view(np.float32), expr, latent)
    u = 2.0 ** -24
    for i0 in (0, 768):
        g = bf[i0:i0 + 256].view(np.float32).astype(np.float64)
        fin = np.isfinite(ref[i0])
        assert np.array_equal(np.isfinite(g), fin), f"{label}: folded rows non-finite pattern"
        assert (np.abs(g[fin] - ref[i0][fin]) <= (112 * u / (1 - 112 * u)) * absum[i0][fin]).all(), f"{label}: folded rows"


CASES = ["random", "stress", "adversarial", "nonfinite", "cancel"]


@pytest.mark.parametrize("how", ["load", "repack"])
@pytest.mark.parametrize("case", CASES)
def test_every_byte(env, eng, case, how):
    """(1) + (3): old parameters packed, every byte of both networks' ten buffers poisoned, the case's parameters packed over
    them; then nfb_set_frame for bias_frame."""
    dev = env[3]
    load(env, eng, params("random", 900), params("random", 901), "repack")
    poison(eng)
    pc, pf = params(case, 11), params(case, 12)
    load(env, eng, pc, pf, how)
    fr = O.synthetic_frame(4, 4, 4)
    eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
    offs = []
    for net, p in ((0, pc), (1, pf)):
        got = read(eng, net)
        offs.append(check_net(env, got, p, f"{case}/{how} net {net}"))
        check_frame(got, p, fr["expr"].numpy(), fr["latent"].numpy(), f"{case}/{how} net {net}")
    print(f"\n{case}/{how}: all buffers bit for bit; W6/b6 elements not the FP32 rounding of float64: {offs}")


@pytest.mark.parametrize("case", ["random", "stress", "adversarial", "nonfinite"])
def test_exact_split_bound(env, eng, case):
    """(2), with the measured max / median relative error printed."""
    pc, pf = params(case, 21), params(case, 22)
    load(env, eng, pc, pf, "repack")
    for net, p in ((0, pc), (1, pf)):
        mx, med = check_split(env, read(eng, net), p, f"{case} net {net}")
        print(f"\n{case} net {net}: |hi + lo - w| / |w| max {mx:.3g} median {med:.3g}")


def test_state_transitions(env, eng):
    """(4): load == repack, repack idempotent, repack(fine = NULL) leaves network 1 alone (and still loaded)."""
    a = (params("random", 31), params("stress", 32))
    b = (params("stress", 33), params("random", 34))
    load(env, eng, *a, "load")
    via_load = [read(eng, n) for n in (0, 1)]
    poison(eng)
    load(env, eng, *a, "repack")
    via_repack = [read(eng, n) for n in (0, 1)]
    load(env, eng, *a, "repack")
    again = [read(eng, n) for n in (0, 1)]
    for n in (0, 1):
        for k in via_load[n]:
            if k == "bias_frame":
                continue
            assert np.array_equal(via_load[n][k], via_repack[n][k]), f"load != repack: net {n} {k}"
            assert np.array_equal(via_repack[n][k], again[n][k]), f"repack not idempotent: net {n} {k}"
    load(env, eng, b[0], None, "repack")
    fine = read(eng, 1)
    for k in fine:
        assert np.array_equal(fine[k], via_repack[1][k]), f"repack(fine = NULL) changed network 1's {k}"
    check_net(env, read(eng, 0), b[0], "coarse-only repack net 0")


# ---- (5) training
def _rays(dev, n, seed):
    H = W = 16
    fr = O.synthetic_frame(seed, H, W)
    ro, rd = O.ray_bundle(H, W, fr["intrinsics"], fr["pose"])
    g = torch.Generator().manual_seed(seed)
    sel = torch.randperm(H * W, generator=g)[:n]
    return (ro.reshape(-1, 3)[sel].to(dev), rd.reshape(-1, 3)[sel].to(dev), torch.rand(n, 3, generator=g).to(dev),
            fr["expr"].to(dev), fr["bg"].reshape(-1, 3)[sel].to(dev))


def _trainer(env, seed):
    nerf, _, _, dev, _ = env
    from nerf import fused_train
    ms = []
    for s in (seed, seed + 1):
        m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True,
                                                            include_input_dir=False)
        m.load_state_dict(O.random_init_params(s))
        ms.append(m.to(dev))
    return fused_train.FusedTrainer(ms[0], ms[1], 4, num_coarse=32, num_fine=32)


def _check_trainer(env, tr, label):
    for net, ps in ((0, tr._pc), (1, tr._pf)):
        p = [t.detach().cpu().numpy() for t in ps]
        check_net(env, read(tr.eng, net), p, f"{label} net {net}")


def test_training_keeps_the_image_current(env):
    """(5): eager steps, step_graph replays, step_images_graph replays (K = 2), each followed by the byte check."""
    _, _, _, dev, _ = env
    from nerf import ray_sampler
    from test_train_images_gpu import dataset
    tr = _trainer(env, 40)
    n = 32
    for i in range(3):
        ro, rd, tgt, expr, bg = _rays(dev, n, 50 + i)
        tr.step(ro, rd, tgt, expr, i % 4, background=bg)
        _check_trainer(env, tr, f"eager step {i}")
    tr.capture(n, has_background=True)
    for i in range(3):
        ro, rd, tgt, expr, bg = _rays(dev, n, 60 + i)
        tr.step_graph(ro, rd, tgt, expr, i % 4, background=bg)
        _check_trainer(env, tr, f"graph step {i}")
    data, _, _ = dataset(ray_sampler, dev, 3, 16, 16, [(2, 12, 3, 13)] * 3)
    tr.capture_images(data, 2, n)
    for i in range(3):
        tr.step_images_graph([i % 3, (i + 1) % 3])
        _check_trainer(env, tr, f"images graph step {i}")


def test_two_trainers_alternating(env):
    """(5), the _own_engine case: two trainers' steps interleaved on the device's one renderer; after each step the buffers
    hold that trainer's bucket."""
    _, _, _, dev, _ = env
    t1, t2 = _trainer(env, 70), _trainer(env, 80)
    assert t1.eng is t2.eng
    n = 32
    for i in range(4):
        tr = (t1, t2)[i % 2]
        ro, rd, tgt, expr, bg = _rays(dev, n, 90 + i)
        tr.step(ro, rd, tgt, expr, 1, background=bg)
        _check_trainer(env, tr, f"trainer {i % 2 + 1} step {i // 2}")
