"""The parameter-gradient backward of nfb_render_backward (csrc/nfb_train.cu: composite_bwd_kernel, the FP16 d-raw operand,
chain::chain_kernel, dw::dw_kernel<false> / <true>, grad_reduce_kernel, finalize_kernel and fin_dir0_kernel) against float64,
stage by stage, each stage fed the kernel's own output of the stage before it, read through NfbTrainDebug (d_raw,
ray_bias_sums, records, scale, dw_partials, accumulators), at every (network, part) slot of the weight-gradient launch's
production split, derived from nfb_debug_schedule(4, ...) at the device's SM count.
  (a) compositing    d raw per sample against float64 autograd of the compositing alone (composite_terms64 of
                     test_input_grads_fp64_gpu) at the kernel's saved colours, sigma inputs, depths and |d|: max-abs / max|ref|
                     and relative L2 per pass, DRAW_TOL.  With a background the last sample's d rgb_raw is exactly 0; rows
                     without a sample are exactly 0.  ray_bias_sums [pass][ray] against the float64 sum of the ray's d-raw rows
                     within gamma(S) times the sum of absolute values.
  (b) operand        the loss scale is a power of two with max |d raw| scale in [2^9, 2^11] (exactly 1 when every output
                     gradient is 0), scale[1] = 1 / scale[0]; every record's d-raw image (16 feature rows) is bit for bit
                     fp16(d_raw scale) rounded to nearest without saturation, rows 4-15 are 0.
  (c) dX chain       every live row of every dY_L image (L = 8 ... 0) against float64 of mask_L (x) (W^T dY_{L+1}) from the
                     kernel's own FP16 image of the layer above (the d-raw image for steps 0 and 3), the kernel's own ReLU mask
                     bits and the FP16 weights the chain streams (fp16(fp32(float64 fold)) for M1 = Wd0[:, :256] Wf and
                     m2 = wa Wf).  Bound per element: half an FP16 ulp of the value (2^-24 below the normal range) plus
                     gamma'(K) times sum |w dy|, gamma'(k) = k 2^-23 / (1 - k 2^-23) (wgmma's FP32 accumulation order and
                     rounding are not documented).  Masked elements are exactly +0; rows without a sample are exactly 0.
  (d) dW partials    every slot the launch filled (part p of a network owns its tiles [p per, min(total, (p + 1) per)),
                     per = ceil(total / parts), through global_tile) against float64 over exactly those tiles' decoded record
                     images times scale[1]: every block dw::make_jobs writes (dY0^T PE, dY3^T PE, dY^T h for layers 1-5 and
                     the skip layer's hidden part, dY6^T h5, dY6^T PEd, h5^T draw with all 16 columns, dY7^T g0, dY8^T g1,
                     g2^T draw, the nine bias column sums), or the compact [dW0 | dW3a | db0 | db3] slot after a PE-only
                     launch.  Per element within gamma'(rows of the share) times sum |dY| |X|; per block relative RMS within
                     DW_RMS; the error level uniform over (network, part) and (network, job group) (DW_KAPPA).
  (e) reduction      bit for bit: every accumulator below kAccBRaw (or in the four PE blocks, the rest exactly 0) is
                     ((0 + p_0) + p_1) + ... over the filled slots in part order, and kAccBRaw..+4 is grad_reduce_kernel's
                     order over ray_bias_sums (256 strided sequential sums, then the fixed tree).
  (f) finalize       from the kernel's accumulators and the FP32 parameters: bit for bit every gradient that is a copy (the
                     layer weights and biases, layers_dir.0[:, 256:280], layers_dir.1/2, layers_dir.0.bias, fc_rgb.weight
                     transposed from kAcc9, fc_rgb.bias, fc_alpha.bias) and the conditioning columns of layers_xyz.0 / .3, the
                     FP32 product db fp32(expression / 3 ; latent); fc_feat.weight/bias, fc_alpha.weight and
                     layers_dir.0[:, :256] against the float64 chain rule through the folds within gamma(k) of the sums of
                     absolute values; layers_dir.3.* get no gradient.
Stale state (test_stale_workspace): after a backward with more filled slots, NaN written into every slot it filled, into d raw
and into ray_bias_sums, a smaller case's accumulators and gradients are finite and bit-identical to a fresh handle's, for a
full launch after a PE-only one and the reverse.

Measured on an H100 80GB HBM3 at a 700 W power limit (CUDA 12.9), worst over all cases and both precisions (the two modes
agree to two digits: the backward streams FP16 operands in both):
  (a) d raw max 2.1e-6, L2 3.3e-6 (128c256f)                                     -> DRAW_TOL (2e-5, 1e-5)
      ray_bias_sums 0.04 of gamma(S)
  (b) bit for bit in every case
  (c) 1.00 of the bound: an FP16 rounding tie (a sum the FP32 accumulator holds exactly, half an ulp from both neighbours)
      meets the half-ulp term with equality; the gamma'(K) term never showed, no element exceeded the bound
  (d) 0.092 of gamma'(rows) (single-tile parts; 0.035 at the production batch, where gamma'(205 x 128) is 3.1e-3), so the
      k 2^-23 allowance for the undocumented wgmma accumulation was not needed; relative RMS per block 8.5e-5 (production
      batch), 8.4e-7 with one tile per part                                          -> DW_RMS 3e-4
      class RMS / overall RMS 3.54 (production batch, by job group: the blocks' operands differ, not the schedule; 2.0-3.0
      elsewhere).  This exceeds the render tests' KAPPA of 2.5                       -> DW_KAPPA 5
  (e) bit for bit in every case
  (f) copies and conditioning products bit for bit; the chain rule through the folds 0.18 of gamma(k)
The splits the launch used, read back through dw_parts, equal nfb_debug_schedule(4, ...) in every case: at 132 SMs the
production batch 5 + 11 parts of 205 / 187 tiles (PE-only 22 + 44 of 47), 6 rays 3 + 6 parts of one tile, 36 rays at 64c+0f
16 parts of 2 tiles with 9 filled.  The file takes about 30 s on one H100.
Planted defects, each built once (the fast cases prod2048, prod2048_input_only, single_tile_parts(_input_only), 100c60f and
empty_trailing_parts), with the stage check that caught it:
  grad_reduce_kernel summing one filled slot too few: (e), 357,000-370,000 accumulators differ, every case.
  dw_kernel's share one tile short (j1 - 1): (d), 370 times gamma'(rows) and relative RMS 4.9e-2 at the production batch,
      every element of a slot with one tile per part (the slot is never written).
  the chain epilogue taking the mask bit of the other column parity: (c), masked elements not +0 from dY8 on.
  pack_bwd_chunk putting m2 at k = 2 of step 3's operand atom (it multiplies d rgb_raw.z instead of d sigma): (c), dY5 at
      7,600 times its bound.
  finalize_kernel reading kAcc9 untransposed for fc_rgb.weight: (f), the copy check of fc_rgb.weight.
The existing suite fails for each as well (test_backward_fp64_gpu.py and test_backward_gpu.py: 42 of 66 tests, 29 of 66 for
the short share), by the end-to-end per-tensor bounds; this file names the stage and the element.
"""
import types

import pytest
import torch

from test_backward_gpu import REC, decode_image, dev_tensor, dy_off, x_off
from test_backward_fp64_gpu import E, make_case, out_grads, rowmap, train_forward, two_iter_rays  # noqa: F401
from test_input_grads_fp64_gpu import ACC_FLOATS, bounded, composite_terms64, debug_state, same_bits
from test_input_grads_gpu import params_of
from test_multi_frame_fp64_gpu import gamma
from test_render_fp64_gpu import CLASS_MIN
from test_train_forward_fp64_gpu import mask_bits, masks_of, width

pytestmark = pytest.mark.gpu

PRECS = ["exact", "fast"]
DRAW_TOL = (2e-5, 1e-5)     # d raw per pass: (max-abs / max|ref|, relative L2)
DW_RMS = 3e-4               # weight-gradient partials: |got - ref|_2 / |ref|_2 per block and slot
DW_KAPPA = 5.0              # weight-gradient partials: worst (network, part) or (network, job group) RMS / overall RMS
U23 = 2.0 ** -23

# nfb_layout.h: the accumulators of one network (float offsets)
K0, K1, K2, K3A, K3B, K4, K5 = 0, 16384, 81920, 147456, 163840, 229376, 294912
K6, K6D, KSIG, K7, K8, K9, KB = 360448, 393216, 397312, 401408, 417792, 434176, 436224
KBRAW = KB + 6 * 256 + 3 * 128
PE_SLOT = 2 * 256 * 64 + 2 * 256  # dw::kPeSlotFloats
assert KBRAW + 4 == ACC_FLOATS


def bias_off(layer):
    return KB + (layer * 256 if layer < 6 else 1536 + (layer - 6) * 128)


def gamma23(k):
    return k * U23 / (1.0 - k * U23)


PE, PED, DRAW = (REC["pe"][0], 64), (REC["ped"][0], 32), (REC["draw"], 16)


def H(layer):
    return (x_off(layer), width(layer))


def DY(layer):
    return (dy_off(layer), width(layer))


# Every block dw::make_jobs writes: (name, accumulator offset, A image, B image (None: the bias column sums of A), job group of
# the output rows [0, 128) and [128, 256)).  Block element [n][k] = sum over sample rows of A[r, n] B[r, k].
BLOCKS = [("dW1", K1, DY(1), H(0), (0, 1)), ("dW2", K2, DY(2), H(1), (0, 1)), ("db1", bias_off(1), DY(1), None, (0, 1)),
          ("db2", bias_off(2), DY(2), None, (0, 1)), ("dW4", K4, DY(4), H(3), (2, 3)), ("dW5", K5, DY(5), H(4), (2, 3)),
          ("db4", bias_off(4), DY(4), None, (2, 3)), ("db5", bias_off(5), DY(5), None, (2, 3)),
          ("dW3b", K3B, DY(3), H(2), (4, 5)), ("dW3a", K3A, DY(3), PE, (4, 5)), ("dW0", K0, DY(0), PE, (4, 5)),
          ("db3", bias_off(3), DY(3), None, (4, 5)), ("db0", bias_off(0), DY(0), None, (4, 5)),
          ("dM1", K6, DY(6), H(5), (6,)), ("db6", bias_off(6), DY(6), None, (6,)), ("dWd0_dir", K6D, DY(6), PED, (6,)),
          ("h5^T draw", KSIG, H(5), DRAW, (6, 7)), ("dWd1", K7, DY(7), H(6), (7,)), ("db7", bias_off(7), DY(7), None, (7,)),
          ("dWd2", K8, DY(8), H(7), (7,)), ("db8", bias_off(8), DY(8), None, (7,)), ("g2^T draw", K9, H(8), DRAW, (7,))]
# the PE-only launch's compact slot: [dW0 | dW3a | db0 | db3]
PE_BLOCKS = {"dW0": 0, "dW3a": 16384, "db0": 32768, "db3": 33024}


def pe_slot_to_acc(dev):
    e = torch.arange(PE_SLOT, device=dev)
    return torch.where(e < 16384, K0 + e, torch.where(e < 32768, K3A + e - 16384, torch.where(e < 33024, KB + e - 32768,
                                                                                               bias_off(3) + e - 33024)))


def split(E, n_units, tc, tf, pe_only):
    """The weight-gradient launch's CTA split at this device's SM count (nfb_debug_schedule(4, ...)): parts per network; the
    PE-only launch runs two job groups, so it deals out the CTAs of num_sms * 8 / 2 SMs."""
    import ctypes as C
    sms = E.sms * 4 if pe_only else E.sms
    buf = (C.c_uint32 * 16)(sms, n_units * tc, n_units * tf)
    assert E.capi.lib.nfb_debug_schedule(4, 0, buf, 16) == 3
    return int(buf[0]), int(buf[1])


def shares(c, s, parts):
    """Per network: (global tiles of the network in share order, per, filled parts)."""
    n_units = (c.n + s.R - 1) // s.R
    out = []
    for net, (t_cnt, base) in enumerate(((s.tc, 0), (s.tf, s.tc))):
        total = n_units * t_cnt
        if parts[net] == 0 or total == 0:
            out.append((None, 0, 0))
            continue
        j = torch.arange(total)
        gt = (j // t_cnt) * (s.tc + s.tf) + base + j % t_cnt
        per = -(-total // parts[net])
        out.append((gt, per, -(-total // per)))
    return out


# ---------------------------------------------------------------------------------------------------------------- state
def backward_state(E, c, s, gouts, mode):
    """One backward (mode "full": parameter gradients; "pe": input-only with d latent and d expression, the PE-only launch)
    and what it left in the training state."""
    pc, pf = params_of(c)
    if mode == "full":
        gc, gf, gl = E.eng.backward(list(gouts), pc, pf)
        ing = {}
    else:
        gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=False, inputs=["expression"])
    torch.cuda.synchronize()
    d = E.eng.train_debug()
    npass = 2 if c.nf else 1
    t = types.SimpleNamespace(kg=(gc, gf, gl), ing=ing, dbg=d, mode=mode, n_tiles=s.n_tiles)
    t.recs = dev_tensor(d.records, (s.n_tiles, d.record_bytes // 2), "<i2")
    t.draw = dev_tensor(d.d_raw, (s.n_tiles, 128, 4)).clone()
    sc = dev_tensor(d.scale, (2,)).clone()
    t.scale, t.inv = float(sc[0]), float(sc[1])
    t.acc = [dev_tensor(d.acc_coarse, (ACC_FLOATS,)).clone()] + ([dev_tensor(d.acc_fine, (ACC_FLOATS,)).clone()] if c.nf else [])
    assert d.ray_bias_sums, "ray_bias_sums after a one-launch backward"
    t.bsum = dev_tensor(d.ray_bias_sums, (npass, c.n, 4)).clone()
    t.parts = (int(d.dw_parts[0]), int(d.dw_parts[1]))
    t.stride = int(d.dw_slot_floats)
    assert bool(d.dw_pe_only) == (mode == "pe") and t.stride == (PE_SLOT if mode == "pe" else KBRAW), (mode, t.stride)
    t.ws = dev_tensor(d.dw_partials, (sum(t.parts), t.stride)).clone()
    return t


# ---------------------------------------------------------------------------------------------------------------- (a), (b)
def check_compositing(c, s, t, gouts, tag):
    worst = [0.0, 0.0, 0.0]
    used = torch.zeros(s.n_tiles, 128, dtype=torch.bool, device=t.draw.device)
    for pas in range(2 if c.nf else 1):
        S = c.nc + c.nf if pas else c.nc
        tile, row = rowmap(c, s, pas)
        used[tile, row] = True
        _, _, ref = composite_terms64(c, s, pas, gouts)
        got = t.draw[tile, row].view(c.n, S, 4)
        assert bool(torch.isfinite(got).all()), (tag, pas)
        d = (got.double() - ref).abs()
        rmax = float(ref.abs().max())
        em = float(d.max()) / rmax if rmax > 0 else (0.0 if float(d.max()) == 0 else float("inf"))
        el = float(d.norm() / ref.norm()) if rmax > 0 else em
        worst[0], worst[1] = max(worst[0], em), max(worst[1], el)
        assert em <= DRAW_TOL[0] and el <= DRAW_TOL[1], (tag, pas, "d raw", em, el)
        if c.bg is not None:
            assert float(got[:, -1, :3].abs().max()) == 0.0, (tag, pas, "the background sample's d rgb_raw")
        gd = got.double()
        w, _ = bounded(f"{tag} ray_bias_sums pass {pas}", t.bsum[pas], gd.sum(1), gd.abs().sum(1) * gamma(S), 1.0)
        worst[2] = max(worst[2], w)
    if bool((~used).any()):
        assert float(t.draw[~used].abs().max()) == 0.0, (tag, "d raw of a row without a sample")
    return worst


def check_operand(t, tag):
    m = float(t.draw.abs().max())
    e = torch.log2(torch.tensor(t.scale, dtype=torch.float64))
    assert float(e) == round(float(e)) and t.inv * t.scale == 1.0, (tag, t.scale, t.inv)
    if m == 0.0:
        assert t.scale == 1.0, (tag, t.scale)
    else:
        assert 2.0 ** 9 <= m * t.scale <= 2.0 ** 11, (tag, m, t.scale)
    img = decode_image(t.recs, REC["draw"], 16)
    want = (t.draw * t.scale).half().float()  # round to nearest even, no saturation (inf past 65504), as pack_f16x2_inf
    bad = int((img[..., :4].contiguous().view(torch.int32) != want.view(torch.int32)).sum())
    assert bad == 0, (tag, "d-raw image differs from fp16(d raw * scale)", bad)
    assert int(torch.count_nonzero(img[..., 4:].contiguous().view(torch.int32))) == 0, (tag, "d-raw image rows 4-15")


# ---------------------------------------------------------------------------------------------------------------- (c)
def chain_weights(m):
    """float64 values of the FP16 weights the chain streams, per produced layer L: [K_in, width(L)]."""
    P = {k: v.detach() for k, v in m.named_parameters()}
    h = lambda w: w.float().half().double()  # noqa: E731
    Wf = P["fc_feat.weight"].double()
    fold = lambda left: h((left.double() @ Wf).float())  # noqa: E731  (float64 fold, rounded to FP32, then to FP16)
    return {8: h(P["fc_rgb.weight"]), 7: h(P["layers_dir.2.weight"]), 6: h(P["layers_dir.1.weight"]),
            5: torch.cat((fold(P["layers_dir.0.weight"][:, :256]), fold(P["fc_alpha.weight"]))),
            4: h(P["layers_xyz.5.weight"]), 3: h(P["layers_xyz.4.weight"]), 2: h(P["layers_xyz.3.weight"][:, 171:]),
            1: h(P["layers_xyz.2.weight"]), 0: h(P["layers_xyz.1.weight"])}


def half_ulp16(x):
    """Half an FP16 ulp of |x| (2^-25 below the normal range)."""
    _, ex = torch.frexp(x)
    e = torch.where(x > 0, ex - 1, torch.full_like(ex, -14)).clamp(min=-14)
    return torch.ldexp(torch.ones_like(x), e - 11)


def check_chain(c, s, t, tag, chunk=1 << 16):
    masks = masks_of(t)
    used = torch.zeros(s.n_tiles, 128, dtype=torch.bool, device=t.draw.device)
    for pas in range(2 if c.nf else 1):
        used[rowmap(c, s, pas)] = True
    draw_img = decode_image(t.recs, REC["draw"], 16)
    weights = [chain_weights(m) for m in ([c.mc] + ([c.mf] if c.nf else []))]
    worst = 0.0
    above = None
    for L in range(8, -1, -1):
        img = decode_image(t.recs, dy_off(L), width(L))
        if bool((~used).any()):
            assert float(img[~used].abs().max()) == 0.0, (tag, L, "dY of a row without a sample")
        bits = mask_bits(masks, L)
        for pas in range(2 if c.nf else 1):
            tile, row = rowmap(c, s, pas)
            W = weights[pas][L]
            K = {8: 3, 5: 129}.get(L, W.shape[0])
            for b in range(0, tile.numel(), chunk):
                tl, rw = tile[b:b + chunk], row[b:b + chunk]
                if L == 8:
                    x = draw_img[tl, rw, :3]
                elif L == 5:
                    x = torch.cat((above[tl, rw], draw_img[tl, rw, 3:4]), 1)
                else:
                    x = above[tl, rw]
                x = x.double()
                mk = bits[tl, rw]
                got = img[tl, rw]
                assert int(torch.count_nonzero(got[~mk].contiguous().view(torch.int32))) == 0, (tag, L, "a masked element is not +0")
                ref = (x @ W) * mk
                mag = (x.abs() @ W.abs()) * mk
                bound = (half_ulp16(torch.maximum(ref.abs(), got.double().abs())) + gamma23(K) * mag) * mk
                w, _ = bounded(f"{tag} dY{L} pass {pas}", got, ref, bound, 1.0)
                worst = max(worst, w)
        above = img
    return worst


# ---------------------------------------------------------------------------------------------------------------- (d)
def check_partials(E, c, s, t, tag):
    n_units = (c.n + s.R - 1) // s.R
    want = split(E, n_units, s.tc, s.tf if c.nf else 0, t.mode == "pe")
    assert t.parts == want, (tag, "dw_parts", t.parts, want)
    sh = shares(c, s, t.parts)
    blocks = [b for b in BLOCKS if t.mode == "full" or b[0] in PE_BLOCKS]
    worst, rms = 0.0, 0.0
    errs, cls_part, cls_group = [], [], []
    for name, off, A, B, groups in blocks:
        nA = A[1]
        a_img = decode_image(t.recs, *A)
        b_img = decode_image(t.recs, *B) if B is not None else None
        nB = B[1] if B is not None else 1
        slot_off = PE_BLOCKS[name] if t.mode == "pe" else off
        for net, (gt, per, filled) in enumerate(sh):
            if gt is None:
                continue
            first = 0 if net == 0 else t.parts[0]
            for p in range(filled):
                tiles = gt[p * per:(p + 1) * per].to(a_img.device)
                a = a_img[tiles].reshape(-1, nA).double()
                b = b_img[tiles].reshape(-1, nB).double() if b_img is not None else torch.ones(a.shape[0], 1, dtype=torch.float64,
                                                                                                device=a.device)
                ref = (a.t() @ b) * t.inv
                mag = (a.abs().t() @ b.abs()) * t.inv
                got = t.ws[first + p, slot_off:slot_off + nA * nB].view(nA, nB)
                tg = f"{tag} {name} net {net} part {p}/{filled}"
                w, r = bounded(tg, got, ref, mag * gamma23(a.shape[0]), 1.0)
                worst = max(worst, w)
                rn = float(ref.norm())
                e2 = float((got.double() - ref).norm())
                if rn > 0:
                    rms = max(rms, e2 / rn)
                    assert e2 <= DW_RMS * rn, (tg, "relative RMS", e2 / rn)
                ok = mag > 0
                rel = ((got.double() - ref).abs() / mag.clamp(min=1e-300)).pow(2)
                grp = torch.tensor(groups, device=a.device).repeat_interleave(nA // len(groups)).view(nA, 1).expand(nA, nB)
                errs.append(rel[ok])
                cls_part.append(torch.full_like(grp[ok], net * 1024 + p))
                cls_group.append(net * 16 + grp[ok])
    errs = torch.cat(errs)
    kappa = max(uniformity(f"{tag} dW partials by part", errs, torch.cat(cls_part)),
                uniformity(f"{tag} dW partials by job group", errs, torch.cat(cls_group)))
    return worst, rms, kappa, sh


def uniformity(tag, errs, classes):
    """test_render_fp64_gpu.check_uniformity at DW_KAPPA: the blocks' error levels differ by their operands' statistics, so the
    job groups spread wider than the render kernel's schedule classes."""
    if errs.numel() == 0 or float(errs.mean()) == 0.0:
        return 0.0
    cnt = torch.bincount(classes)
    se = torch.bincount(classes, weights=errs.double())
    ok = cnt >= CLASS_MIN
    if int(ok.sum()) < 2:
        return 0.0
    worst = float(((se[ok] / cnt[ok]).sqrt() / errs.double().mean().sqrt()).max())
    assert worst <= DW_KAPPA, (tag, worst)
    return worst


# ---------------------------------------------------------------------------------------------------------------- (e)
def check_reduce(c, t, sh, tag):
    for net, (gt, per, filled) in enumerate(sh):
        if gt is None:
            continue
        first = 0 if net == 0 else t.parts[0]
        emu = torch.zeros(t.stride, device=t.ws.device)
        for k in range(filled):
            emu = emu + t.ws[first + k]
        acc = t.acc[net]
        if t.mode == "pe":
            pos = pe_slot_to_acc(acc.device)
            assert same_bits(acc[pos], emu), (tag, net, "PE blocks differ from the fixed-order sum of the slots")
            rest = torch.ones(KBRAW, dtype=torch.bool, device=acc.device)
            rest[pos] = False
            assert int(torch.count_nonzero(acc[:KBRAW][rest].view(torch.int32))) == 0, (tag, net, "an accumulator outside the PE blocks")
        else:
            bad = int((acc[:KBRAW].view(torch.int32) != emu.view(torch.int32)).sum())
            assert bad == 0, (tag, net, "accumulators differ from the fixed-order sum of the slots", bad)
    for pas in range(2 if c.nf else 1):
        b = t.bsum[pas]
        m = -(-c.n // 256)
        pad = torch.zeros(m * 256, 4, device=b.device)
        pad[:c.n] = b
        s = torch.zeros(256, 4, device=b.device)
        for k in range(m):  # thread i sums rays i, i + 256, ... in order
            s = s + pad[k * 256:(k + 1) * 256]
        h = 128
        while h > 0:
            s = torch.cat((s[:h] + s[h:2 * h], s[h:]))
            h //= 2
        want = torch.zeros(4, device=b.device) + s[0]
        assert same_bits(t.acc[pas][KBRAW:KBRAW + 4], want), (tag, pas, "d b_rgb / d b_sigma differ from grad_reduce_kernel's order")


# ---------------------------------------------------------------------------------------------------------------- (f)
def check_finalize(c, t, tag):
    cond = torch.cat(((c.expr.double() / 3.0).float(), c.latent.float()))
    worst = 0.0
    for net, m in enumerate([c.mc] + ([c.mf] if c.nf else [])):
        g = t.kg[net]
        a = t.acc[net]
        P = [v.detach() for v in params_of(c)[net]]
        blk = lambda off, r, k: a[off:off + r * k].view(r, k)  # noqa: E731
        db = {L: a[bias_off(L):bias_off(L) + (256 if L < 6 else 128)] for L in range(9)}
        w0 = torch.cat((blk(K0, 256, 64)[:, :63], db[0][:, None] * cond[None, :]), 1)
        w3 = torch.cat((blk(K3A, 256, 64)[:, :63], db[3][:, None] * cond[None, :], blk(K3B, 256, 256)), 1)
        copies = {0: w0, 1: db[0], 2: blk(K1, 256, 256), 3: db[1], 4: blk(K2, 256, 256), 5: db[2], 6: w3, 7: db[3],
                  8: blk(K4, 256, 256), 9: db[4], 10: blk(K5, 256, 256), 11: db[5], 15: a[KBRAW + 3:KBRAW + 4], 17: db[6],
                  18: blk(K7, 128, 128), 19: db[7], 20: blk(K8, 128, 128), 21: db[8], 24: blk(K9, 128, 16)[:, :3].t(),
                  25: a[KBRAW:KBRAW + 3]}
        for i, want in copies.items():
            assert same_bits(g[i], want.reshape(g[i].shape)), (tag, net, i, "finalize copy / product")
        assert same_bits(g[16][:, 256:], blk(K6D, 128, 32)[:, :24]), (tag, net, "layers_dir.0[:, 256:280]")
        assert g[22] is None and g[23] is None
        ad = a.double()
        dM1, dm2, db6, dbs = ad[K6:K6 + 32768].view(128, 256), ad[KSIG:KSIG + 4096].view(256, 16)[:, 3], db[6].double(), ad[KBRAW + 3]
        Wd0, Wf, bf, wa = P[16].double()[:, :256], P[12].double(), P[13].double(), P[14].double()[0]
        checks = [
            ("fc_feat.weight", g[12], Wd0.t() @ dM1 + wa[:, None] * dm2[None, :], Wd0.abs().t() @ dM1.abs() + (wa.abs()[:, None] * dm2.abs()[None, :]), 129),
            ("fc_feat.bias", g[13], Wd0.t() @ db6 + wa * dbs, Wd0.abs().t() @ db6.abs() + wa.abs() * dbs.abs(), 129),
            ("fc_alpha.weight", g[14][0], Wf @ dm2 + dbs * bf, Wf.abs() @ dm2.abs() + dbs.abs() * bf.abs(), 257),
            ("layers_dir.0[:, :256]", g[16][:, :256], dM1 @ Wf.t() + db6[:, None] * bf[None, :],
             dM1.abs() @ Wf.abs().t() + db6.abs()[:, None] * bf.abs()[None, :], 257)]
        for name, got, ref, mag, k in checks:
            w, _ = bounded(f"{tag} net {net} {name}", got, ref, mag * gamma(k), 1.0)
            worst = max(worst, w)
    return worst


# ---------------------------------------------------------------------------------------------------------------- cases
def run_stages(E, c, tag, mode="full", gouts=None, expect=None):
    train_forward(E, c)
    s = debug_state(E, c)
    gouts = out_grads(E, c) if gouts is None else gouts
    t = backward_state(E, c, s, gouts, mode)
    comp = check_compositing(c, s, t, gouts, tag)
    check_operand(t, tag)
    ch = check_chain(c, s, t, tag)
    dw, rms, kappa, sh = check_partials(E, c, s, t, tag)
    if expect:
        expect(t, sh)
    check_reduce(c, t, sh, tag)
    fin = check_finalize(c, t, tag) if mode == "full" else 0.0
    split_s = ", ".join(f"{t.parts[n]} parts, {sh[n][1]} tiles each, {sh[n][2]} filled" for n in range(2) if sh[n][0] is not None)
    print(f"{tag}: {split_s}; d raw max {comp[0]:.1e} L2 {comp[1]:.1e}, ray bias sums {comp[2]:.2f} of gamma(S); "
          f"chain {ch:.2f} of its bound; partials {dw:.2e} of gamma'(rows), RMS {rms:.1e}, class RMS / overall {kappa:.2f}; "
          f"finalize {fin:.2e} of gamma(k)")


def single_tile(t, sh):
    assert all(per == 1 and filled == parts for (gt, per, filled), parts in zip(sh, t.parts) if gt is not None), (t.parts, sh)


def empty_trailing(t, sh):
    assert sh[1][0] is None and sh[0][2] < t.parts[0] and sh[0][1] >= 2, (t.parts, sh)


CASES = {
    # 2048 rays at 64c+64f: 1024 units, 3072 tiles (5 + 11 parts of 205 / 187 tiles on 132 SMs; PE-only 22 + 44)
    "prod2048": (lambda E, p: make_case(E, 2048, 64, 64, p, stress=False, seed=50), "full", None),
    "prod2048_input_only": (lambda E, p: make_case(E, 2048, 64, 64, p, stress=False, seed=50), "pe", None),
    # 4 * SMs + 37 rays: every chain CTA runs two or more units
    "64c64f": (lambda E, p: make_case(E, two_iter_rays(E), 64, 64, p, seed=128), "full", None),
    # 6 rays at 64c+64f: 3 + 6 tiles, one tile per part (a dropped or doubled tile is a 100 % error)
    "single_tile_parts": (lambda E, p: make_case(E, 6, 64, 64, p, seed=6), "full", single_tile),
    "single_tile_parts_input_only": (lambda E, p: make_case(E, 6, 64, 64, p, seed=6), "pe", single_tile),
    # 36 rays at 64c+0f: 18 tiles over the parts of one network, per = 2, the trailing parts get none
    "empty_trailing_parts": (lambda E, p: make_case(E, 36, 64, 0, p, seed=36), "full", empty_trailing),
    # one ray per unit
    "128c256f": (lambda E, p: make_case(E, 2 * E.sms + 5, 128, 256, p, seed=384), "full", None),
    # partly filled last tiles of both passes (200 and 320 rows per unit)
    "100c60f": (lambda E, p: make_case(E, two_iter_rays(E), 100, 60, p, seed=160), "full", None),
    "white_nobg": (lambda E, p: make_case(E, 300, 64, 64, p, seed=3, white=True, bg=False), "full", None),
    "nobg": (lambda E, p: make_case(E, 300, 64, 64, p, seed=3, bg=False), "full", None),
    "dir_z": (lambda E, p: make_case(E, 300, 64, 64, p, seed=7, dir_z=True), "full", None),
    "deterministic": (lambda E, p: make_case(E, 300, 64, 64, p, seed=7, perturb=False, noise_std=0.0), "full", None),
}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", list(CASES))
def test_param_backward_stages_against_float64(E, case, prec):
    build, mode, expect = CASES[case]
    run_stages(E, build(E, prec), f"{case} {prec}", mode=mode, expect=expect)


@pytest.mark.parametrize("prec", PRECS)
def test_zero_output_gradients(E, prec):
    """All-zero output gradients: the loss scale is exactly 1 and every stage is exactly 0."""
    c = make_case(E, 300, 64, 64, prec, seed=11)
    gouts = [None if g is None else torch.zeros_like(g) for g in out_grads(E, c)]
    run_stages(E, c, f"zero {prec}", gouts=gouts)


def test_debug_hook_fields(E):
    """dw_partials / dw_slot_floats / dw_parts / dw_pe_only / ray_bias_sums are NULL / 0 after a training forward, describe the
    last launch after a backward, and stay NULL / 0 (ray_bias_sums set) after an input-only backward with no weight-gradient
    launch."""
    c = make_case(E, 300, 64, 64, "fast", seed=5)
    n_units = (c.n + 1) // 2
    gouts = out_grads(E, c)
    pc, pf = params_of(c)

    def fields():
        torch.cuda.synchronize()
        d = E.eng.train_debug()
        return bool(d.dw_partials), int(d.dw_slot_floats), (int(d.dw_parts[0]), int(d.dw_parts[1])), int(d.dw_pe_only), bool(d.ray_bias_sums)
    train_forward(E, c)
    assert fields() == (False, 0, (0, 0), 0, False)
    E.eng.backward(list(gouts), pc, pf)
    assert fields() == (True, KBRAW, split(E, n_units, 1, 2, False), 0, True)
    E.eng.backward(list(gouts), pc, pf, want_latent=False, want_params=False, inputs=["ray_origins"])
    assert fields() == (False, 0, (0, 0), 0, True)
    E.eng.backward(list(gouts), pc, pf, want_params=False, inputs=["expression"])
    assert fields() == (True, PE_SLOT, split(E, n_units, 1, 2, True), 1, True)
    train_forward(E, c)
    assert fields() == (False, 0, (0, 0), 0, False)


# ---------------------------------------------------------------------------------------------------------------- stale state
def results(env, c, gouts, mode):
    train_forward(env, c)
    pc, pf = params_of(c)
    if mode == "full":
        gc, gf, gl = env.eng.backward(list(gouts), pc, pf)
        out = [g for g in gc + gf if g is not None] + [gl]
    else:
        _, _, gl, ing = env.eng.backward(list(gouts), pc, pf, want_params=False, inputs=["expression"])
        out = [gl, ing["expression"]]
    torch.cuda.synchronize()
    d = env.eng.train_debug()
    out += [dev_tensor(d.acc_coarse, (ACC_FLOATS,)).clone(), dev_tensor(d.acc_fine, (ACC_FLOATS,)).clone()]
    return out


def poison(env, c):
    """NaN into every weight-gradient slot the last backward filled, into d raw and into the per-ray bias sums (plain stores
    through the pointers the debug hook hands out)."""
    torch.cuda.synchronize()
    d = env.eng.train_debug()
    dev_tensor(d.dw_partials, ((d.dw_parts[0] + d.dw_parts[1]) * d.dw_slot_floats,)).fill_(float("nan"))
    dev_tensor(d.d_raw, (int(d.n_tiles) * 512,)).fill_(float("nan"))
    dev_tensor(d.ray_bias_sums, ((2 if c.nf else 1) * c.n * 4,)).fill_(float("nan"))
    torch.cuda.synchronize()


@pytest.mark.parametrize("prec", PRECS)
def test_stale_workspace(E, prec):
    """A backward with more filled slots (2 * SMs + 37 rays), NaN into what it left, then a 6-ray backward (one tile per part)
    on the same handle: every accumulator and gradient is finite and bit-identical to the 6-ray case on a fresh handle.  The
    transitions full -> PE-only, PE-only -> full and full -> full."""
    from nerf import _engine
    big = make_case(E, two_iter_rays(E), 64, 64, prec, seed=40)
    small = make_case(E, 6, 64, 64, prec, seed=41)
    gb, gs = out_grads(E, big, seed=42), out_grads(E, small, seed=43)
    fresh = types.SimpleNamespace(**vars(E))
    fresh.eng = _engine.Renderer(E.dev)
    for big_mode, small_mode in (("full", "pe"), ("pe", "full"), ("full", "full")):
        results(E, big, gb, big_mode)
        poison(E, big)
        got = results(E, small, gs, small_mode)
        want = results(fresh, small, gs, small_mode)
        for i, (a, b) in enumerate(zip(got, want)):
            assert bool(torch.isfinite(a).all()), (prec, big_mode, small_mode, i, "non-finite after a poisoned workspace")
            assert same_bits(a, b), (prec, big_mode, small_mode, i, "differs from a fresh handle")
