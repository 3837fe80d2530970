"""The exact-grad backward of nfb_render_backward (NFB_PREC_EXACT_GRAD, DESIGN.md §6c: chain::chain_x3_kernel,
dw::dw_x3_kernel<false> / <true>, grad_reduce_kernel, finalize_kernel, ing::row_x3_kernel, raysum_x3_kernel, framesum_kernel)
against float64, stage by stage, each stage fed the kernel's own hi + lo output of the stage before it, read through
NfbTrainDebug (records of 2 MiB: the hi image at offset o, the lo image at o + 1 MiB; d_raw, scale, dw_partials, dw_parts,
rows, ray_sums, frame_sums, accumulators) and the streamed weights (NfbWeightDebug bwd / bwd_lo, decoded through
tests/weight_pack_reference.Layout).  test_exact_grad_gpu.py checks this mode end to end and at the kernel's forward state in
bulk; this file checks every stage, half and slot on its own.
  (a) operand        the loss scale as in exact mode; the hi d-raw image bit for bit fp16_rn(d raw scale), the lo image bit
                     for bit fp16_rn(d raw scale - float(hi)) (the subtraction is exact in FP32); rows 4-15 and rows without a
                     sample 0 in both halves.  (The compositing backward is exact mode's and is checked as there.)
  (b) dX chain       every live row of dY_L (L = 8 ... 0), hi + lo, against float64 of what chain_body<true> forms from the
                     kernel's own hi + lo image of the layer above (the d-raw image for steps 0 and 3), its mask bits and the
                     streamed hi / lo weights: sum Wh Yh + Wh Yl + Wl Yh, masked (the lo.lo term is left out on purpose; its
                     size, the distance to the full product, is printed).  Masked elements are +0 in both halves; every pair
                     is canonical: |lo| <= half the gap from hi towards lo, and fp16_rn(hi + lo) == hi except where lo's own
                     rounding lands on that half gap (a tie of hi + lo; counted and printed).  Bound per element: the
                     representation, half an FP16 ulp of lo (2^-25 where lo is subnormal, |value| below ~2^-3, so there
                     hi + lo keeps fewer than 22 bits), plus gamma'(3K) sum |terms|, gamma'(k) = k 2^-23 / (1 - k 2^-23).
                     Per layer relative RMS within CHAIN_X3_RMS (a dropped lo stage, ~2^-12 relative per term, stays inside
                     the element bound; the RMS bound is what sees it); the error uniform over column half x warpgroup
                     (KAPPA of test_render_fp64_gpu).
  (c) dW partials    every slot dw_x3_kernel filled (full launch, or the PE-only compact slot), over exactly that slot's tiles
                     of the decoded hi + lo images: (sum Ah Bh + Ah Bl + Al Bh) scale[1], bias column sums sum (Ah + Al)
                     scale[1].  Per element within gamma'(3 rows) sum |.| (bias: gamma'(2 rows)); per block and slot the RMS
                     error within DW_X3_RMS of that bound's RMS; uniform by (network, part) and by (network, job group) within
                     DW_KAPPA.
                     dw_parts == nfb_debug_schedule(4, ...).
  (d) reduction,     bit for bit, test_param_backward_fp64_gpu.check_reduce / check_finalize.
      finalize
  (e) input rows     row_x3_kernel through test_input_grads_fp64_gpu.check_rows (ROW_TOL, KAPPA) fed the kernel's own decoded
                     hi + lo dY0, dY3, dY6; the per-ray sums and the conditioning gradients as there.
  (f) multi-frame    ray_sums bit for bit the ascending FP32 sum over samples of float(hi) + float(lo) (exact) times scale[1];
                     frame_sums and the conditioning gradients as stages (c)-(e) of test_multi_frame_fp64_gpu.py (F = 5 and
                     F = 217).
Cases: the CASES table of test_param_backward_fp64_gpu.py at exact_grad; all-zero output gradients (scale 1, every stage exactly
0 in both halves); the lo floor (per-ray output gradients spread over 1e-6 ... 1: the share of elements whose lo is subnormal and
the error there, hi + lo against hi alone, per layer); the stale workspace; a dY past 65504 (hi = inf and lo non-finite in the
record images, not only in the final gradients).

Measured on an H100 80GB HBM3 at a 700 W power limit (CUDA 12.9), worst over all cases:
  (a) bit for bit in every case
  (b) 1.00 of the element bound (the representation term met with equality); relative RMS per layer 1.6e-6 (prod2048;
      1.0e-6 elsewhere)                                                              -> CHAIN_X3_RMS 1e-5 (6x)
      the lo.lo term left out moves the result by 4.7e-8 relative RMS; class RMS / overall 1.25 (KAPPA 2.5)
      ties of hi + lo: 614 (36 rays) to 7.7 million (prod2048): a pair whose lo rounded onto half an FP16 gap is a tie, and
      about half of those round hi + lo to hi's other neighbour, so "fp16_rn(hi + lo) == hi" holds only away from them
  (c) 0.072 of gamma'(3 rows) (one tile per part; 0.021 at the production batch); RMS per block and slot 0.041 of the
      bound's RMS (one tile per part; 0.011 at the production batch)                 -> DW_X3_RMS 0.15 (3.7x)
      Relative to the sums of absolute values that RMS grows in proportion to the rows of the share (1.9e-6 at 128 rows,
      9.3e-5 at 24,000): the FP32 accumulation, the same size as exact mode's FP16 partials (8.5e-5).  So a defect confined
      to the lo terms (~2^-12 of each term, ~2^-12 / sqrt(rows) of the sum) shows only where a part holds one or two tiles.
      class RMS / overall 2.99 by job group at the production batch                  (DW_KAPPA 5)
  (d) bit for bit in every case; finalize 0.17 of gamma(k)
  (e) rows 1.2e-7 of the absolute sum (ROW_TOL 5e-7), class RMS / overall 1.37; rays 1.2e-7, conditioning 1.1e-7
  (f) ray sums bit for bit, 0.13 of gamma(S); frame sums bit for bit, 1.0 of their bound at F = 217 (one rounding of a
      two-ray frame); latent / expression 5.7e-3, columns 0.51
  lo floor: 64-83 % of the live dY elements per layer lie below 2^-3 (lo subnormal); there the error of hi + lo is 3.6e-3
      (dY8) to 7.3e-2 (dY4) of the error of hi alone: hi + lo keeps a 14x to 280x advantage there
  overflow: dY0 scaled to about 4 x 65504 gives 4,550 inf hi, every lo beside them non-finite
The file takes about 30 s on one H100.

Planted defects, each built once into a library of its own and run against this file and the existing exact-grad tests
(test_exact_grad_gpu.py and test_exact_grad_train_gpu.py, 25 tests):
  1. the bias stages skip A lo (part == 0 for part != 1): (c), the bias column sums (db1, db3) at 8.5-9.7 times gamma'(2 rows)
     with one tile per part, 5.9 times with two; the larger shares pass (see (c)).  The existing tests all pass: missed.
  2. the (A hi, B lo) stage streams B hi on the last tile of each share: (c), dW1 / dW3a at 23 (production batch) to 21,800
     (one tile per part) times the element bound, every case.  Existing: 10 of 25 fail.
  3. the lo of the d-raw operand's z and sigma lanes (l23) left 0: (a), 1,736 to 531,000 lo d-raw entries differ, every case.
     Existing: 3 of 25 fail, only the checks at the kernel's forward state.
  4. the epilogue writes lo for column half 0 only: (b), dY5 (the first 256-wide layer) at 10.2-10.5 times the element
     bound, every case; (f) the ray sums.  Existing: 14 of 25 fail.
  5. the fine network's chain reads the coarse network's wstream_lo: (b), dY8 of the fine pass at 725-3,650 times the
     bound, every two-pass case.  Existing: 9 of 25 fail.
  6. raysum_x3 reads hi only for pass 1: (f), ray_sums of pass 1 bit for bit, ~270,000 entries at F = 5 and F = 217.
     Existing: 1 of 25 fails (the multi-frame check at the kernel's forward state).
"""
import pytest
import torch

import test_param_backward_fp64_gpu as PB
import weight_pack_reference as WP
from test_backward_fp64_gpu import make_case, out_grads, rowmap, train_forward, two_iter_rays
from test_backward_gpu import REC, decode_image, dev_tensor, dy_off
from test_exact_grad_gpu import E, MIB  # noqa: F401  (a renderer handle of its own: exact-grad re-packs the lo stream too)
from test_input_grads_fp64_gpu import bounded, check_cond, check_rays, check_rows, debug_state
from test_input_grads_fp64_gpu import backward_state as input_backward_state
from test_input_grads_gpu import params_of, wanted
from test_multi_frame_fp64_gpu import (check_cond_columns, check_cond_grads, check_framesums, check_raysums, frame_state,
                                       layout, sums_state)
from test_multi_frame_gpu import frames, render
from test_render_fp64_gpu import check_uniformity
from test_train_forward_fp64_gpu import mask_bits, masks_of, width

pytestmark = pytest.mark.gpu

PREC = "exact_grad"
CHAIN_X3_RMS = 1e-5      # dX chain: |got - ref|_2 / |ref|_2 per layer (both passes)
DW_X3_RMS = 0.15         # weight-gradient partials: |got - ref|_2 / (gamma'(3 rows) |sum of absolute values|_2) per block and slot
FLOOR = 2.0 ** -3        # below this magnitude the lo half of an FP16 pair is subnormal


# ---------------------------------------------------------------------------------------------------------------- operands
def hl(recs, off, rows):
    """The decoded hi and lo images of one record image: FP32 [tiles, 128, rows] each."""
    return decode_image(recs, off, rows), decode_image(recs, MIB + off, rows)


def stream_weights(E, net, lay):
    """float64 (hi, lo) of the transposed weights chain_x3_kernel streams for network `net`, per produced layer L: [K_in, width(L)]
    (L = 5: the 128 rows of M1^T, then m2 at row 128), decoded from NfbWeightDebug.bwd / .bwd_lo through the packing layout."""
    w = E.eng.weights_debug(net)
    assert w.bwd_lo and w.bwd_lo_bytes == w.bwd_bytes
    out = []
    for ptr in (w.bwd, w.bwd_lo):
        buf = dev_tensor(ptr, (w.bwd_bytes // 2,), "<i2")
        steps = {}
        for s, u, rows, off in lay.bwd_units:
            pos = torch.from_numpy(WP.unit_positions(rows, off) // 2).to(buf.device)
            steps.setdefault(s, []).append(buf[pos.reshape(-1)].view(rows, 64))
        W = {}
        for s, units in steps.items():
            M = torch.cat(units, 1).view(torch.float16).double()  # [rows, K]: element (n, k) = W[k][n]
            L = 8 - s
            if s == 0:
                m = M[:, :3].t()
            elif s == 3:
                m = torch.cat((M[:, 64:192].t(), M[:, 3:4].t()))
            else:
                m = M.t()
            W[L] = m[:, :width(L)].contiguous()
        out.append(W)
    return out


def check_operand_x3(t, tag):
    PB.check_operand(t, tag)  # the scale, the hi image and its rows 4-15
    v = t.draw * t.scale
    hi = v.half().float()
    want = (v - hi).half().float()  # v - hi is exact in FP32
    img = decode_image(t.recs, MIB + REC["draw"], 16)
    bad = int((img[..., :4].contiguous().view(torch.int32) != want.view(torch.int32)).sum())
    assert bad == 0, (tag, "lo d-raw image differs from fp16(d raw * scale - hi)", bad)
    assert int(torch.count_nonzero(img[..., 4:].contiguous().view(torch.int32))) == 0, (tag, "lo d-raw image rows 4-15")


def half_gap16(hi, lo):
    """Half the distance from hi to its FP16 neighbour in lo's direction (2^-25 at the subnormal spacing)."""
    a = hi.abs()
    h = PB.half_ulp16(a)
    _, ex = torch.frexp(a)
    pow2 = (a == torch.ldexp(torch.ones_like(a), ex - 1)) & (a >= 2.0 ** -14)
    toward_zero = (torch.sign(lo) * torch.sign(hi)) < 0
    return torch.where(pow2 & toward_zero, h / 2, h)


# ---------------------------------------------------------------------------------------------------------------- (b)
def check_chain_x3(E, c, s, t, tag, floor=None, chunk=1 << 16):
    masks = masks_of(t)
    used = torch.zeros(s.n_tiles, 128, dtype=torch.bool, device=t.draw.device)
    for pas in range(2 if c.nf else 1):
        used[rowmap(c, s, pas)] = True
    dr_h, dr_l = hl(t.recs, REC["draw"], 16)
    lay = WP.Layout(E.capi.lib)
    weights = [stream_weights(E, net, lay) for net in range(2 if c.nf else 1)]
    worst, rms_worst, lolo, ties, kappa = 0.0, 0.0, 0.0, 0, 0.0
    above = None
    for L in range(8, -1, -1):
        img_h, img_l = hl(t.recs, dy_off(L), width(L))
        if bool((~used).any()):
            for img in (img_h, img_l):
                assert int(torch.count_nonzero(img[~used].view(torch.int32))) == 0, (tag, L, "dY of a row without a sample")
        bits = mask_bits(masks, L)
        e2, r2, f2 = 0.0, 0.0, 0.0
        errs, cls = [], []
        fl = [0, 0, 0.0, 0.0]  # floor elements, live elements, squared error of hi + lo and of hi alone there
        for pas in range(2 if c.nf else 1):
            tile, row = rowmap(c, s, pas)
            Wh, Wl = weights[pas][0][L], weights[pas][1][L]
            K = {8: 3, 5: 129}.get(L, Wh.shape[0])
            aWh, aWl = Wh.abs(), Wl.abs()
            for b in range(0, tile.numel(), chunk):
                tl, rw = tile[b:b + chunk], row[b:b + chunk]
                if L == 8:
                    xh, xl = dr_h[tl, rw, :3], dr_l[tl, rw, :3]
                elif L == 5:
                    xh = torch.cat((above[0][tl, rw], dr_h[tl, rw, 3:4]), 1)
                    xl = torch.cat((above[1][tl, rw], dr_l[tl, rw, 3:4]), 1)
                else:
                    xh, xl = above[0][tl, rw], above[1][tl, rw]
                xh, xl = xh.double(), xl.double()
                mk = bits[tl, rw]
                gh, gl = img_h[tl, rw], img_l[tl, rw]
                for g in (gh, gl):
                    assert int(torch.count_nonzero(g[~mk].contiguous().view(torch.int32))) == 0, (tag, L, "a masked element is not +0")
                # canonical pairs: |lo| within half the gap of hi, and hi + lo (exact in FP32) rounds back to hi but at a tie
                gap = half_gap16(gh.double(), gl.double())
                assert bool((gl.double().abs() <= gap).all()), (tag, L, "|lo| beyond half an FP16 gap of hi")
                tie = gl.double().abs() == gap
                back = (gh + gl).half().float()
                assert bool(((back == gh) | tie).all()), (tag, L, "fp16_rn(hi + lo) != hi")
                ties += int((tie & (gl != 0)).sum())
                ref = (xh @ Wh + xl @ Wh + xh @ Wl) * mk
                full = ((xh + xl) @ (Wh + Wl)) * mk
                mag = ((xh.abs() + xl.abs()) @ aWh + xh.abs() @ aWl) * mk
                got = gh.double() + gl.double()
                bound = (PB.half_ulp16(gl.double().abs()) + PB.gamma23(3 * K) * mag) * mk
                w, r = bounded(f"{tag} dY{L} pass {pas}", got, ref, bound, 1.0)
                worst = max(worst, w)
                e2 += float((got - ref).pow(2).sum())
                r2 += float(ref.pow(2).sum())
                f2 += float((full - ref).pow(2).sum())
                col = torch.arange(width(L), device=mk.device).view(1, -1).expand_as(mk)
                errs.append(r[mk].pow(2))
                cls.append(((col >= 128).long() * 2 + (rw.view(-1, 1) >= 64).long().expand_as(mk))[mk])
                if floor is not None:
                    live = mk & (got != 0)
                    low = live & (got.abs() < FLOOR)
                    fl[0] += int(low.sum())
                    fl[1] += int(live.sum())
                    fl[2] += float((got - ref)[low].pow(2).sum())
                    fl[3] += float((gh.double() - ref)[low].pow(2).sum())
        if r2 > 0:
            rms = (e2 / r2) ** 0.5
            rms_worst = max(rms_worst, rms)
            lolo = max(lolo, (f2 / r2) ** 0.5)
        if errs:
            kappa = max(kappa, check_uniformity(f"{tag} dY{L} by column half x warpgroup", torch.cat(errs), torch.cat(cls)))
        if floor is not None and fl[1]:
            gain = (fl[2] / fl[3]) ** 0.5 if fl[3] > 0 else 0.0
            floor.append((L, fl[0] / fl[1], gain))
        above = (img_h, img_l)
    return worst, rms_worst, lolo, ties, kappa


# ---------------------------------------------------------------------------------------------------------------- (c)
def check_partials_x3(E, c, s, t, tag):
    n_units = (c.n + s.R - 1) // s.R
    want = PB.split(E, n_units, s.tc, s.tf if c.nf else 0, t.mode == "pe")
    assert t.parts == want, (tag, "dw_parts", t.parts, want)
    sh = PB.shares(c, s, t.parts)
    blocks = [b for b in PB.BLOCKS if t.mode == "full" or b[0] in PB.PE_BLOCKS]
    worst, rms = 0.0, (0.0, "")
    errs, cls_part, cls_group = [], [], []
    for name, off, A, B, groups in blocks:
        nA = A[1]
        ah, al = hl(t.recs, *A)
        bh, bl = hl(t.recs, *B) if B is not None else (None, None)
        nB = B[1] if B is not None else 1
        slot_off = PB.PE_BLOCKS[name] if t.mode == "pe" else off
        for net, (gt, per, filled) in enumerate(sh):
            if gt is None:
                continue
            first = 0 if net == 0 else t.parts[0]
            for p in range(filled):
                tiles = gt[p * per:(p + 1) * per].to(ah.device)
                a_h, a_l = ah[tiles].reshape(-1, nA).double(), al[tiles].reshape(-1, nA).double()
                rows = a_h.shape[0]
                if bh is not None:
                    b_h, b_l = bh[tiles].reshape(-1, nB).double(), bl[tiles].reshape(-1, nB).double()
                    ref = (a_h.t() @ (b_h + b_l) + a_l.t() @ b_h) * t.inv
                    mag = (a_h.abs().t() @ (b_h.abs() + b_l.abs()) + a_l.abs().t() @ b_h.abs()) * t.inv
                    g = PB.gamma23(3 * rows)
                else:
                    ref = (a_h + a_l).sum(0).view(nA, 1) * t.inv
                    mag = (a_h.abs() + a_l.abs()).sum(0).view(nA, 1) * t.inv
                    g = PB.gamma23(2 * rows)
                got = t.ws[first + p, slot_off:slot_off + nA * nB].view(nA, nB)
                tg = f"{tag} {name} net {net} part {p}/{filled}"
                w, _ = bounded(tg, got, ref, mag * g, 1.0)
                worst = max(worst, w)
                mn = float(mag.norm()) * g
                if mn > 0:
                    rms = max(rms, (float((got.double() - ref).norm()) / mn, tg))
                ok = mag > 0
                rel = ((got.double() - ref).abs() / mag.clamp(min=1e-300)).pow(2)
                grp = torch.tensor(groups, device=ah.device).repeat_interleave(nA // len(groups)).view(nA, 1).expand(nA, nB)
                errs.append(rel[ok])
                cls_part.append(torch.full_like(grp[ok], net * 1024 + p))
                cls_group.append(net * 16 + grp[ok])
    errs = torch.cat(errs)
    kappa = max(PB.uniformity(f"{tag} dW partials by part", errs, torch.cat(cls_part)),
                PB.uniformity(f"{tag} dW partials by job group", errs, torch.cat(cls_group)))
    return worst, rms, kappa, sh


# ---------------------------------------------------------------------------------------------------------------- (e)
def check_input_rows(E, c, s, gouts, tag):
    """An input-gradient backward (row_x3_kernel) of the same forward; its rows from the kernel's own hi + lo dY0, dY3, dY6."""
    t = input_backward_state(E, c, s, gouts)
    recs = dev_tensor(t.dbg.records, (s.n_tiles, t.dbg.record_bytes // 2), "<i2")
    dy = []
    for L in (0, 3, 6):
        h, lo = hl(recs, dy_off(L), width(L))
        dy.append(h + lo)  # exact in FP32
    rw, kappa, gap = check_rows(E, c, s, t, tag, dy=dy)
    ry = check_rays(c, s, t, tag)
    cond = check_cond(c, t, tag)
    return rw, kappa, ry, cond


# ---------------------------------------------------------------------------------------------------------------- cases
def run_stages(E, c, tag, mode="full", gouts=None, expect=None, floor=None, rows=True):
    train_forward(E, c)
    s = debug_state(E, c)
    gouts = out_grads(E, c) if gouts is None else gouts
    t = PB.backward_state(E, c, s, gouts, mode)
    assert t.dbg.record_bytes == 2 * MIB
    PB.check_compositing(c, s, t, gouts, tag)
    check_operand_x3(t, tag)
    ch, ch_rms, lolo, ties, ch_kappa = check_chain_x3(E, c, s, t, tag, floor=floor)
    print(f"{tag}: chain {ch:.2f} of its bound, RMS {ch_rms:.1e} ({ch_rms / CHAIN_X3_RMS:.2f} of CHAIN_X3_RMS), lo.lo left out "
          f"{lolo:.1e}, {ties} ties, class RMS / overall {ch_kappa:.2f}")
    assert ch_rms <= CHAIN_X3_RMS, (tag, "dX chain relative RMS", ch_rms)
    dw, (rms, where), kappa, sh = check_partials_x3(E, c, s, t, tag)
    split_s = ", ".join(f"{t.parts[n]} parts, {sh[n][1]} tiles each, {sh[n][2]} filled" for n in range(2) if sh[n][0] is not None)
    print(f"{tag}: {split_s}; partials {dw:.2e} of gamma'(3 rows), RMS {rms:.1e} of its RMS ({rms / DW_X3_RMS:.2f} of DW_X3_RMS, {where}), "
          f"class RMS / overall {kappa:.2f}")
    assert rms <= DW_X3_RMS, (where, "relative RMS", rms)
    if expect:
        expect(t, sh)
    PB.check_reduce(c, t, sh, tag)
    fin = PB.check_finalize(c, t, tag) if mode == "full" else 0.0
    if rows:
        rw, r_kappa, ry, cond = check_input_rows(E, c, s, gouts, tag)
        print(f"{tag}: finalize {fin:.2e} of gamma(k); rows {rw:.1e} (class RMS / overall {r_kappa:.2f}), rays {ry:.1e}, "
              f"conditioning {cond:.1e}")
    return t, s


@pytest.mark.parametrize("case", list(PB.CASES))
def test_exact_grad_stages_against_float64(E, case):
    build, mode, expect = PB.CASES[case]
    run_stages(E, build(E, PREC), f"{case} {PREC}", mode=mode, expect=expect)


def test_zero_output_gradients(E):
    """All-zero output gradients: the loss scale is exactly 1 and every stage is exactly 0, in both halves."""
    c = make_case(E, 300, 64, 64, PREC, seed=11)
    gouts = [None if g is None else torch.zeros_like(g) for g in out_grads(E, c)]
    t, s = run_stages(E, c, f"zero {PREC}", gouts=gouts, rows=False)
    assert t.scale == 1.0 and t.inv == 1.0
    ti = input_backward_state(E, c, s, gouts)
    assert int(torch.count_nonzero(ti.rows.view(torch.int32))) == 0
    for off, rows in [(REC["draw"], 16)] + [(dy_off(L), width(L)) for L in range(9)]:
        for img in hl(t.recs, off, rows):
            assert int(torch.count_nonzero(img.view(torch.int32))) == 0, (off, "a zero backward left a nonzero dY bit")
    assert int(torch.count_nonzero(t.ws.view(torch.int32))) == 0
    for acc in t.acc:
        assert int(torch.count_nonzero(acc.view(torch.int32))) == 0


def test_lo_floor(E):
    """Per-ray output gradients spread over 1e-6 ... 1 (log-uniform): after the loss scale many dY lie below 2^-3, where lo is
    an FP16 subnormal and hi + lo keeps fewer bits.  Every stage keeps its bounds; per layer the share of such elements and
    the error of hi + lo there over the error of hi alone (the FP16 value exact mode's record would hold) are printed."""
    c = make_case(E, two_iter_rays(E), 64, 64, PREC, seed=90)
    g = torch.Generator().manual_seed(91)
    spread = (10.0 ** (-6.0 * torch.rand(c.n, generator=g))).to(E.dev)
    gouts = [None if x is None else x * (spread.view(-1, 1) if x.dim() == 2 else spread) for x in out_grads(E, c)]
    floor = []
    run_stages(E, c, f"lo floor {PREC}", gouts=gouts, floor=floor)
    for L, share, gain in floor:
        print(f"lo floor dY{L}: {100 * share:.1f} % of the live elements below 2^-3; there error(hi + lo) / error(hi) {gain:.2e}")
    assert any(share > 0.1 for _, share, _ in floor), floor  # the case reaches the floor


def test_stale_workspace(E):
    """test_param_backward_fp64_gpu.test_stale_workspace at exact_grad: NaN in the slots, d raw and bias sums a bigger backward
    left, then a smaller one on the same handle, bit-identical to a fresh handle's."""
    PB.test_stale_workspace(E, PREC)


def test_dy_overflow_is_visible_in_both_halves(E):
    """Weights re-balanced so that the forward is unchanged in exact arithmetic (layers_xyz.0 divided by g, layers_xyz.1
    multiplied by g: ReLU is positively homogeneous) but dY0 after the loss scale reaches about 4 times 65504: where hi is inf
    the lo image is non-finite too (hi + lo never turns the overflow into a finite number), and only dY0 overflows."""
    from test_backward_fp64_gpu import model
    c = make_case(E, two_iter_rays(E), 64, 64, PREC, seed=80)
    gouts = out_grads(E, c, seed=81)
    train_forward(E, c)
    s = debug_state(E, c)
    t = PB.backward_state(E, c, s, gouts, "full")
    used = [rowmap(c, s, pas) for pas in (0, 1)]
    big = max(float(decode_image(t.recs, dy_off(0), 256)[u].abs().max()) for u in used)
    gain = 4.0 * 65504.0 / big

    def rebalance(m):
        p = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
        p["layers_xyz.0.weight"] /= gain
        p["layers_xyz.0.bias"] /= gain
        p["layers_xyz.1.weight"] *= gain
        return model(E, 0, True, params=p)
    c.mc, c.mf = rebalance(c.mc), rebalance(c.mf)
    train_forward(E, c)
    s = debug_state(E, c)
    t = PB.backward_state(E, c, s, gouts, "full")
    assert t.scale == 1.0 / t.inv
    for L in range(1, 9):
        for img in hl(t.recs, dy_off(L), width(L)):
            assert bool(torch.isfinite(img).all()), (L, "only dY0 overflows")
    h, lo = hl(t.recs, dy_off(0), 256)
    inf = torch.isinf(h)
    assert int(inf.sum()) > 0, "dY0 did not overflow"
    assert bool((~torch.isfinite(lo[inf])).all()), "a finite lo beside an inf hi"
    assert bool(torch.isfinite(lo[~inf]).all()), "a non-finite lo beside a finite hi"
    assert not all(bool(torch.isfinite(x).all()) for x in list(t.kg[0]) + list(t.kg[1]) if x is not None)
    print(f"dY0 past 65504 (gain {gain:.3g}): {int(inf.sum())} inf hi, every lo beside them non-finite")


# ---------------------------------------------------------------------------------------------------------------- (f)
def dy_rows_x3(c, s, t):
    """Per pass [n, S, 512]: float(hi) + float(lo) of the dY0 | dY3 records of every (ray, sample) row (exact in FP32)."""
    recs = dev_tensor(t.dbg.records, (s.n_tiles, t.dbg.record_bytes // 2), "<i2")
    imgs = []
    for L in (0, 3):
        h, lo = hl(recs, dy_off(L), 256)
        imgs.append(h + lo)
    out = []
    for pas in range(2 if c.nf else 1):
        tile, row = rowmap(c, s, pas)
        S = c.nc + c.nf if pas else c.nc
        out.append(torch.cat([img[tile, row] for img in imgs], 1).view(c.n, S, 512))
    return out


@pytest.mark.parametrize("nfr,kind", [(5, "interleave"), (217, "blocks")], ids=["F5", "F217_blocks"])
def test_multi_frame_sums(E, nfr, kind):
    from test_backward_fp64_gpu import saved_state
    c = make_case(E, two_iter_rays(E), 64, 64, PREC, seed=nfr, dir_z=True)
    ex, la = frames(E, nfr, nfr)
    fi = layout(kind, c.n, nfr, nfr)
    E.eng.sync_weights(c.mc, c.mf)
    E.eng.set_frames(ex, la)
    render(E, c, True, fi)
    s = saved_state(E, c)
    st = frame_state(E, c)
    gouts = out_grads(E, c)
    pc, pf = params_of(c)
    valid = torch.ones(c.n, dtype=torch.bool, device=E.dev)
    for mode in ("input_only", "full"):
        gc, gf, gl, ing = E.eng.backward(list(gouts), pc, pf, want_params=mode == "full", inputs=wanted(c), frames=True)
        t = sums_state(E, c, st)
        assert t.dbg.record_bytes == 2 * MIB
        tag = f"F{nfr} {mode}"
        rsum, _ = check_raysums(E, c, s, t, tag, valid, dy=dy_rows_x3(c, s, t))
        fsum = check_framesums(c, st, t, tag)
        cond = check_cond_grads(c, st, t, gl, ing["expression"], tag)
        cols = check_cond_columns(c, st, t, gc, gf, tag) if mode == "full" else 0.0
        print(f"{tag}: share of the gamma bound: ray sums {rsum:.2e}, frame sums {fsum:.2e}, latent / expression {cond:.2e}, "
              f"columns {cols:.2e}")


def test_hooks_describe_exact_grad(E):
    """The debug hook of an exact-grad backward: 2 MiB records, the lo weight stream of both networks loaded."""
    c = make_case(E, 64, 64, 64, PREC, seed=2)
    train_forward(E, c)
    s = debug_state(E, c)
    t = PB.backward_state(E, c, s, out_grads(E, c), "full")
    assert t.dbg.record_bytes == 2 * MIB
    lay = WP.Layout(E.capi.lib)
    for net in (0, 1):
        hi, lo = stream_weights(E, net, lay)
        assert sorted(hi) == list(range(9)) and all(bool(torch.isfinite(hi[L]).all() and torch.isfinite(lo[L]).all()) for L in hi)
        assert sum(int(torch.count_nonzero(lo[L])) for L in lo) > sum(hi[L].numel() for L in hi) // 4  # the lo half is populated
