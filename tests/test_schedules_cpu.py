"""Host-only checks of the compile-time schedules the kernels execute (nfb_debug_schedule): every weight byte of the packed
streams is consumed exactly once per tile by the render program and by the backward chain, units fit their ring slots, A
operands come from the activation buffer's four K atoms, and the weight-gradient jobs tile the accumulator space without overlap.  These are
the invariants a change to csrc/nfb_layout.h or to one of the program builders can silently break; no GPU involved."""
import ctypes as C

import pytest

STREAM_X1 = 864256      # nfb_layout.h kStreamBytesX1
STREAM_BWD = 835584     # kBwdStreamBytes
REC_BYTES = 1 << 20
ACC_FLOATS = 499204     # kAccFloats


@pytest.fixture(scope="module")
def lib(built_lib):
    lb = C.CDLL(built_lib)
    lb.nfb_debug_schedule.restype = C.c_int
    lb.nfb_debug_schedule.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_uint32), C.c_int]
    return lb


def entries(lib, which):
    n = lib.nfb_debug_schedule(which, -1, None, 0)
    assert n > 0
    out = []
    buf = (C.c_uint32 * 10)()
    for i in range(n):
        w = lib.nfb_debug_schedule(which, i, buf, 10)
        assert w > 0
        out.append([int(buf[k]) for k in range(w)])
    assert lib.nfb_debug_schedule(which, n, buf, 10) == -1
    return out


def spans(ents):
    return [((e[3] & 0xFFFFF) << 4, (e[3] >> 20) * 128) for e in ents]


def assert_exact_cover(sp, total):
    sp = sorted(sp)
    pos = 0
    for off, nbytes in sp:
        assert off == pos, (off, pos)
        pos += nbytes
    assert pos == total


def test_one_tile_program_covers_the_weight_stream(lib):
    ents = entries(lib, 0)
    assert len(ents) == 32
    sp = spans(ents)
    assert_exact_cover(sp, STREAM_X1)
    for e, (off, nbytes) in zip(ents, sp):
        assert nbytes <= 32768 and off % 1024 == 0          # one ring slot, swizzle-aligned
        assert e[0] * 128 == nbytes                          # MMA N == rows of the unit
        assert (e[2] & 1 and e[1] == 0) or e[1] < 4          # A operand: the PE buffer or one K atom of the activation buffer
    assert sum(1 for e in ents if e[2] & 16) == 10           # one "step complete" unit per step
    assert sum(1 for e in ents if e[2] & 8) == 10            # one "first unit" per step


def test_backward_chain_program(lib):
    ents = entries(lib, 2)
    assert len(ents) == 28
    assert_exact_cover(spans(ents), STREAM_BWD)
    for e, (off, nbytes) in zip(ents, spans(ents)):
        assert e[0] in (128, 256) and e[0] * 128 == nbytes
        assert (e[2] & 1 and e[1] == 0) or e[1] < 4
    assert sum(1 for e in ents if e[2] & 16) == 9            # nine steps


def test_weight_gradient_jobs(lib):
    jobs = entries(lib, 3)
    assert len(jobs) == 21
    used = []
    for a_off, a_rows, a_half, b_off, b_rows, bias_layer, out_off, out_ld, out_row0, group in jobs:
        bias_layer = bias_layer - (1 << 32) if bias_layer >= (1 << 31) else bias_layer   # -1 = no bias, sent as uint32
        assert 0 <= a_off and a_off + 2 * a_rows * 128 <= REC_BYTES and a_rows in (128, 256) and a_half * 128 < a_rows
        assert 0 <= b_off and b_off + 2 * b_rows * 128 <= REC_BYTES and b_rows in (16, 32, 64, 128, 256) and b_rows == out_ld
        assert -1 <= bias_layer <= 8 and 0 <= group < 8
        lo = out_off + out_row0 * out_ld
        used.append((lo, lo + 128 * out_ld))
    used.sort()
    for (a0, a1), (b0, b1) in zip(used, used[1:]):
        assert a1 <= b0, "weight-gradient jobs overlap in the accumulator space"
    assert used[-1][1] <= ACC_FLOATS
    # groups 2q / 2q+1 (q < 3) are the two output halves of the same layers in the same order: neighbouring CTAs stream the same
    # B images of the same tiles at the same time (one HBM read, one L2 hit); per-tile bytes of the groups are balanced
    by_group = [[j for j in jobs if j[9] == g] for g in range(8)]
    for q in range(3):
        lo, hi = by_group[2 * q], by_group[2 * q + 1]
        assert len(lo) == len(hi) and len(lo) >= 2
        for a, b in zip(lo, hi):
            assert a[0] == b[0] and a[3] == b[3] and a[4] == b[4] and (a[2], b[2]) == (0, 1) and a[6] == b[6] and (a[8], b[8]) == (0, 128)
    load = [sum(2 * 128 * (128 + j[4]) for j in grp) for grp in by_group]
    assert max(load) <= 1.2 * min(load), load
    biased = [j[5] for j in jobs if j[5] < (1 << 31)]
    assert sorted(set(biased)) == list(range(9))                         # every layer's bias is produced ...
    assert len([b for b in biased if b <= 5]) == 12                      # ... by both halves of the 256-wide layers, once each


@pytest.mark.parametrize("sms,t0,t1", [(148, 1024, 2048), (148, 128, 256), (148, 24, 48), (148, 5, 0), (148, 1, 2), (148, 3, 1000),
                                        (148, 1000, 3), (8, 10, 20), (132, 2048, 2048), (148, 0, 7)])
def test_weight_gradient_cta_split(lib, sms, t0, t1):
    """launch_dw's host logic (csrc/nfb_train.cu: dw_split): the CTAs of the one weight-gradient launch are split between the two
    networks in proportion to their tile counts; every non-empty network gets at least one part, never more parts than tiles,
    and the 64c+64f training batch (1024 + 2048 tiles) gets 6 + 12 parts of 8 CTAs = the same 171 tiles per CTA."""
    buf = (C.c_uint32 * 16)(sms, t0, t1)
    assert lib.nfb_debug_schedule(4, 0, buf, 16) == 3
    p0, p1, groups = int(buf[0]), int(buf[1]), int(buf[2])
    assert groups == 8
    assert (p0 >= 1) == (t0 > 0) and (p1 >= 1) == (t1 > 0)
    assert p0 <= max(t0, 0) and p1 <= max(t1, 0)
    assert (p0 + p1) * groups <= max(sms, 16)
    if (sms, t0, t1) == (148, 1024, 2048):
        assert (p0, p1) == (6, 12) and -(-t0 // p0) == -(-t1 // p1) == 171
    if t0 > 0 and t1 > 0 and min(t0, t1) >= 18:  # proportional within one part
        assert abs(p0 / (p0 + p1) - t0 / (t0 + t1)) <= 1.0 / (p0 + p1)
