"""The host restatement of the packed weight buffers (tests/weight_pack_reference.py) checked against the unit programs the
kernels follow (nfb_debug_schedule), no GPU involved: the (step, unit, row, 16-byte chunk) ranges cover each stream exactly
once, every weight element the forward reads through the x1 stream lands there exactly once and every element of the nine
matrices the backward chain runs through lands in the bwd stream exactly once, transposed, and the padding is exactly the rest.
test_weight_pack_fp64_gpu.py compares what the pack kernels wrote with this restatement byte for byte."""
import numpy as np
import pytest

import weight_pack_reference as R


@pytest.fixture(scope="module")
def layout(built_lib):
    import ctypes as C
    return R.Layout(C.CDLL(built_lib))


def decode(off_in_unit):
    """Inverse of the swizzle: (row, K index in the atom) of byte offsets inside a unit."""
    n = off_in_unit // 128
    return n, ((((off_in_unit % 128) >> 4) ^ (n & 7)) << 3) + ((off_in_unit % 16) >> 1)


@pytest.mark.parametrize("stream", ["fwd", "bwd"])
def test_unit_chunks_cover_each_stream_once(layout, stream):
    """Per unit the rows x 8 chunks of 16 bytes, walked in program order, tile [0, stream bytes) with no gap and no overlap;
    steps come in order with their units in K order; the row count of a unit is the step's N."""
    us = layout.fwd_units if stream == "fwd" else layout.bwd_units
    total = R.X1_BYTES if stream == "fwd" else R.BWD_BYTES
    ks = R.FWD_K if stream == "fwd" else R.BWD_K
    seen = np.zeros(total // 16, np.int64)
    for s, u, rows, off in us:
        assert off % 1024 == 0 and rows in (16, 128, 144, 256)
        np.add.at(seen, off // 16 + np.arange(rows * 8), 1)
    assert (seen == 1).all()
    assert [s for s, _, _, _ in us] == sorted(s for s, _, _, _ in us)
    for s in range(len(ks)):
        assert [u for t, u, _, _ in us if t == s] == list(range(ks[s] // 64))
    assert [r for s, u, r, _ in us if u == 0] == ([256] * 6 + [144, 128, 128, 16] if stream == "fwd" else [128] * 3 + [256] * 6)
    for name, n in (("x1", R.X1_BYTES // 2), ("x3", R.X1_BYTES), ("bwd", R.BWD_BYTES // 2)):
        assert (layout.covers[name] == 1).all(), name   # and so every FP16 slot of the three streams is written once
        assert getattr(layout, name).size == n


def test_swizzle_is_the_sw128_pattern(layout):
    """The restatement's position rule, decoded back: (row, k) of every slot of a unit, in 128-byte rows whose 16-byte chunks are
    XORed with row & 7; chunk j of row n stays within row n and distinct (n, k) never share a byte."""
    p = R.unit_positions(256, 0)
    n, k = decode(p)
    assert (n == np.arange(256)[:, None]).all() and (k == np.arange(64)[None, :]).all()
    assert np.unique(p).size == p.size and p.max() < 256 * 128


def forward_read():
    """Source indices of every weight element the forward MLP multiplies through the x1 stream (the model's forward with the
    conditioning columns folded into per-frame biases and fc_feat folded into W6)."""
    idx = []
    for t, (rows, cols) in ((0, (256, 171)), (6, (256, 427))):
        c = np.arange(cols)
        keep = (c < 63) | (c >= 171)
        idx.append((R.BASE[t] + np.arange(rows)[:, None] * cols + c[keep][None, :]).ravel())
    for t in (2, 4, 8, 10, 18, 20, 24):
        idx.append(R.BASE[t] + np.arange(R.SIZES[t]))
    idx.append(R.BASE[R.W6] + np.arange(129 * 256))
    return np.sort(np.concatenate(idx))


def test_forward_elements_land_once(layout):
    """x1 holds every forward-read element exactly once and nothing else but padding; the x3 hi units and lo units each hold
    the same assignment as x1 (two slots per element)."""
    got = layout.x1[layout.x1 >= 0]
    assert np.array_equal(np.sort(got), forward_read())
    assert (layout.x1 >= -1).all()
    hi, lo = layout.x3[~layout.x3_lo], layout.x3[layout.x3_lo]
    assert np.array_equal(np.sort(hi), np.sort(layout.x1)) and np.array_equal(np.sort(lo), np.sort(layout.x1))
    # same position rule: x1 slot i of unit at off <-> x3 hi slot i of unit at 2 off, lo slot rows * 64 later
    for s, u, rows, off in layout.fwd_units:
        a = layout.x1[off // 2:off // 2 + rows * 64]
        assert np.array_equal(layout.x3[off:off + rows * 64], a) and np.array_equal(layout.x3[off + rows * 64:off + rows * 128], a)


def test_chain_elements_land_once_transposed(layout):
    """bwd holds every element of fc_rgb.weight, layers_dir.2/.1, M1 = W6[:128] and m2 = W6[128], layers_xyz.5/.4,
    layers_xyz.3[:, 171:], layers_xyz.2/.1 exactly once, and slot (row n, k) of step s holds W[k][n] of that step's matrix."""
    want = [R.BASE[t] + np.arange(R.SIZES[t]) for t in (24, 20, 18, 10, 8, 4, 2)]
    want.append(R.BASE[6] + (np.arange(256)[:, None] * 427 + 171 + np.arange(256)[None, :]).ravel())
    want.append(R.BASE[R.W6] + np.arange(129 * 256))
    got = layout.bwd[layout.bwd >= 0]
    assert np.array_equal(np.sort(got), np.sort(np.concatenate(want)))
    mats = {0: (24, 128, 0), 1: (20, 128, 0), 2: (18, 128, 0), 4: (10, 256, 0), 5: (8, 256, 0), 6: (6, 427, 171), 7: (4, 256, 0),
            8: (2, 256, 0)}
    for s, u, rows, off in layout.bwd_units:
        b = off + np.arange(rows * 128, step=2)
        n, k = decode(b - off)
        src = layout.bwd[b // 2]
        kk = 64 * u + k
        if s == 3:
            kind = np.where(kk < 64, np.where(kk == 3, R.BASE[R.W6] + 128 * 256 + n, -1), R.BASE[R.W6] + (kk - 64) * 256 + n)
        else:
            t, ld, c0 = mats[s]
            kind = np.where((kk < 3) | (s != 0), R.BASE[t] + kk * ld + c0 + n, -1)
        assert np.array_equal(src, kind), (s, u)


def test_padding_is_the_complement(layout):
    """Padding slots are exactly: x1 / x3 rows 129..143 of step 6 and 3..15 of step 9, K index 63 of the PE atoms of steps 0
    and 3; bwd K indices 3..63 of step 0's operand atom and every K index but 3 of step 3's."""
    pad = np.zeros(R.X1_BYTES // 2, bool)
    for s, u, rows, off in layout.fwd_units:
        n, k = decode(np.arange(rows * 128, step=2))
        p = (s == 6) & (n >= 129) | (s == 9) & (n >= 3) | (s in (0, 3)) & (u == 0) & (k == 63)
        pad[(off + np.arange(rows * 128, step=2)) // 2] = p
    assert np.array_equal(layout.x1 == -1, pad)
    assert int(pad.sum()) == 15 * 256 + 13 * 128 + 2 * 256
    padb = np.zeros(R.BWD_BYTES // 2, bool)
    for s, u, rows, off in layout.bwd_units:
        n, k = decode(np.arange(rows * 128, step=2))
        padb[(off + np.arange(rows * 128, step=2)) // 2] = ((s == 0) & (k >= 3)) | ((s == 3) & (u == 0) & (k != 3))
    assert np.array_equal(layout.bwd == -1, padb)
    assert int(padb.sum()) == 128 * 61 + 256 * 63
