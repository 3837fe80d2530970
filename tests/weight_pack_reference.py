"""numpy restatement of the packed weight buffers nfb_load_weights / nfb_repack write (csrc/nfb_pack.cu: fold_feat_kernel,
repack_kernel), from the 26 FP32 state_dict tensors, written from the model (ConditionalBlendshapePaperNeRFModel.forward,
nerf/models.py; the reference's models.py:218-261) and the layout rule of DESIGN.md §3 — not from the pack kernels.

  forward step s, row n, logical K index k -> the state_dict element it stands for:
    0       layers_xyz.0.weight[n, k] for k < 63 (the PE columns); k = 63 is padding (the PE atom has 63 lanes)
    1, 2    layers_xyz.{1,2}.weight[n, k]
    3       layers_xyz.3.weight[n, k] for k < 63, padding at k = 63, layers_xyz.3.weight[n, 171 + (k - 64)] for k >= 64
            (columns 63..170 of layers_xyz.0 / .3 multiply the per-frame conditioning; they live in w0c / w3c)
    4, 5    layers_xyz.{4,5}.weight[n, k]
    6       W6[n, k]: the float64 fold layers_dir.0[:, :256] . fc_feat (rows 0..127), fc_alpha . fc_feat (row 128), to FP32
    7, 8    layers_dir.{1,2}.weight[n, k]
    9       fc_rgb.weight[n, k] for n < 3
  backward chain step s, row n, K index k -> W^T of the layer it runs through (nfb_layout.h bwd_step_info):
    0       fc_rgb.weight[k, n] for k < 3 (the d-raw operand atom)
    1, 2    layers_dir.2 / .1 .weight[k, n]
    3       m2[n] = W6[128, n] at k = 3 of the operand atom; then M1^T: W6[k - 64, n]
    4..8    layers_xyz.5, .4, .3[:, 171:], .2, .1 .weight[k, n]
  Rows beyond the matrix (W6 rows 129..143, fc_rgb rows 3..15) and every unnamed K index are padding: +0 (bits 0x0000).

Where an element lands: unit u of step s (64 K indices [64u, 64u + 64), all rows of the step) sits at the byte offset the
kernels' unit program gives (nfb_debug_schedule(0 / 2, ...)); inside the unit element (n, k) is at
n * 128 + ((k >> 3 & 7) ^ (n & 7)) * 16 + 2 * (k & 7).  x1 holds fp16_rn(w); x3 holds per unit the same hi unit at twice the
x1 offset, then lo = fp16_rn(w - hi) rows * 128 bytes after it; bwd holds fp16_rn(w).  The other buffers: bias_static =
layers_xyz.{0..5}.bias, b6 [144], layers_dir.1.bias, layers_dir.2.bias, fc_rgb.bias, zeros to 1952 floats; w0c / w3c =
layers_xyz.0 / .3 .weight[:, 63:171] ([256][108]); wd0b_t = layers_dir.0.weight[:, 256:280]^T ([24][128]).

A position's "source" is an index into the concatenation of the 26 flattened tensors followed by W6 ([144][256]), or -1
for padding; the buffers are values gathered through those indices, so the tests can check both where every element went and
what it holds."""
import ctypes as C

import numpy as np

PARAM_ORDER = ([f"layers_xyz.{i}.{k}" for i in range(6) for k in ("weight", "bias")]
               + ["fc_feat.weight", "fc_feat.bias", "fc_alpha.weight", "fc_alpha.bias"]
               + [f"layers_dir.{i}.{k}" for i in range(4) for k in ("weight", "bias")]
               + ["fc_rgb.weight", "fc_rgb.bias"])
SHAPES = ([(256, 171), (256,), (256, 256), (256,), (256, 256), (256,), (256, 427), (256,), (256, 256), (256,), (256, 256), (256,)]
          + [(256, 256), (256,), (1, 256), (1,)] + [(128, 280), (128,), (128, 128), (128,), (128, 128), (128,), (128, 128), (128,)]
          + [(3, 128), (3,)])
W6 = 26                       # pseudo-tensor index of the fold, [144][256]
W6_ROWS = 144
SIZES = [int(np.prod(s)) for s in SHAPES] + [W6_ROWS * 256]
BASE = np.concatenate([[0], np.cumsum(SIZES)]).astype(np.int64)
X1_BYTES, BWD_BYTES, BIAS_FLOATS = 864256, 835584, 1952
DIM_XYZ, DIM_COND, DIM_DIR = 63, 108, 24
FWD_K = [64, 256, 256, 320, 256, 256, 256, 128, 128, 128]
FWD_VALID_ROWS = [256] * 6 + [129, 128, 128, 3]
BWD_K = [64, 128, 128, 192, 256, 256, 256, 256, 256]
BWD_SRC = {1: 20, 2: 18, 4: 10, 5: 8, 6: 6, 7: 4, 8: 2}  # backward step -> layer weight it runs through (transposed)
UNIT_FIRST = 8                                          # nfb_layout.h kUnitFirst


def units(lib, which):
    """(step, unit, rows, byte offset) of every unit of the forward (which = 0) or backward (2) stream, in program order, from
    nfb_debug_schedule: the step advances at each entry flagged as a step's first unit."""
    lib.nfb_debug_schedule.restype = C.c_int
    lib.nfb_debug_schedule.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_uint32), C.c_int]
    buf = (C.c_uint32 * 10)()
    out, s, u = [], -1, 0
    for i in range(lib.nfb_debug_schedule(which, -1, None, 0)):
        assert lib.nfb_debug_schedule(which, i, buf, 10) == 4
        if buf[2] & UNIT_FIRST:
            s, u = s + 1, 0
        out.append((s, u, int(buf[3]) >> 20, (int(buf[3]) & 0xFFFFF) << 4))
        u += 1
    return out


def _src(t, rows, cols, ld, valid):
    """Source indices of tensor t's elements at (rows, cols) of a row-major matrix with leading dimension ld; -1 where not valid."""
    return np.where(valid, BASE[t] + np.where(valid, rows * ld + cols, 0), -1)


def fwd_source(s, rows):
    """[rows, K] source indices of forward step s (module docstring)."""
    n = np.arange(rows)[:, None]
    k = np.arange(FWD_K[s])[None, :]
    valid = n < FWD_VALID_ROWS[s]
    if s in (0, 3):
        col = np.where(k < DIM_XYZ, k, DIM_XYZ + DIM_COND + (k - 64))
        return _src(2 * s, n, col, 171 if s == 0 else 427, valid & (k != DIM_XYZ))
    if s <= 5:
        return _src(2 * s, n, k, 256, valid & (k >= 0))
    if s == 6:
        return _src(W6, n, k, 256, valid & (k >= 0))
    return _src({7: 18, 8: 20, 9: 24}[s], n, k, 128, valid & (k >= 0))


def bwd_source(s, rows):
    """[rows, K] source indices of backward chain step s: element (n, k) = W[k][n]."""
    n = np.arange(rows)[:, None]
    k = np.arange(BWD_K[s])[None, :]
    if s == 0:
        return _src(24, k, n, 128, (k < 3) & (n >= 0))
    if s == 3:
        op = _src(W6, 128, n, 256, (k == 3) & (n >= 0))
        return np.where(k < 64, op, _src(W6, k - 64, n, 256, (k >= 64) & (n >= 0)))
    t = BWD_SRC[s]
    if s == 6:
        return _src(t, k, DIM_XYZ + DIM_COND + n, 427, (k >= 0) & (n >= 0))
    return _src(t, k, n, 128 if s <= 2 else 256, (k >= 0) & (n >= 0))


def unit_positions(rows, off):
    """[rows, 64] byte offsets of the elements (n, k) of a unit starting at `off`."""
    n = np.arange(rows)[:, None]
    k = np.arange(64)[None, :]
    return off + n * 128 + ((((k >> 3) & 7) ^ (n & 7)) << 4) + 2 * (k & 7)


class Layout:
    """Per FP16 slot of x1, x3 and bwd: the source index it holds (-1 padding, -2 no unit covers it); x3_lo marks lo slots.
    covers[name] counts how many (step, unit, row, element) positions landed on each slot."""

    def __init__(self, lib):
        self.fwd_units, self.bwd_units = units(lib, 0), units(lib, 2)
        self.x1 = np.full(X1_BYTES // 2, -2, np.int64)
        self.x3 = np.full(X1_BYTES, -2, np.int64)
        self.x3_lo = np.zeros(X1_BYTES, bool)
        self.bwd = np.full(BWD_BYTES // 2, -2, np.int64)
        self.covers = dict(x1=np.zeros(X1_BYTES // 2, np.int64), x3=np.zeros(X1_BYTES, np.int64), bwd=np.zeros(BWD_BYTES // 2, np.int64))
        hi_lo = []  # (x3 hi slot, x3 lo slot) of each element
        srcs = {}
        for s, u, rows, off in self.fwd_units:
            src = srcs.setdefault(("f", s), fwd_source(s, rows))[:, 64 * u:64 * u + 64]
            p = unit_positions(rows, off) // 2
            self.x1[p] = src
            np.add.at(self.covers["x1"], p.ravel(), 1)
            p3 = unit_positions(rows, 2 * off) // 2
            for q in (p3, p3 + rows * 64):
                self.x3[q] = src
                np.add.at(self.covers["x3"], q.ravel(), 1)
            self.x3_lo[p3 + rows * 64] = True
            hi_lo.append(np.stack([p3.ravel(), p3.ravel() + rows * 64]))
        self.x3_hi_slot, self.x3_lo_slot = np.concatenate(hi_lo, axis=1)
        for s, u, rows, off in self.bwd_units:
            src = srcs.setdefault(("b", s), bwd_source(s, rows))[:, 64 * u:64 * u + 64]
            p = unit_positions(rows, off) // 2
            self.bwd[p] = src
            np.add.at(self.covers["bwd"], p.ravel(), 1)


def flat_params(params):
    """The 26 tensors (dict by state_dict name, or list in PARAM_ORDER; numpy or torch) as FP32 numpy arrays."""
    ts = [params[k] for k in PARAM_ORDER] if isinstance(params, dict) else list(params)
    out = []
    for t, shape in zip(ts, SHAPES):
        a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
        assert a.dtype == np.float32 and a.shape == shape, (a.dtype, a.shape, shape)
        out.append(a)
    return out


def fold64(p):
    """The fold in float64 with compensated (Neumaier) summation of the exact FP32 x FP32 products: W6 [144][256] and b6 [144]
    (rows 129..143 zero), and the sums of absolute values of the terms (for b6 including |bias|)."""
    left = np.concatenate([p[16][:, :256], p[14]]).astype(np.float64)   # [129, 256]
    wf, bf = p[12].astype(np.float64), p[13].astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        def nsum(s, terms):  # terms: iterable of arrays; s: the start value
            c = np.zeros_like(s)
            a = np.abs(s)
            for t in terms:
                u = s + t
                c += np.where(np.abs(s) >= np.abs(t), (s - u) + t, (t - u) + s)
                s = u
                a = a + np.abs(t)
            return s + c, a
        w, wa = nsum(np.zeros((129, 256)), (left[:, j, None] * wf[None, j, :] for j in range(256)))
        b, ba = nsum(np.concatenate([p[17], p[15]]).astype(np.float64), (left[:, j] * bf[j] for j in range(256)))
    z = lambda a, shape: np.concatenate([a, np.zeros(shape)])  # noqa: E731
    return z(w, (15, 256)), z(b, (15,)), z(wa, (15, 256)), z(ba, (15,))


def fp16(v):
    with np.errstate(over="ignore", invalid="ignore"):
        return v.astype(np.float16)


def values(p, w6):
    """FP32 values by source index (module docstring), with one more +0 at the end that padding (-1) reads."""
    return np.concatenate([a.ravel() for a in p] + [np.asarray(w6, np.float32).ravel(), np.zeros(1, np.float32)])


def expected(p, w6, b6, layout):
    """Expected contents of every buffer for FP32 tensors p (flat_params) with the fold's FP32 result w6 [144][256] / b6 [144]:
    dict of x1, x3, bwd (uint16 words) and bias_static, w0c, w3c, wd0b_t (float32)."""
    vals = values(p, w6)

    def gather(src):
        assert (src >= -1).all(), "a slot no unit covers"
        return vals[np.where(src < 0, len(vals) - 1, src)]

    x1 = fp16(gather(layout.x1))
    w3 = gather(layout.x3)
    hi = fp16(w3)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = fp16(w3 - hi.astype(np.float32))
    x3 = np.where(layout.x3_lo, lo, hi)
    bias = np.concatenate([p[2 * i + 1] for i in range(6)] + [np.asarray(b6, np.float32), p[19], p[21], p[25], np.zeros(13, np.float32)])
    assert bias.size == BIAS_FLOATS
    return dict(x1=x1.view(np.uint16), x3=x3.view(np.uint16), bwd=fp16(gather(layout.bwd)).view(np.uint16),
                bias_static=bias.astype(np.float32), w0c=np.ascontiguousarray(p[0][:, DIM_XYZ:DIM_XYZ + DIM_COND]),
                w3c=np.ascontiguousarray(p[6][:, DIM_XYZ:DIM_XYZ + DIM_COND]), wd0b_t=np.ascontiguousarray(p[16][:, 256:280].T))


def frame_rows64(p, bias_static, expr, latent):
    """float64 of the folded bias rows nfb_set_frame writes: bias_static[i] + W[n, 63:171] . c for i = n (step 0) and
    768 + n (step 3), c = [fp32(expr / 3) ; latent]; and the sums of absolute values of the terms."""
    c = np.concatenate([(np.asarray(expr, np.float32) / np.float32(3)).astype(np.float32), np.asarray(latent, np.float32)]).astype(np.float64)
    out, absum = {}, {}
    for i0, w in ((0, p[0]), (768, p[6])):
        wc = w[:, DIM_XYZ:DIM_XYZ + DIM_COND].astype(np.float64)
        b = bias_static[i0:i0 + 256].astype(np.float64)
        out[i0] = b + wc @ c
        absum[i0] = np.abs(b) + np.abs(wc) @ np.abs(c)
    return out, absum
