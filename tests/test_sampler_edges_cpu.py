"""The exact cumulative sum behind both device ray samplers (csrc/nfb_sampler.h) at the edges of its arithmetic, through the
host-only hook nfb_host_map_cdf: every one of the H*W partial sums must equal np.cumsum of the reference's importance map, bit
for bit, and the hook must return 0 (which it does only when the map's segments fit the kMaxSegs table the device uses).

Coverage beyond test_sampler_cpu.py (all at p = 0.9):
  * p from 1e-15 to 1 - 1e-15.  Far from 0.9 one of the map's two constants drops below half an ulp of the running sum, so
    np.cumsum stops moving on those adds (absorbed adds, nfb_sampler.h's d = 0 case).  Before that case had a segment of its
    own, every absorbed add took a segment: 63,285 segments for the 512^2 reference box at p = 1e-12.  Eight of the maps
    below then overflowed the 16,384-entry table, so the hook returned NFB_ERR_UNSUPPORTED for them (the device searched
    segments it never wrote).
  * frames with H != W both ways, 1-pixel boxes in every corner, a full-width box (zero-length q_out runs between box rows),
    a full-frame box (q_in == q_out), an empty box (one run), a 1024^2 single-column full-height box (2,049 runs) and the
    2048^2 box of 2,047 rows: 4,095 runs, the run table's capacity (kMaxRuns = 4096).  A 2,048-row box has 4,097 runs and
    must be refused.
  * zeroed entries (the pixels earlier rounds of np.random.choice found): random sets of 1, 37 and 2,047; the first and last
    entry of every run; one whole run; 2,047 consecutive entries around the first absorbed add.
No GPU."""
import ctypes as C

import numpy as np
import pytest

NFB_ERR_UNSUPPORTED = 2
P_VALUES = [1e-15, 1e-12, 1e-6, 0.5, 0.9, 1 - 1e-6, 1 - 1e-12, 1 - 1e-15]
MAPS = {  # name: (H, W, bbox = probs[b0:b1, b2:b3])
    "512 reference box": (512, 512, (150, 400, 128, 380)),
    "96x160": (96, 160, (20, 70, 30, 130)),
    "160x96": (160, 96, (30, 130, 20, 70)),
    "pixel top left": (96, 160, (0, 1, 0, 1)),
    "pixel top right": (96, 160, (0, 1, 159, 160)),
    "pixel bottom left": (96, 160, (95, 96, 0, 1)),
    "pixel bottom right": (96, 160, (95, 96, 159, 160)),
    "full width": (96, 160, (20, 60, 0, 160)),
    "full frame": (96, 160, (0, 96, 0, 160)),
    "empty box": (96, 160, (40, 40, 5, 9)),
    "1024 one column": (1024, 1024, (0, 1024, 517, 518)),
    "2048 capacity": (2048, 2048, (0, 2047, 3, 2045)),
}


@pytest.fixture(scope="module")
def lib(built_lib):
    import nerf  # noqa: F401
    from nerf import _capi
    return _capi


def host_cdf(capi, m, zeroed, n):
    """(return code, nfb_host_map_cdf at every k < n) for the map with the flat indices `zeroed` set to zero."""
    z = np.ascontiguousarray(np.unique(np.asarray(zeroed, dtype=np.int64)))
    ks = np.arange(n, dtype=np.int64)
    out = np.full(n, np.nan)
    rc = capi.lib.nfb_host_map_cdf(C.byref(m), z.ctypes.data_as(C.POINTER(C.c_longlong)) if z.size else None, int(z.size),
                                   ks.ctypes.data_as(C.POINTER(C.c_longlong)), n, out.ctypes.data_as(C.POINTER(C.c_double)))
    return rc, out


def runs_of(H, W, bbox):
    """[(first flat index, length)] of the map's constant runs in row-major order (the box as importance_map clamps it)."""
    b0, b1, b2, b3 = max(0, min(bbox[0], H)), max(0, min(bbox[1], H)), max(0, min(bbox[2], W)), max(0, min(bbox[3], W))
    if b1 <= b0 or b3 <= b2:
        return [(0, H * W)]
    runs = [(0, b0 * W + b2)]
    for row in range(b0, b1):
        runs.append((row * W + b2, b3 - b2))
        end = H * W if row == b1 - 1 else (row + 1) * W + b2
        runs.append((row * W + b3, end - (row * W + b3)))
    return runs


def first_absorbed(flat):
    """Index of the first positive entry np.cumsum adds without moving the sum, or None."""
    cs = np.cumsum(flat)
    k = np.flatnonzero((flat[1:] > 0) & (cs[1:] == cs[:-1]))
    return int(k[0]) + 1 if k.size else None


def zeroed_sets(H, W, bbox, flat, seed):
    n = H * W
    rng = np.random.default_rng(seed)
    runs = [(k0, ln) for k0, ln in runs_of(H, W, bbox) if ln > 0]
    sets = {f"random {c}": rng.choice(n, size=c, replace=False) for c in (1, 37, 2047)}
    sets["run ends"] = np.array([k for k0, ln in runs for k in (k0, k0 + ln - 1)])
    whole = [r for r in runs if r[1] <= 2047]  # a selection zeroes at most 2047 entries
    if whole:
        k0, ln = max(whole, key=lambda r: r[1])
        sets["whole run"] = np.arange(k0, k0 + ln)
    a = first_absorbed(flat)
    if a is not None:
        lo = min(max(0, a - 1023), n - 2047)
        sets["around the first absorbed add"] = np.arange(lo, lo + 2047)
    return sets


@pytest.mark.parametrize("p", P_VALUES)
@pytest.mark.parametrize("name", list(MAPS))
def test_every_partial_sum_equals_numpy_cumsum(lib, name, p):
    from nerf import ray_sampler
    H, W, bbox = MAPS[name]
    m, flat = ray_sampler.importance_map(H, W, bbox, p)
    assert sorted(set(flat.tolist())) == sorted({m.q_in, m.q_out})
    cases = {"none": np.zeros(0, dtype=np.int64)}
    cases.update(zeroed_sets(H, W, bbox, flat, seed=H * 7 + W + int(p * 1000)))
    for what, z in cases.items():
        pz = flat.copy()
        pz[z] = 0.0
        want = np.cumsum(pz)
        rc, got = host_cdf(lib, m, z, H * W)
        assert rc == 0, (name, p, what, rc)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (name, p, what, bad.size, int(bad[0]), got[bad[0]], want[bad[0]])


def test_the_sweep_reaches_absorbed_adds(lib):
    """The p sweep above is not vacuous: np.cumsum absorbs adds on these maps (and not at the reference's p = 0.9)."""
    from nerf import ray_sampler
    for name, p, absorbs in (("512 reference box", 1e-12, True), ("512 reference box", 1 - 1e-12, True),
                             ("2048 capacity", 1e-15, True), ("2048 capacity", 1 - 1e-12, True),
                             ("1024 one column", 1 - 1e-15, True), ("512 reference box", 0.9, False), ("2048 capacity", 0.9, False)):
        H, W, bbox = MAPS[name]
        flat = ray_sampler.importance_map(H, W, bbox, p)[1]
        assert (first_absorbed(flat) is not None) == absorbs, (name, p)


@pytest.mark.parametrize("W,bbox,ok", [(8, (0, 2047, 3, 5), True), (8, (1, 2048, 0, 8), True), (8, (0, 2048, 3, 5), False),
                                       (2048, (0, 2048, 3, 2045), False)])
def test_run_table_capacity(lib, W, bbox, ok):
    """2,047 box rows give 4,095 runs: the table's capacity, exact.  2,048 rows give 4,097: NFB_ERR_UNSUPPORTED."""
    from nerf import ray_sampler
    H = 2048
    m, flat = ray_sampler.importance_map(H, W, bbox, 0.9)
    assert len(runs_of(H, W, bbox)) == (4095 if ok else 4097)
    rc, got = host_cdf(lib, m, [], H * W)
    if ok:
        assert rc == 0 and np.array_equal(got, np.cumsum(flat))
    else:
        assert rc == NFB_ERR_UNSUPPORTED
