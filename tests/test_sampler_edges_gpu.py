"""Both device ray samplers against numpy's own np.random.choice at the edges of their exact cumulative sum: nfb_sample_rays (one
image) and nfb_sample_rays_images (K images, one block each), fed the uniform draws numpy consumed, must return numpy's indices
and numpy's state (rounds run, draws consumed) bit for bit.  test_post_gpu.py and test_train_images_gpu.py cover p = 0.9,
square frames and K <= 8; this file covers:
  * p from 1e-15 to 1 - 1e-15 at 512^2 (absorbed adds, nfb_sampler.h; before the fix these maps overflowed the segment table);
  * n = 1, and n = H * W (every pixel of a 32 x 64 frame, through numpy's many late rounds);
  * frames with H != W both ways: pixel (k % H, k // H) as the reference indexes its coords, rays against the oracle's ray
    bundle, target and background gathered at that pixel;
  * K = NFB_MAX_STEP_IMAGES = 64 with repeats, the last draw slice ending the buffer;
  * the documented rejection of an index out of range, a map of another shape, a box outside the frame and a map of more
    runs than the table holds (NaN rows, -1 indices, frame slot K, state 0, shortfall untouched, other blocks unaffected);
  * the shortfall counter over several graph replays, and the first-occurrence scratch left clean after short and wide calls.
    (This found capture_images keeping its warm-up selection's shortfall in FusedTrainer.shortfall; it no longer does.)

Each of these defects, planted once in sample_images_kernel / gather_pixels, failed this file on an H100 (none was kept):
  * pixel (k // W, k % W) instead of (k % H, k // H) when H != W: test_frames_with_h_ne_w, both shapes (pixel_rc);
  * the rejection path writing frame 0 instead of K: test_rejected_images_follow_the_documented_path (frame_index);
  * shortfall assigned instead of accumulated: test_rejected_images_follow_the_documented_path (the untouched counter of
    the good blocks reads 0) and test_graph_replays_accumulate_the_shortfall ([472, 750] after three replays, not
    [1358, 2223]).
The file runs in about 13 s."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import nerface_oracle as O
from test_post_gpu import numpy_choice_with_recorded_draws
from test_train_images_gpu import batch_buffers, make_model

pytestmark = pytest.mark.gpu
NFB_ERR_UNSUPPORTED = 2
P_VALUES = [1e-15, 1e-12, 1e-6, 0.5, 0.9, 1 - 1e-6, 1 - 1e-12, 1 - 1e-15]
ROWS = ("ray_origins", "ray_directions", "target", "background", "pixel_rc", "indices", "frame_index")


@pytest.fixture(scope="module")
def E(built_lib):
    import nerf
    from nerf import _capi, _engine, fused_train, ray_sampler
    return SimpleNamespace(nerf=nerf, capi=_capi, engine=_engine, fused_train=fused_train, rs=ray_sampler, dev=torch.device("cuda", 0))


def make_data(E, H, W, bboxs, p=0.9, seed=0):
    frs = [O.synthetic_frame(seed + i, H, W) for i in range(len(bboxs))]
    g = torch.Generator().manual_seed(seed + 100)
    images = torch.rand(len(bboxs), H, W, 3, generator=g)
    poses = torch.stack([f["pose"][:3, :4].reshape(-1) for f in frs])
    exprs = torch.stack([f["expr"] for f in frs])
    data = E.rs.TrainImages(images.to(E.dev), poses, exprs, bboxs, frs[0]["intrinsics"], background=frs[0]["bg"], p=p, device=E.dev)
    return data, frs, images


def draw_slices(flats, n, rounds, seed):
    """Slice k of a [K, rounds * n] buffer starts with the draws numpy's choice consumed on flats[k] (None: none) and continues
    with other uniforms, so a slice read from the wrong offset selects other pixels.  Returns (buffer, [(indices, state)])."""
    buf = np.random.default_rng(seed).random((len(flats), rounds * n))
    want = []
    for k, flat in enumerate(flats):
        if flat is None:
            want.append(None)
            continue
        idx, draws = numpy_choice_with_recorded_draws(flat.size, n, flat, seed + k)
        d = np.concatenate(draws)
        assert len(draws) <= rounds
        buf[k, :d.size] = d
        want.append((idx, [n, len(draws), d.size]))
    return buf, want


def batched(E, eng, data, ids, n, draws, rounds, table, out=None):
    out = out if out is not None else batch_buffers(E.dev, len(ids), n)
    eng.sample_images(data, torch.tensor(ids, dtype=torch.int32, device=E.dev), n, draws, rounds, table, out)
    torch.cuda.synchronize()
    return out


def single(E, H, W, bbox, p, n, draws, rounds, frame, image, background):
    """nfb_sample_rays with every gather, for the same image, pose and background as a TrainImages entry."""
    smp = E.rs.RaySampler(H, W, [bbox], p=p, size=n, device=E.dev)
    out = smp.sample(0, draws=draws, pose=frame["pose"], intrinsics=frame["intrinsics"], image=image, background=background,
                     max_rounds=rounds)
    torch.cuda.synchronize()
    return out


def check_block(out, k, n, want, ref=None):
    """Block k of a batched call: numpy's indices and state; with ref (nfb_sample_rays on the same slice) its gathers bitwise."""
    s = slice(k * n, (k + 1) * n)
    idx, state = want
    assert out["state"][k].cpu().tolist() == state, (k, out["state"][k].tolist(), state)
    assert np.array_equal(out["indices"][s].cpu().numpy(), idx), k
    if ref is not None:
        assert ref["state"].cpu().tolist() == state and np.array_equal(ref["indices"].cpu().numpy(), idx), k
        for name in ("pixel_rc", "ray_origins", "ray_directions", "target", "background"):
            if name in ref:
                assert torch.equal(out[name][s], ref[name]), (k, name)
        assert (out["frame_index"][s] == k).all(), k


@pytest.mark.parametrize("p", P_VALUES)
def test_p_sweep_matches_numpy_choice(E, p):
    """512^2, n = 2048, the reference's box and a wider one (both >= 4096 pixels, so numpy needs few rounds at p near 1)."""
    H = W = 512
    n, rounds = 2048, 16
    bboxs = [(150, 400, 128, 380), (40, 300, 60, 500)]
    data, frs, images = make_data(E, H, W, bboxs, p)
    flats = [E.rs.importance_map(H, W, bb, p)[1] for bb in bboxs]
    buf, want = draw_slices(flats, n, rounds, seed=11 + P_VALUES.index(p))
    draws = torch.from_numpy(buf.reshape(-1)).to(E.dev)
    table = torch.randn(2, 32, device=E.dev)
    out = batched(E, E.engine.renderer_for(E.dev), data, [0, 1], n, draws, rounds, table)
    for k in range(2):
        ref = single(E, H, W, bboxs[k], p, n, draws[k * rounds * n:(k + 1) * rounds * n], rounds, frs[k], images[k], frs[0]["bg"])
        check_block(out, k, n, want[k], ref)
    assert int(out["shortfall"].abs().sum()) == 0


@pytest.mark.parametrize("n", [1, 32 * 64])
def test_one_ray_and_every_pixel(E, n):
    """n = 1 (one draw, one round) and n = H * W = 2048 (every pixel: numpy's late rounds zero all but a few entries); the draw
    buffer holds exactly the rounds numpy ran."""
    H, W, bbox = 32, 64, (4, 20, 10, 40)
    data, frs, images = make_data(E, H, W, [bbox])
    flat = E.rs.importance_map(H, W, bbox, 0.9)[1]
    idx, draws = numpy_choice_with_recorded_draws(H * W, n, flat, 5)
    rounds = len(draws)
    buf, want = draw_slices([flat], n, rounds, seed=5)
    if n == H * W:
        assert rounds > 4 and sorted(idx.tolist()) == list(range(H * W))
    d = torch.from_numpy(buf.reshape(-1)).to(E.dev)
    out = batched(E, E.engine.renderer_for(E.dev), data, [0], n, d, rounds, torch.randn(1, 32, device=E.dev))
    check_block(out, 0, n, want[0], single(E, H, W, bbox, 0.9, n, d, rounds, frs[0], images[0], frs[0]["bg"]))


@pytest.mark.parametrize("H,W,bbox", [(96, 160, (20, 70, 30, 130)), (160, 96, (30, 130, 20, 70))])
def test_frames_with_h_ne_w(E, H, W, bbox):
    """Flat index k addresses the probability map row-major but the pixel (k % H, k // H) (train_transformed_rays.py:303-331), in
    range for any H and W: pixel_rc, rays against the oracle's ray bundle, target and background at that pixel, both entries."""
    n, rounds = 2048, 16
    data, frs, images = make_data(E, H, W, [bbox])
    flat = E.rs.importance_map(H, W, bbox, 0.9)[1]
    buf, want = draw_slices([flat], n, rounds, seed=H)
    d = torch.from_numpy(buf.reshape(-1)).to(E.dev)
    out = batched(E, E.engine.renderer_for(E.dev), data, [0], n, d, rounds, torch.randn(1, 32, device=E.dev))
    ref = single(E, H, W, bbox, 0.9, n, d, rounds, frs[0], images[0], frs[0]["bg"])
    idx = want[0][0]
    rows, cols = idx % H, idx // H
    ro, rd = O.ray_bundle(H, W, frs[0]["intrinsics"], frs[0]["pose"])
    for got in (out, ref):
        assert np.array_equal(got["pixel_rc"].cpu().numpy(), np.stack((rows, cols), axis=1))
        assert torch.equal(got["ray_directions"].cpu(), rd[rows, cols]) and torch.equal(got["ray_origins"].cpu(), ro[rows, cols])
        assert torch.equal(got["target"].cpu(), images[0][rows, cols]) and torch.equal(got["background"].cpu(), frs[0]["bg"][rows, cols])
    check_block(out, 0, n, want[0], ref)


def test_sixty_four_images_with_repeats(E):
    """K = NFB_MAX_STEP_IMAGES at 512^2, n = 2048, five images drawn with repeats: block k equals nfb_sample_rays on draw slice k
    and numpy's choice; the draws are exactly K * max_rounds * n doubles, so the last block reads the buffer's last slice."""
    H = W = 512
    n, rounds, K = 2048, 8, E.capi.NFB_MAX_STEP_IMAGES
    bboxs = [(150, 400, 128, 380), (40, 300, 60, 500), (0, 512, 0, 512), (200, 260, 10, 400), (0, 1, 511, 512)]
    data, frs, images = make_data(E, H, W, bboxs, seed=3)
    ids = np.random.default_rng(2).integers(0, len(bboxs), K).tolist()
    assert len(set(ids)) == len(bboxs)
    flats = [E.rs.importance_map(H, W, bb, 0.9)[1] for bb in bboxs]
    buf, want = draw_slices([flats[i] for i in ids], n, rounds, seed=40)
    draws = torch.from_numpy(buf.reshape(-1)).to(E.dev)
    assert draws.numel() == K * rounds * n
    table = torch.randn(len(bboxs), 32, device=E.dev)
    out = batched(E, E.engine.renderer_for(E.dev), data, ids, n, draws, rounds, table)
    for k, i in enumerate(ids):
        ref = single(E, H, W, bboxs[i], 0.9, n, draws[k * rounds * n:(k + 1) * rounds * n], rounds, frs[i], images[i], frs[0]["bg"])
        check_block(out, k, n, want[k], ref)
        assert torch.equal(out["expressions"][k], data.expressions[i]) and torch.equal(out["latents"][k], table[i])
    assert int(out["shortfall"].abs().sum()) == 0


def test_rejected_images_follow_the_documented_path(E):
    """include/nfb.h, nfb_sample_rays_images: an index outside [0, n_images), a map of another shape, a box outside the frame
    (either side) and a map of more runs than the table holds read nothing: NaN rays, target, background, expression and latent
    rows, -1 indices and pixel_rc, frame slot K, state 0, shortfall untouched; the other blocks are bitwise those of a launch
    without the rejected images.  nfb_sample_rays refuses the 4,097-run map."""
    H, W, n, rounds = 2048, 8, 256, 8
    bboxs = [(100, 300, 2, 6), (0, 64, 0, 8), (5, 50, 1, 3), (10, 20, 2, 6), (10, 20, 2, 6), (0, 2048, 2, 6)]
    data, frs, images = make_data(E, H, W, bboxs, seed=7)
    maps = [E.rs.importance_map(H, W, bb, 0.9)[0] for bb in bboxs]
    maps[2] = E.rs.importance_map(H, 4, bboxs[2], 0.9)[0]  # another shape
    maps[3].bbox[3] = W + 1                                  # past the right edge
    maps[4].bbox[0] = -1                                     # above the top
    data.maps.copy_(torch.frombuffer(bytearray(bytes((E.capi.NfbRayMap * len(maps))(*maps))), dtype=torch.uint8))
    ids = [0, -1, 2, 1, len(bboxs), 3, 4, 5, 0]
    good = [k for k, i in enumerate(ids) if i in (0, 1)]
    K = len(ids)
    flats = [E.rs.importance_map(H, W, bboxs[i], 0.9)[1] if i in (0, 1) else None for i in ids]
    buf, want = draw_slices(flats, n, rounds, seed=70)
    draws = torch.from_numpy(buf.reshape(-1)).to(E.dev)
    table = torch.randn(len(bboxs), 32, device=E.dev)
    eng = E.engine.renderer_for(E.dev)
    out = batch_buffers(E.dev, K, n)
    shortfall0 = torch.arange(K, device=E.dev, dtype=torch.int64) * 10 + 3
    out["shortfall"].copy_(shortfall0)
    batched(E, eng, data, ids, n, draws, rounds, table, out)
    ctrl = batched(E, eng, data, [i if i in (0, 1) else 0 for i in ids], n, draws, rounds, table)
    assert torch.equal(out["shortfall"], shortfall0)
    for k in range(K):
        s = slice(k * n, (k + 1) * n)
        if k in good:
            check_block(out, k, n, want[k])
            for name in ROWS:
                assert torch.equal(out[name][s], ctrl[name][s]), (k, name)
            assert torch.equal(out["expressions"][k], ctrl["expressions"][k]) and torch.equal(out["latents"][k], ctrl["latents"][k])
            continue
        for name in ("ray_origins", "ray_directions", "target", "background"):
            assert torch.isnan(out[name][s]).all(), (k, ids[k], name)
        assert torch.isnan(out["expressions"][k]).all() and torch.isnan(out["latents"][k]).all(), (k, ids[k])
        assert (out["indices"][s] == -1).all() and (out["pixel_rc"][s] == -1).all(), (k, ids[k])
        assert (out["frame_index"][s] == K).all(), (k, ids[k])
        assert out["state"][k].tolist() == [0, 0, 0], (k, ids[k])
    idx, st = torch.empty(n, dtype=torch.int64, device=E.dev), torch.zeros(3, dtype=torch.int32, device=E.dev)
    rc = E.capi.lib.nfb_sample_rays(eng._h, C.byref(maps[5]), C.c_void_p(draws.data_ptr()), n, rounds, C.c_void_p(idx.data_ptr()),
                                    C.c_void_p(st.data_ptr()), None, E.engine._stream())
    assert rc == NFB_ERR_UNSUPPORTED


def test_graph_replays_accumulate_the_shortfall(E):
    """A captured step with one round of draws over a 12-pixel box holding 90 % of the mass comes up short every replay:
    capture leaves the counter as it was (its warm-up selection is not a step), each replay adds n - n_found (the sum of
    eager samplings of the same draws), and the eager step raises."""
    bboxs = [(10, 14, 12, 15), (10, 50, 12, 44)]
    data, frs, images = make_data(E, 64, 64, bboxs)
    ids, n, replays = [0, 1], 2048, 3
    models = [make_model(E.nerf, O.random_init_params(s), E.dev) for s in (100, 101)]
    tr = E.fused_train.FusedTrainer(*models, n_latent=2, num_coarse=32, num_fine=32)
    tr.capture_images(data, 2, n, max_rounds=1, device_draws=False)
    assert int(tr.shortfall.abs().sum()) == 0
    g = torch.Generator(device=E.dev).manual_seed(9)
    draws = [torch.rand(2 * n, dtype=torch.float64, device=E.dev, generator=g) for _ in range(replays)]
    eng = E.engine.Renderer(E.dev)  # eager samplings on a handle of their own: the graph's buffers stay as captured
    want = torch.zeros(2, dtype=torch.int64)
    for d in draws:
        found = batched(E, eng, data, ids, n, d, 1, torch.zeros(2, 32, device=E.dev))["state"][:, 0].cpu().long()
        want += n - found
    for d in draws:
        tr.step_images_graph(ids, draws=d)
    torch.cuda.synchronize()
    assert int(want.min()) > 0 and torch.equal(tr.shortfall[:2].cpu(), want), (tr.shortfall[:2].tolist(), want.tolist())
    with pytest.raises(RuntimeError, match="fewer than"):
        tr.step_images(data, ids, n, draws=draws[0], max_rounds=1)


def test_scratch_is_clean_after_short_and_wide_calls(E):
    """The first-occurrence table is all INT_MAX between calls: after a K = 64 call and after a short selection (on another frame
    size, over the same scratch), a call equals the same call on a fresh handle."""
    eng = E.engine.Renderer(E.dev)
    big, _, _ = make_data(E, 512, 512, [(150, 400, 128, 380), (40, 300, 60, 500), (0, 512, 0, 512)], seed=20)
    tight, _, _ = make_data(E, 64, 64, [(10, 14, 12, 15), (10, 50, 12, 44)], seed=30)
    n = 2048
    g = torch.Generator(device=E.dev).manual_seed(17)
    table = torch.randn(3, 32, device=E.dev)
    probe_draws = torch.rand(4 * 4 * n, dtype=torch.float64, device=E.dev, generator=g)
    wide_draws = torch.rand(64 * 8 * n, dtype=torch.float64, device=E.dev, generator=g)
    probe = lambda h: batched(E, h, big, [2, 0, 1, 0], n, probe_draws, 4, table)  # noqa: E731
    wide = lambda: batched(E, eng, big, [k % 3 for k in range(64)], n, wide_draws, 8, table)  # noqa: E731
    want = probe(E.engine.Renderer(E.dev))
    wide()
    after_wide = probe(eng)
    short = batched(E, eng, tight, [0, 1], n, torch.rand(2 * n, dtype=torch.float64, device=E.dev, generator=g), 1, table)
    assert int(short["state"][0, 0]) < n
    after_short = probe(eng)
    for name, t in want.items():
        if t is not None:
            assert torch.equal(after_wide[name], t) and torch.equal(after_short[name], t), name
