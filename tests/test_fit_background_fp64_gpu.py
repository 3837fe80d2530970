"""The fitting step (nfb_fit_rows_grad, nerf.FusedFitter) and the learned-background step (nfb_background_rows_grad,
FusedTrainer(background=, background_loss=)) against float64 end to end, on frames that are not square (48x80, 80x48 and 37x64)
with fx != fy and principal points off the centre (INTR: fx 61.3, fy 47.9, cx0 0.47, cy0 0.53), so that a swap of fx and fy, of
width and height or of H and W anywhere in the path changes the result; the importance boxes reach the last row and the last
column.
  (a) rows           nfb_fit_rows_grad bit for bit test_fit_cpu.pose_rows_fp32 on real nfb_sample_rays_images batches (repeats,
                     n = 300: two rays for some of the 256 threads); on an image with an identity rotation the sampler's
                     ray_directions[:, :2] equal camera_dirs bit for bit.  nfb_background_rows_grad on an [H,W,3] table bit for
                     bit background_rows_fp32, with and without the loss term, added onto a nonzero table and from zero (then
                     within gamma(2 hits) of float64), rays in the last row and the last column among them.
  (b) reference      reference_step: a float64 autograd step independent of the library.  The step's own pixel_rc, its noise
                     (fused_train._draw_noise redrawn under the step's seed) and its saved depths (train_debug); rays rebuilt from
                     float64 pose rows, o = t, d = R ((col - W cx0) / fx, -(row - H cy0) / fy, -1); torch_reference.
                     render_at_depths(per_ray_cond=True) on float64 copies of both networks, with float64 expression, latent and
                     background leaves; loss = mse(rgb_c, t) + mse(rgb_f, t) + (latent_reg / K) sum_k ||l_k|| + w mean(w_last
                     ||bg - t||^2), as train_transformed_rays.py:355-389 forms it.  Targets and background colours are gathered
                     from the images and tables at pixel_rc, not taken from the sampler.
  (c) end to end     FusedFitter.gradients in all seven fitted-table combinations at K = 1, 3 (with a repeat) and 8, 128 rays per
                     image (one reference per case: batch, noise and depths are bitwise the same in every combination; tables not
                     fitted stay exactly zero); FusedTrainer step gradients at K = 1 (single-frame kernels; the regulariser is
                     Adam's there, so the reference leaves it out) and K = 3 with a repeat, background_loss 0, 0.001 and 1.0.
                     Fast, exact and exact-grad throughout, and the bucket's background rows bit for bit background_rows_fp32 of
                     the step's own per-ray gradients (the FusedTrainer call site).
  (d) over budget    NFB_TRAIN_MEM_MB=48 (about 32 rays per chunk): the chunked backward with the background input gradient
                     and the w_last output gradient, against the float64 step at the depths of the same step within the budget.
Pose and background rows are sums over rays whose terms cancel, so each component is bounded relative to the sum of |float64
per-ray term| (pose: (dd cx, dd cy, -dd, do) from the reference's per-ray ray gradients; background: the reference's per-ray
background gradient), and by the relative L2 over the table.  Expression and latent rows, and the network parameters, are held
by max and L2 relative to the table or tensor (test_backward_fp64_gpu.errors).  The regulariser's share of a latent row,
(latent_reg / K) l / ||l||, is 14 to 21 times the render's in the fitting cases and 1,800 times in the unsupervised K = 3
trainer cases (max over the table), so the render share (both sides minus the float64 regulariser) is checked on its own too.

BOUNDS, from measurements on an NVIDIA H100 80GB HBM3 at a 700 W power limit (CUDA 12.9), about 2.5 times the worst case over
every case of the file, (max, L2), fast / exact / exact-grad.  The starting points were the existing end-to-end bounds: TOL
(dense 2048-ray parameter gradients, exact (5e-3, 2e-3), fast (4e-2, 3e-2)), PROBE_TOL (single rays), IN_TOL and E2E_IN_TOL
(per-ray input gradients, fast good to about 0.16 max).  The parameters of these 128- and 384-ray steps land between TOL and
PROBE_TOL; the rows, sums over 128 rays or more, land far below the per-ray input bounds, so they get bounds of their own:
  pose rows         worst 8.5e-3 / 3.9e-3, 7.8e-4 / 4.8e-4, 7.9e-4 / 4.9e-4 (K = 8)       -> (2e-2, 1e-2), (2e-3, 1.5e-3) x 2
  background rows   worst 2.3e-3 / 2.3e-6, 1.1e-3 / 1.1e-6, 1.1e-3 / 1.1e-6               -> (6e-3, 1e-5), (3e-3, 5e-6) x 2
                    (the per-ray background gradient is w_last times the colour gradient, from the FP32 forward; the max comes
                    from a one-ray pixel whose w_last is small)
  expression        worst 9.5e-4 / 9.9e-4, 3.7e-4 / 4.3e-4, 8.5e-5 / 9.0e-5               -> (3e-3, 3e-3), (1e-3, 1.2e-3), (2.5e-4, 2.5e-4)
  latent            worst 1.2e-2 / 9.6e-3, 1.2e-3 / 1.1e-3, 1.0e-3 / 1.0e-3 (trainer, K = 1) -> (3e-2, 2.5e-2), (3e-3, 3e-3) x 2
                    render share: the same worst cases (the K = 1 trainer's rows carry no regulariser), 2.8e-4 / 3.0e-4 exact
                    at K = 3 -> the latent bounds
  parameters        worst 3.9e-2 / 2.4e-2, 1.2e-2 / 2.9e-3, 1.2e-2 / 2.8e-3 (K = 1)      -> (8e-2, 5e-2), (3e-2, 7.5e-3) x 2
The fast-mode pose bound, 2e-2 of the sum of |term|, stays meaningful: the smallest planted defect below moves rows by 0.19.
The file takes about 20 s on one H100.

Planted defects, each built once into a library or a package of its own and run against this file and against
test_fit_gpu.py + test_train_background_gpu.py (60 tests):
  1. fit_pose_slots_kernel passing (fy, fx) to camera_dir: here 12 of 36 fail, test_fit_rows_on_non_square_frames at every
     geometry (bitwise) and test_fit_gradients_against_float64 in all 9 cases (pose rows at 0.19-0.24 of the sum of |term|).
     The two files: all 60 pass.
  2. nfb_fit_rows_grad forming wcx from the height and hcy from the width: here the same 12 fail (pose rows at 1.4-1.6).  The
     two files: all 60 pass.
  3. FusedTrainer calling background_rows_grad with (W, H): here 21 fail, every trainer and over-budget case (the call-site
     check, bitwise).  The two files: all 60 pass (their tables are square).
  4. Renderer.backward_into dropping the w_last output gradient: here 15 fail, every supervised case, w = 0.001 included (the
     worst parameter tensor off by 0.09-0.16 of its max at w = 0.001, by 1.0 at w = 1).  test_train_background_gpu.py fails 4
     of its supervised cases too: its autograd side runs Renderer.backward, which this defect leaves alone.
  5. _engine._out_grads, which backward and backward_into share, dropping the w_last output gradient: here the same 15 fail.
     The two files: all 60 pass, since their autograd side loses the gradient as the fused step does.
"""
import types

import numpy as np
import pytest
import torch

import nerface_oracle as O
import torch_reference as TR
from test_backward_fp64_gpu import errors
from test_backward_gpu import dev_tensor
from test_fit_cpu import camera_dirs, pose_rows_fp32
from test_train_background_cpu import background_rows_fp32, pixel_keys
from test_train_background_gpu import check_f64

pytestmark = pytest.mark.gpu

NEAR, FAR = 0.2, 0.8
INTR = [61.3, 47.9, 0.47, 0.53]  # fx != fy, W cx0 != H cy0, neither centre at 0.5
GEOMS = {"48x80": (48, 80), "80x48": (80, 48), "37x64": (37, 64)}
PRECS = ["fast", "exact", "exact_grad"]
COMBOS = [("pose",), ("expression",), ("latent",), ("pose", "expression"), ("pose", "latent"), ("expression", "latent"),
          ("pose", "expression", "latent")]
LATENT_REG = 0.005
N_RAYS = 128    # rays per image of the end-to-end steps
ROUNDS = 16

# (max, L2) per quantity and precision, about 2.5 times the measured worst case (module docstring).  Pose and background rows:
# max |got - ref| / sum |float64 per-ray term| per component, and the relative L2 over the table.  Expression, latent and the
# network parameters: max |got - ref| / max |ref| and the relative L2, per table or tensor.
BOUNDS = {
    "pose": {"fast": (2e-2, 1e-2), "exact": (2e-3, 1.5e-3), "exact_grad": (2e-3, 1.5e-3)},
    "background": {"fast": (6e-3, 1e-5), "exact": (3e-3, 5e-6), "exact_grad": (3e-3, 5e-6)},
    "expression": {"fast": (3e-3, 3e-3), "exact": (1e-3, 1.2e-3), "exact_grad": (2.5e-4, 2.5e-4)},
    "latent": {"fast": (3e-2, 2.5e-2), "exact": (3e-3, 3e-3), "exact_grad": (3e-3, 3e-3)},
    "parameters": {"fast": (8e-2, 5e-2), "exact": (3e-2, 7.5e-3), "exact_grad": (3e-2, 7.5e-3)},
}


@pytest.fixture(scope="module")
def env(built_lib):
    import nerf
    from nerf import _engine, fused_train, ray_sampler
    return types.SimpleNamespace(nerf=nerf, engine=_engine, ft=fused_train, rs=ray_sampler, dev=torch.device("cuda", 0))


@pytest.fixture(autouse=True)
def own_renderer(env, monkeypatch):
    """A renderer handle of the test's own: an exact-grad step adds a launch to every later re-pack on its handle, which other
    test files count."""
    eng = env.engine.Renderer(env.dev)
    monkeypatch.setitem(env.engine._renderers, ("cuda", env.dev.index), eng)
    yield eng
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------- the scene
def boxes(H, W, n):
    """Importance boxes, cycled over n images: most reach the last row or the last column, one holds the whole frame; each
    holds at least a quarter of the frame, so that 16 rounds of draws find a few hundred distinct pixels."""
    b = [(H // 3, H, W // 2, W), (0, H, 0, W), (2, H - 5, 3, W), (H // 2, H, 0, W // 2), (1, H // 2, W // 3, W)]
    return [b[i % len(b)] for i in range(n)]


def scene(H, W, n_img, seed):
    frs = [O.synthetic_frame(seed + i, H, W) for i in range(n_img)]
    g = torch.Generator().manual_seed(seed + 100)
    return types.SimpleNamespace(
        H=H, W=W, n=n_img, bg=frs[0]["bg"], images=torch.rand(n_img, H, W, 3, generator=g),
        poses=torch.stack([f["pose"][:3, :4].reshape(-1) for f in frs]), exprs=torch.stack([f["expr"] for f in frs]),
        lats=torch.randn(n_img, 32, generator=g) * 0.1, boxes=boxes(H, W, n_img))


def train_images(env, sc, background=None):
    return env.rs.TrainImages(sc.images.to(env.dev), sc.poses, sc.exprs, sc.boxes, INTR, background=background, device=env.dev)


def make_model(env, seed):
    m = env.nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True,
                                                            include_input_dir=False)
    m.load_state_dict(O.random_init_params(seed))
    return m.to(env.dev)


def draws_for(env, k, n, seed):
    return torch.rand(k * ROUNDS * n, dtype=torch.float64, device=env.dev, generator=torch.Generator(device=env.dev).manual_seed(seed))


def sample(env, eng, data, ids, n, seed, **extra):
    """One nfb_sample_rays_images call of K = len(ids) slots; every slot must find its n pixels."""
    N = len(ids) * n
    sb = dict(pixel_rc=torch.full((N, 2), -7, dtype=torch.int32, device=env.dev),
              state=torch.zeros(len(ids), 3, dtype=torch.int32, device=env.dev))
    sb.update({name: torch.zeros(N, 3, device=env.dev) for name in extra})
    eng.sample_images(data, torch.tensor(ids, dtype=torch.int32, device=env.dev), n, draws_for(env, len(ids), n, seed), ROUNDS,
                      torch.zeros(data.n_images, 32, device=env.dev), sb)
    torch.cuda.synchronize()
    assert bool((sb["state"][:, 0] == n).all())
    return sb


def reaches_the_edges(rc, H, W):
    return bool((rc[:, 0] == H - 1).any()) and bool((rc[:, 1] == W - 1).any())


# ---------------------------------------------------------------------------------------------------------------- (a) rows
@pytest.mark.parametrize("geom", list(GEOMS))
def test_fit_rows_on_non_square_frames(env, own_renderer, geom):
    """nfb_fit_rows_grad bit for bit pose_rows_fp32 (with the frame's own H and W) on a real sampler batch, repeats included;
    image 0 has an identity rotation, so the sampler's ray directions are (cx, cy) of camera_dirs bit for bit."""
    H, W = GEOMS[geom]
    eng, dev = own_renderer, env.dev
    sc = scene(H, W, 5, seed=7)
    sc.poses[0] = torch.tensor([1.0, 0, 0, 0.1, 0, 1.0, 0, -0.2, 0, 0, 1.0, 0.7])
    data = train_images(env, sc)
    ids, n = [0, 3, 1, 0, 4, 2], 300
    K, N = len(ids), len(ids) * n
    sb = sample(env, eng, data, ids, n, seed=H * W, ray_directions=True)
    rc = sb["pixel_rc"].cpu().numpy()
    assert reaches_the_edges(rc, H, W)
    g = torch.Generator().manual_seed(H + W)
    scale = 10.0 ** torch.randint(-4, 1, (N, 1), generator=g).float()
    go, gd = torch.randn(N, 3, generator=g) * scale, torch.randn(N, 3, generator=g) * scale
    gexpr = torch.randn(K, 76, generator=g)
    P0, E0 = torch.randn(5, 12, generator=g), torch.randn(5, 76, generator=g)
    P, Ex = P0.clone().to(dev), E0.clone().to(dev)
    eng.fit_rows_grad(data, torch.tensor(ids, dtype=torch.int32, device=dev), n, sb["pixel_rc"], go.to(dev), gd.to(dev), P,
                      gexpr.to(dev), Ex)
    torch.cuda.synchronize()
    want_p, want_e, _ = pose_rows_fp32(ids, n, 5, rc, go.numpy(), gd.numpy(), INTR, H, W, P0.numpy(), gexpr.numpy(), E0.numpy())
    assert np.array_equal(P.cpu().numpy(), want_p) and np.array_equal(Ex.cpu().numpy(), want_e)
    cx, cy = camera_dirs(rc, INTR[0], INTR[1], np.float32(W * INTR[2]), np.float32(H * INTR[3]))
    rd = sb["ray_directions"].cpu().numpy()
    for k in (0, 3):
        s = slice(k * n, (k + 1) * n)
        assert np.array_equal(rd[s, 0], cx[s]) and np.array_equal(rd[s, 1], cy[s]), k


@pytest.mark.parametrize("geom", list(GEOMS))
def test_background_rows_on_non_square_tables(env, own_renderer, geom):
    """nfb_background_rows_grad on an [H,W,3] table bit for bit background_rows_fp32 (added onto a nonzero table), with and without
    the loss term, pixels of the last row and the last column among the rays; from zero within gamma(2 hits) of float64."""
    H, W = GEOMS[geom]
    eng, dev = own_renderer, env.dev
    sc = scene(H, W, 4, seed=11)
    data = train_images(env, sc)
    ids, n = [1, 3, 1, 0, 2, 1], 300
    N = len(ids) * n
    sb = sample(env, eng, data, ids, n, seed=3 * H + W)
    rc = sb["pixel_rc"].cpu().numpy()
    assert reaches_the_edges(rc, H, W)
    rng = np.random.default_rng(H * W)
    gr = (rng.standard_normal((N, 3)) * 10.0 ** rng.integers(-4, 1, (N, 1))).astype(np.float32)
    gl = (rng.standard_normal((N, 3)) * 1e-2).astype(np.float32)
    t0 = torch.randn(H, W, 3, generator=torch.Generator().manual_seed(H)) * 1e-3
    for gl_ in (None, gl):
        for table0 in (t0, torch.zeros(H, W, 3)):
            t = table0.to(dev)
            eng.background_rows_grad(sb["pixel_rc"], H, W, torch.from_numpy(gr).to(dev),
                                     None if gl_ is None else torch.from_numpy(gl_).to(dev), t)
            torch.cuda.synchronize()
            got = t.reshape(-1, 3).cpu().numpy()
            assert np.array_equal(got, background_rows_fp32(rc, H, W, gr, gl_, table0.numpy())), (gl_ is None)
        check_f64(got, rc, H, W, gr, gl_)
        keys = pixel_keys(rc, H, W)
        assert got[keys[rc[:, 0] == H - 1]].any() and got[keys[rc[:, 1] == W - 1]].any()


# ---------------------------------------------------------------------------------------------------------------- (b) float64
def reference_step(mc, mf, sc, ids, n, pixel_rc, noise, noise_std, z_c, z_f, bg_table=None, learn_bg=False, bg_weight=0.0,
                   latent_reg=0.0, want_params=False):
    """One step's loss in float64 autograd, independent of the library: rays rebuilt from float64 pose rows at pixel_rc,
    torch_reference.render_at_depths at the kernel's depths and noise, every ray conditioned on its image's expression and latent
    rows, the background table gathered at pixel_rc; loss = mse(rgb_c, t) + mse(rgb_f, t) + (latent_reg / K) sum_k ||l_k||
    + bg_weight * mean(w_last ||bg - t||^2) (train_transformed_rays.py:355-389).  Returns the table gradients, the parameter
    gradients (want_params) and the per-ray float64 gradients of the ray origins, directions and background colours."""
    dev = z_c.device
    f64 = lambda t: t.detach().to(dev, torch.float64)  # noqa: E731
    leaf = lambda t: f64(t).clone().requires_grad_(True)  # noqa: E731
    net = lambda m: None if m is None else {k: (leaf(v) if want_params else f64(v)) for k, v in m.named_parameters()}  # noqa: E731
    pc, pf = net(mc), net(mf)
    P, X, L = leaf(sc.poses), leaf(sc.exprs), leaf(sc.lats)
    k, N = len(ids), len(ids) * n
    img = torch.tensor(ids, device=dev).repeat_interleave(n)
    rc = pixel_rc.to(dev).long()
    fx, fy, cx0, cy0 = INTR
    cam = torch.stack(((rc[:, 1].double() - sc.W * cx0) / fx, -(rc[:, 0].double() - sc.H * cy0) / fy,
                       torch.full((N,), -1.0, dtype=torch.float64, device=dev)), 1)
    pose = P.view(-1, 3, 4)[img]
    ro = pose[:, :, 3]
    rd = (pose[:, :, :3] @ cam[:, :, None])[:, :, 0]
    ro.retain_grad()
    rd.retain_grad()
    B = leaf(bg_table) if learn_bg else (f64(bg_table) if bg_table is not None else None)
    bg = B[rc[:, 0], rc[:, 1]] if B is not None else None
    if learn_bg:
        bg.retain_grad()
    rays = torch.cat((ro, rd, torch.full((N, 1), NEAR, dtype=torch.float64, device=dev),
                      torch.full((N, 1), FAR, dtype=torch.float64, device=dev)), 1)
    nz = {key: f64(noise[key]) for key in ("n_c", "n_f") if noise and noise.get(key) is not None}
    out = TR.render_at_depths(rays, pc, pf, X[img], L[img], f64(z_c), f64(z_f) if z_f is not None else None, NEAR, FAR, noise_std, nz,
                              False, bg, per_ray_cond=True)
    t = f64(sc.images.to(dev)[img, rc[:, 0], rc[:, 1]])
    loss = ((out[0] - t) ** 2).mean()
    if pf is not None:
        loss = loss + ((out[3] - t) ** 2).mean()
    if latent_reg:
        loss = loss + latent_reg / k * sum(L[j].norm() for j in ids)
    if bg_weight:
        loss = loss + bg_weight * (out[6] * ((bg - t) ** 2).sum(1)).mean()
    loss.backward()
    reg = torch.zeros_like(L)  # the regulariser's share of the latent rows, (latent_reg / K) l / ||l|| per slot
    for j in ids:
        reg[j] += latent_reg / k * L[j].detach() / L[j].detach().norm()
    grads = lambda p: None if p is None else [p[q].grad for q in TR.PARAM_ORDER]  # noqa: E731
    return types.SimpleNamespace(pose=P.grad, expression=X.grad, latent=L.grad, latent_reg=reg, background=B.grad if learn_bg else None,
                                 gc=grads(pc) if want_params else None, gf=grads(pf) if want_params else None,
                                 g_ro=ro.grad, g_rd=rd.grad, g_bg=bg.grad if learn_bg else None, cam=cam, img=img, rc=rc)


def saved_depths(eng, N, nc, nf):
    torch.cuda.synchronize()
    d = eng.train_debug()
    return dev_tensor(d.z_coarse, (N, nc)).clone(), dev_tensor(d.z_fine, (N, nc + nf)).clone()


# ---------------------------------------------------------------------------------------------------------------- (c) checks
def check_rows(tag, got, ref, mag, used, tol):
    """A table whose rows are sums over rays: every component of a used row within tol[0] * sum |float64 per-ray term| of
    float64, the relative L2 over the table within tol[1], unused rows exactly zero.  Returns (worst |got - ref| / sum |term|,
    L2)."""
    got, ref = got.double(), ref.double()
    assert bool(torch.isfinite(got).all()), tag
    assert not bool(got[~used].any()), (tag, "a row no ray touched is not zero")
    err = (got - ref).abs()[used]
    ratio = float((err / mag[used].clamp(min=1e-300)).max())
    l2 = float((got - ref)[used].norm() / ref[used].norm())
    assert ratio <= tol[0] and l2 <= tol[1], (tag, ratio, l2)
    return ratio, l2


def check_table(tag, got, ref, used, tol):
    """Rows that are one gradient each (expression, latent): max and L2 relative to the table's float64 rows; unused rows zero."""
    assert bool(torch.isfinite(got).all()), tag
    assert not bool(got[~used].any()), (tag, "a row no ray touched is not zero")
    em, el = errors(got[used], ref[used])
    assert em <= tol[0] and el <= tol[1], (tag, em, el)
    return em, el


def check_latent(tag, got, R, used, prec):
    """The latent rows, and their render share without the regulariser's (latent_reg / K) l / ||l||, which outweighs the
    render's share by orders of magnitude and would hide it: (latent, render share) as (max, L2) each."""
    whole = check_table(f"{tag} latent", got, R.latent, used, BOUNDS["latent"][prec])
    share = check_table(f"{tag} latent render share", got.double() - R.latent_reg, R.latent - R.latent_reg, used, BOUNDS["latent"][prec])
    if bool(R.latent_reg.any()):
        print(f"{tag}: max |regulariser share| / max |render share| of the latent rows "
              f"{float(R.latent_reg.abs().max() / (R.latent - R.latent_reg).abs().max()):.1e}")
    return whole, share


def pose_terms(R):
    """[N,12] float64 per-ray terms of the pose rows: (dd cx, dd cy, -dd, do) per row q of the 3x4 matrix."""
    t = torch.zeros(R.g_rd.shape[0], 12, dtype=torch.float64, device=R.g_rd.device)
    for q in range(3):
        t[:, 4 * q] = R.g_rd[:, q] * R.cam[:, 0]
        t[:, 4 * q + 1] = R.g_rd[:, q] * R.cam[:, 1]
        t[:, 4 * q + 2] = -R.g_rd[:, q]
        t[:, 4 * q + 3] = R.g_ro[:, q]
    return t


def used_rows(ids, n_rows, dev):
    u = torch.zeros(n_rows, dtype=torch.bool, device=dev)
    u[torch.tensor(ids, device=dev)] = True
    return u


FIT_CASES = {"K1_37x64": ([2], (37, 64)), "K3_repeat_80x48": ([2, 0, 2], (80, 48)), "K8_48x80": ([5, 1, 7, 0, 3, 6, 2, 4], (48, 80))}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", list(FIT_CASES))
def test_fit_gradients_against_float64(env, own_renderer, case, prec):
    """FusedFitter.gradients in all seven fitted-table combinations against one float64 reference of the step (the batch, noise
    and depths are the same in every combination): pose rows per component relative to sum |per-ray term| and by relative L2,
    expression and latent rows by max and L2 relative to their table; tables not fitted stay exactly zero."""
    ids, (H, W) = FIT_CASES[case]
    eng, dev, n = own_renderer, env.dev, N_RAYS
    k, N = len(ids), len(ids) * N_RAYS
    sc = scene(H, W, 8, seed=20 + k)
    mc, mf = make_model(env, 100).requires_grad_(False), make_model(env, 101).requires_grad_(False)
    draws = draws_for(env, k, n, seed=30 + k)
    R = first = None
    worst = {}
    for combo in COMBOS:
        fit = env.nerf.FusedFitter(mc, mf, sc.images.to(dev), sc.boxes, INTR, sc.poses, sc.exprs, sc.lats, background=sc.bg.to(dev),
                                   fit=combo, precision=prec, latent_reg=LATENT_REG)
        torch.manual_seed(40 + k)
        fit.gradients(ids, n, draws=draws, max_rounds=ROUNDS)
        z_c, z_f = saved_depths(eng, N, 64, 64)
        rc = fit._last["pixel_rc"].clone()
        if R is None:
            assert reaches_the_edges(rc.cpu(), H, W) or k == 1
            torch.manual_seed(40 + k)
            noise = env.ft._draw_noise(fit.opts, dev, N)
            R = reference_step(mc, mf, sc, ids, n, rc, noise, 0.1, z_c, z_f, bg_table=sc.bg, latent_reg=LATENT_REG)
            mag = torch.zeros(8, 12, dtype=torch.float64, device=dev).index_add_(0, R.img, pose_terms(R).abs())
            used = used_rows(ids, 8, dev)
            first = (rc, z_c, z_f)
        else:  # the same batch, noise and depths: one reference serves every combination
            assert torch.equal(rc, first[0]) and torch.equal(z_c, first[1]) and torch.equal(z_f, first[2]), combo
        tag = f"fit {case} {prec} {'+'.join(combo)}"
        for t in ("pose", "expression", "latent"):
            got = fit._table(fit.grads, t)
            if t not in combo:
                assert not bool(got.any()), (tag, t)
            elif t == "pose":
                r = check_rows(f"{tag} pose", got, R.pose, mag, used, BOUNDS["pose"][prec])
                worst["pose"] = [max(a, b) for a, b in zip(worst.get("pose", (0, 0)), r)]
            elif t == "expression":
                r = check_table(f"{tag} expression", got, R.expression, used, BOUNDS["expression"][prec])
                worst[t] = [max(a, b) for a, b in zip(worst.get(t, (0, 0)), r)]
            else:
                for name, r in zip(("latent", "latent render share"), check_latent(tag, got, R, used, prec)):
                    worst[name] = [max(a, b) for a, b in zip(worst.get(name, (0, 0)), r)]
    print(f"FP64E2E fit {case} {prec}: " + ", ".join(f"{t} {a:.2e} / L2 {b:.2e}" for t, (a, b) in worst.items()))


def learner(env, sc, prec, weight):
    return env.ft.FusedTrainer(make_model(env, 100), make_model(env, 101), n_latent=sc.n, num_coarse=64, num_fine=64, perturb=True,
                               noise_std=0.1, latent_reg=LATENT_REG, latent_codes=sc.lats, precision=prec,
                               background=sc.images.mean(0), background_loss=weight)


def trainer_gradients(env, tr, data, ids, n, seed):
    """The fused step's gradients into tr.grads (no Adam): sample, then _images_gradients under torch seed `seed`."""
    tr._own_engine()
    dv = tr._images_data(data)
    sb = tr._images_buffers(dv, len(ids), n)
    sb["img"].copy_(torch.tensor(ids, dtype=torch.int32))
    tr._images_sample(dv, sb, n, draws_for(env, len(ids), n, seed), ROUNDS)
    torch.manual_seed(seed)
    tr._images_gradients(sb, len(ids), n)
    torch.cuda.synchronize()
    return sb


def check_trainer(tag, tr, sb, R, sc, ids, weight, prec):
    H, W, dev = sc.H, sc.W, tr.dev
    rc = sb["pixel_rc"]
    # the Python call site: the bucket's background rows are nfb_background_rows_grad of the step's own per-ray gradients at (H, W)
    want = background_rows_fp32(rc.cpu().numpy(), H, W, sb["g_bg"].cpu().numpy(), sb["g_bgl"].cpu().numpy() if weight else None)
    assert np.array_equal(tr._bg_grads.reshape(-1, 3).cpu().numpy(), want), tag
    pairs = [(f"{net}/{q}", g, r) for net, gs, rs in (("coarse", tr._gc, R.gc), ("fine", tr._gf, R.gf))
             for q, g, r in zip(TR.PARAM_ORDER, gs, rs) if not q.startswith("layers_dir.3")]
    pm = [0.0, 0.0]
    for name, g, r in pairs:
        assert g is not None and r is not None, (tag, name)
        em, el = errors(g, r)
        pm = [max(pm[0], em), max(pm[1], el)]
    assert pm[0] <= BOUNDS["parameters"][prec][0] and pm[1] <= BOUNDS["parameters"][prec][1], (tag, "parameters", pm)
    lat, share = check_latent(tag, tr._latent_grads(), R, used_rows(ids, sc.n, dev), prec)
    key = torch.from_numpy(pixel_keys(rc.cpu().numpy(), H, W)).to(dev)
    assert bool((key >= 0).all())
    mag = torch.zeros(H * W, 3, dtype=torch.float64, device=dev).index_add_(0, key, R.g_bg.abs())
    hit = torch.zeros(H * W, dtype=torch.bool, device=dev)
    hit[key] = True
    bgr = check_rows(f"{tag} background", tr._bg_grads.reshape(-1, 3), R.background.reshape(-1, 3), mag, hit, BOUNDS["background"][prec])
    print(f"FP64E2E {tag}: parameters {pm[0]:.2e} / L2 {pm[1]:.2e}, latent {lat[0]:.2e} / L2 {lat[1]:.2e}, render share "
          f"{share[0]:.2e} / L2 {share[1]:.2e}, background rows {bgr[0]:.2e} / L2 {bgr[1]:.2e}")


TRAIN_CASES = {"K1_80x48": ([1], (80, 48)), "K3_repeat_48x80": ([2, 0, 2], (48, 80))}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("weight", [0.0, 0.001, 1.0])
@pytest.mark.parametrize("case", list(TRAIN_CASES))
def test_learned_background_step_against_float64(env, case, weight, prec):
    """FusedTrainer(background=, background_loss=weight) step gradients against the float64 step: network parameters, latent
    rows and background rows (K = 1: the single-frame kernels, whose regulariser Adam adds; K >= 2: the multi-frame ones), and the
    bucket's background rows bit for bit the kernel's documented order over the step's own per-ray gradients."""
    ids, (H, W) = TRAIN_CASES[case]
    k, n = len(ids), N_RAYS
    sc = scene(H, W, 3, seed=50 + k)
    data = train_images(env, sc)
    tr = learner(env, sc, prec, weight)
    sb = trainer_gradients(env, tr, data, ids, n, seed=60 + k)
    z_c, z_f = saved_depths(tr.eng, k * n, 64, 64)
    torch.manual_seed(60 + k)
    noise = env.ft._draw_noise(tr.opts, env.dev, k * n)
    R = reference_step(tr.mc, tr.mf, sc, ids, n, sb["pixel_rc"], noise, 0.1, z_c, z_f, bg_table=tr.background, learn_bg=True,
                       bg_weight=weight, latent_reg=LATENT_REG if k >= 2 else 0.0, want_params=True)
    check_trainer(f"train {case} w={weight} {prec}", tr, sb, R, sc, ids, weight, prec)


# ---------------------------------------------------------------------------------------------------------------- (d) budget
@pytest.mark.parametrize("prec", PRECS)
def test_supervised_background_over_the_memory_budget(env, prec, monkeypatch):
    """NFB_TRAIN_MEM_MB=48 (about 32 rays per chunk): the chunked backward with the per-ray background gradient and the w_last
    output gradient, against the float64 step at the depths of the same step within the budget."""
    ids, (H, W), weight = [1, 0, 1], (37, 64), 1.0
    k, n = len(ids), N_RAYS
    sc = scene(H, W, 3, seed=70)
    data = train_images(env, sc)
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "20000")
    one = learner(env, sc, prec, weight)
    sb1 = trainer_gradients(env, one, data, ids, n, seed=80)
    z_c, z_f = saved_depths(one.eng, k * n, 64, 64)
    monkeypatch.setenv("NFB_TRAIN_MEM_MB", "48")
    tr = learner(env, sc, prec, weight)
    sb = trainer_gradients(env, tr, data, ids, n, seed=80)
    with pytest.raises(RuntimeError, match="train_debug"):  # chunked: no one-launch state to read
        tr.eng.train_debug()
    assert torch.equal(sb["pixel_rc"], sb1["pixel_rc"])
    torch.manual_seed(80)
    noise = env.ft._draw_noise(tr.opts, env.dev, k * n)
    R = reference_step(tr.mc, tr.mf, sc, ids, n, sb["pixel_rc"], noise, 0.1, z_c, z_f, bg_table=tr.background, learn_bg=True,
                       bg_weight=weight, latent_reg=LATENT_REG, want_params=True)
    check_trainer(f"chunked w={weight} {prec}", tr, sb, R, sc, ids, weight, prec)
