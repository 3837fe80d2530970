"""Which library calls each Python host path makes, without a GPU: nerf._capi.lib is replaced by a recorder that returns
NFB_OK, and the device's renderer is a Renderer whose tensors live on the CPU.  Every call is recorded as its function name,
the null-ness of each pointer argument ('p' set, '0' null), and, for the structs passed by pointer, the null-ness of each
pointer field and the value of each scalar field (fields in the order of include/nfb.h); the 26-pointer parameter and
gradient arrays show one character per entry (in PARAM_ORDER; entries 22 and 23 are layers_dir.3.*, which gets no
gradient).  No address is recorded, so the traces are literals: they pin which entry point, argument and struct member
every public call uses, e.g. that the single-frame autograd backward always asks for d latent while the multi-frame one asks
only when the latents require grad, and that the multi-frame backward returns the expression gradient [F,76] outside
NfbInputGrads."""
import ctypes as C
import itertools
import types

import pytest
import torch

N, NC, NF, F = 6, 4, 2, 3


def _p(v):
    return "p" if v else "0"


def _struct(s):
    parts = []
    for name, ftype in s._fields_:
        v = getattr(s, name)
        if ftype is C.c_void_p:
            parts.append(_p(v))
        elif issubclass(ftype, C.Array):
            if ftype._type_ is C.c_void_p:
                parts.append("".join(_p(x) for x in v))
        else:
            parts.append(f"{v:g}" if isinstance(v, float) else str(v))
    return f"{type(s).__name__}({','.join(parts)})"


def _arg(a):
    if a is None:
        return "0"
    if isinstance(a, C.c_void_p):
        return _p(a.value)
    if type(a).__name__ == "CArgObject":  # C.byref(...)
        return _struct(a._obj) if isinstance(a._obj, C.Structure) else "p"
    if isinstance(a, C.Array):
        return "".join(_p(x) for x in a) if a._type_ is C.c_void_p else f"{a._type_.__name__}[{len(a)}]"
    if isinstance(a, float):
        return f"{a:g}"
    return str(a)


class Recorder:
    """Stands in for the ctypes library: every nfb_* call is recorded and returns NFB_OK."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("nfb_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append(f"{name}({' '.join(_arg(a) for a in args)})")
            return 0
        return call


@pytest.fixture
def rec(built_lib, monkeypatch):
    return recording_renderer(monkeypatch)


def recording_renderer(monkeypatch):
    from nerf import _capi, _engine
    r = Recorder()
    monkeypatch.setattr(_capi, "lib", r)
    monkeypatch.setattr(_engine, "_stream", lambda: C.c_void_p(0))
    eng = _engine.Renderer(torch.device("cuda", 0))  # its nfb_create goes to the recorder
    eng.device = torch.device("cpu")
    monkeypatch.setattr(_engine, "renderer_for", lambda device: eng)
    r.calls.clear()
    return types.SimpleNamespace(lib=r, eng=eng)


def _model(seed):
    import nerf
    torch.manual_seed(seed)
    return nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True,
                                                           include_input_dir=False)


def _params(m):
    from nerf._engine import PARAM_ORDER
    sd = dict(m.named_parameters())
    return [sd[k] for k in PARAM_ORDER]


def _rays(n=N):
    g = torch.Generator().manual_seed(n)
    return torch.rand(n, 3, generator=g), torch.rand(n, 3, generator=g)


def _noise(n=N):
    return dict(t_rand=torch.rand(n, NC), n_c=torch.randn(n, NC), u=torch.rand(n, NF), n_f=torch.randn(n, NC + NF))


def _render(eng, frames, train, noise=True, fine=True):
    ro, rd = _rays()
    kw = dict(frame_index=torch.arange(N) % F) if frames else {}
    if frames:
        eng.set_frames(torch.rand(F, 76), torch.rand(F, 32))
    else:
        eng.set_frame(torch.rand(76), torch.rand(32))
    return eng.render(ro, rd, 0.2, 0.8, NC, NF if fine else 0, perturb=True, noise_std=0.1, background=torch.rand(N, 3),
                      dir_z=None if frames else torch.rand(N), noise=_noise() if noise else None, train=train, **kw)


def _ret(r):
    """Renderer.backward's result: tuple length, which gradients came back, and the shapes of the latent and input ones."""
    gl = "None" if r[2] is None else "x".join(map(str, r[2].shape))
    s = [f"len={len(r)}", "gc=" + ("None" if r[0] is None else "".join(_p(t is not None) for t in r[0])),
         "gf=" + ("None" if r[1] is None else "".join(_p(t is not None) for t in r[1])), f"glat={gl}"]
    if len(r) == 4:
        s.append("inputs=" + ",".join(f"{k}:{'x'.join(map(str, v.shape))}" for k, v in sorted(r[3].items())))
    return "-> " + " ".join(s)


def _out_grads():
    return [torch.rand(N, 3), None, torch.rand(N), torch.rand(N, 3), None, None, torch.rand(N)]


# ---- the cases: each returns the trace of library calls (and results) the public call produced

def case_render(r, frames, train):
    _render(r.eng, frames, train, noise=train)
    return r.lib.calls


def case_render_coarse_only(r):
    _render(r.eng, False, False, noise=False, fine=False)
    return r.lib.calls


def case_render_camera(r, num_fine):
    r.eng.render_camera(torch.eye(4), [2.0, 2.0, 1.5, 1.0], 2, 3, 0, 2, 0.2, 0.8, NC, num_fine, background=torch.rand(N, 3))
    return r.lib.calls


def case_render_frame_host(r):
    r.eng.render_frame_host(torch.eye(4), [2.0, 2.0, 1.5, 1.0], 2, 3, 0, 2, 0.2, 0.8, torch.rand(76), torch.rand(32), torch.rand(N, 3),
                            NC, NF, torch.empty(11, N))
    return r.lib.calls


BACKWARD_INPUTS = {"none": None, "empty": [], "expr": ["expression"],
                   "all": ["ray_origins", "ray_directions", "dir_z", "background", "expression"]}


def case_backward(r, frames, want_latent, want_params, inputs):
    _render(r.eng, frames, True)
    r.lib.calls.clear()
    mc, mf = _model(1), _model(2)
    inp = BACKWARD_INPUTS[inputs]
    if frames and inp is not None and "dir_z" in inp:
        inp = [k for k in inp if k != "dir_z"]  # the multi-frame forward above has no dir_z
    res = r.eng.backward(_out_grads(), _params(mc), _params(mf), want_latent=want_latent, want_params=want_params, inputs=inp,
                         frames=frames)
    return r.lib.calls + [_ret(res)]


def case_backward_frames_after_single(r):
    _render(r.eng, False, True)
    r.lib.calls.clear()
    with pytest.raises(RuntimeError, match="multi-frame training forward"):
        r.eng.backward(_out_grads(), _params(_model(1)), None, frames=True)
    return r.lib.calls


def case_backward_into(r, frames):
    from nerf._engine import PARAM_ORDER
    _render(r.eng, frames, True)
    r.lib.calls.clear()
    pc, pf = _params(_model(1)), _params(_model(2))
    gc = [None if k.startswith("layers_dir.3") else torch.empty_like(p) for k, p in zip(PARAM_ORDER, pc)]
    gf = [None if k.startswith("layers_dir.3") else torch.empty_like(p) for k, p in zip(PARAM_ORDER, pf)]
    og = (torch.rand(N, 3), None, None, torch.rand(N, 3), None, None, None)
    r.eng.backward_into(og, pc, pf, gc, gf, torch.empty(F, 32) if frames else torch.empty(32), frames=frames)
    return r.lib.calls


def _cfg(perturb=True):
    import nerf
    blk = dict(num_coarse=NC, num_fine=NF, perturb=perturb, lindisp=False, radiance_field_noise_std=0.1 if perturb else 0.0,
               white_background=False, chunksize=4)
    return nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, train=blk, validation=dict(blk, perturb=False, radiance_field_noise_std=0.0)),
                             dataset=dict(no_ndc=True, near=0.2, far=0.8)))


def _dropin_inputs(frozen, frames, latent_grad=True):
    mc, mf = _model(1), _model(2)
    ro, rd = _rays()
    expr = torch.rand(F, 76) if frames else torch.rand(76)
    lat = torch.rand(F, 32) if frames else torch.rand(32)
    bg = torch.rand(N, 3)
    if frozen:
        for p in list(mc.parameters()) + list(mf.parameters()):
            p.requires_grad_(False)
        for t in (ro, expr, lat, bg) if latent_grad else (ro, expr, bg):
            t.requires_grad_(True)
    return mc, mf, ro, rd, expr, lat, bg


def case_run_one_iter(r, frozen, latent_grad=True):
    import nerf
    mc, mf, ro, rd, expr, lat, bg = _dropin_inputs(frozen, False, latent_grad)
    out = nerf.run_one_iter_of_nerf(2, 3, 1.0, mc, mf, ro, rd, _cfg(), mode="train", expressions=expr, background_prior=bg,
                                    latent_code=lat)
    (out[0].sum() + out[3].sum() + out[6].sum()).backward()
    return r.lib.calls


def case_run_one_iter_eval(r):
    import nerf
    mc, mf, ro, rd, expr, lat, bg = _dropin_inputs(False, False)
    with torch.no_grad():
        nerf.run_one_iter_of_nerf(2, 3, 1.0, mc, mf, ro, rd, _cfg(), mode="validation", expressions=expr, background_prior=bg,
                                  latent_code=lat)
    return r.lib.calls


def case_render_frames(r, frozen, latent_grad=True):
    import nerf
    mc, mf, ro, rd, expr, lat, bg = _dropin_inputs(frozen, True, latent_grad)
    out = nerf.render_frames(ro, rd, torch.arange(N) % F, expr, lat, mc, mf, _cfg(), background_prior=bg)
    (out[0].sum() + out[3].sum() + out[6].sum()).backward()
    return r.lib.calls


def _trainer(r):
    from nerf import fused_train
    tr = fused_train.FusedTrainer(_model(1), _model(2), n_latent=4, num_coarse=NC, num_fine=NF)
    r.lib.calls.clear()
    return tr


def case_trainer_step(r):
    tr = _trainer(r)
    ro, rd = _rays()
    tr.step(ro, rd, torch.rand(N, 3), torch.rand(76), 2, background=torch.rand(N, 3))
    return r.lib.calls + [f"row={int(tr._row)} iter={tr.iter}"]


def case_trainer_images(r, k):
    tr = _trainer(r)
    data = types.SimpleNamespace(background=torch.zeros(1))
    sb = tr._images_buffers(data, k, N // k)
    tr._images_gradients(sb, k, N // k)
    return r.lib.calls


CASES = {f"render/{'frames' if fr else 'single'}/{'train' if tr else 'eval'}": (case_render, (fr, tr))
         for fr in (False, True) for tr in (False, True)}
CASES.update({f"backward/{'frames' if fr else 'single'}/lat{int(wl)}/par{int(wp)}/{inp}": (case_backward, (fr, wl, wp, inp))
              for fr, wl, wp, inp in itertools.product((False, True), (False, True), (False, True), BACKWARD_INPUTS)})
CASES["render/single/eval_coarse_only"] = (case_render_coarse_only, ())
CASES.update({f"render_camera/nf{nf}": (case_render_camera, (nf,)) for nf in (0, NF)})
CASES["render_frame_host"] = (case_render_frame_host, ())
CASES["backward/frames_after_single"] = (case_backward_frames_after_single, ())
CASES.update({f"backward_into/{'frames' if fr else 'single'}": (case_backward_into, (fr,)) for fr in (False, True)})
CASES.update({f"run_one_iter/{'frozen' if fz else 'trainable'}": (case_run_one_iter, (fz,)) for fz in (False, True)})
CASES["run_one_iter/frozen_fixed_latent"] = (case_run_one_iter, (True, False))
CASES["render_frames/frozen_fixed_latent"] = (case_render_frames, (True, False))
CASES["run_one_iter/eval"] = (case_run_one_iter_eval, ())
CASES.update({f"render_frames/{'frozen' if fz else 'trainable'}": (case_render_frames, (fz,)) for fz in (False, True)})
CASES["trainer/step"] = (case_trainer_step, ())
CASES.update({f"trainer/images_k{k}": (case_trainer_images, (k,)) for k in (1, 3)})


def trace(r, case):
    fn, args = CASES[case]
    return list(fn(r, *args))


# the 26-entry arrays: every parameter, and every gradient but layers_dir.3.*
P26, G26 = "p" * 26, "p" * 22 + "00pp"

EXPECTED = {
    "backward/frames/lat0/par0/all": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 0 p NfbInputGrads(p,p,0,p,0) 0)",
        "-> len=4 gc=None gf=None glat=None inputs=background:6x3,expression:3x76,ray_directions:6x3,ray_origins:6x3",
    ],
    "backward/frames/lat0/par0/empty": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 0 0 NfbInputGrads(0,0,0,0,0) 0)",
        "-> len=4 gc=None gf=None glat=None inputs=",
    ],
    "backward/frames/lat0/par0/expr": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 0 p NfbInputGrads(0,0,0,0,0) 0)",
        "-> len=4 gc=None gf=None glat=None inputs=expression:3x76",
    ],
    "backward/frames/lat0/par0/none": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 0 0 NfbInputGrads(0,0,0,0,0) 0)",
        "-> len=3 gc=None gf=None glat=None",
    ],
    "backward/frames/lat0/par1/all": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} 0 p NfbInputGrads(p,p,0,p,0) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=None inputs=background:6x3,expression:3x76,ray_directions:6x3,ray_origins:6x3",
    ],
    "backward/frames/lat0/par1/empty": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} 0 0 NfbInputGrads(0,0,0,0,0) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=None inputs=",
    ],
    "backward/frames/lat0/par1/expr": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} 0 p NfbInputGrads(0,0,0,0,0) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=None inputs=expression:3x76",
    ],
    "backward/frames/lat0/par1/none": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} 0 0 NfbInputGrads(0,0,0,0,0) 0)",
        f"-> len=3 gc={G26} gf={G26} glat=None",
    ],
    "backward/frames/lat1/par0/all": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 p p NfbInputGrads(p,p,0,p,0) 0)",
        "-> len=4 gc=None gf=None glat=3x32 inputs=background:6x3,expression:3x76,ray_directions:6x3,ray_origins:6x3",
    ],
    "backward/frames/lat1/par0/empty": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 p 0 NfbInputGrads(0,0,0,0,0) 0)",
        "-> len=4 gc=None gf=None glat=3x32 inputs=",
    ],
    "backward/frames/lat1/par0/expr": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 p p NfbInputGrads(0,0,0,0,0) 0)",
        "-> len=4 gc=None gf=None glat=3x32 inputs=expression:3x76",
    ],
    "backward/frames/lat1/par0/none": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 p 0 NfbInputGrads(0,0,0,0,0) 0)",
        "-> len=3 gc=None gf=None glat=3x32",
    ],
    "backward/frames/lat1/par1/all": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} p p NfbInputGrads(p,p,0,p,0) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=3x32 inputs=background:6x3,expression:3x76,ray_directions:6x3,ray_origins:6x3",
    ],
    "backward/frames/lat1/par1/empty": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} p 0 NfbInputGrads(0,0,0,0,0) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=3x32 inputs=",
    ],
    "backward/frames/lat1/par1/expr": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} p p NfbInputGrads(0,0,0,0,0) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=3x32 inputs=expression:3x76",
    ],
    "backward/frames/lat1/par1/none": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} p 0 NfbInputGrads(0,0,0,0,0) 0)",
        f"-> len=3 gc={G26} gf={G26} glat=3x32",
    ],
    "backward/frames_after_single": [],
    "backward/single/lat0/par0/all": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 0 NfbInputGrads(p,p,p,p,p) 0)",
        "-> len=4 gc=None gf=None glat=None inputs=background:6x3,dir_z:6,expression:76,ray_directions:6x3,ray_origins:6x3",
    ],
    "backward/single/lat0/par0/empty": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 0 NfbInputGrads(0,0,0,0,0) 0)",
        "-> len=4 gc=None gf=None glat=None inputs=",
    ],
    "backward/single/lat0/par0/expr": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 0 NfbInputGrads(0,0,0,0,p) 0)",
        "-> len=4 gc=None gf=None glat=None inputs=expression:76",
    ],
    "backward/single/lat0/par0/none": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 0 0 0)",
        "-> len=3 gc=None gf=None glat=None",
    ],
    "backward/single/lat0/par1/all": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} 0 NfbInputGrads(p,p,p,p,p) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=None inputs=background:6x3,dir_z:6,expression:76,ray_directions:6x3,ray_origins:6x3",
    ],
    "backward/single/lat0/par1/empty": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} 0 NfbInputGrads(0,0,0,0,0) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=None inputs=",
    ],
    "backward/single/lat0/par1/expr": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} 0 NfbInputGrads(0,0,0,0,p) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=None inputs=expression:76",
    ],
    "backward/single/lat0/par1/none": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} 0 0 0)",
        f"-> len=3 gc={G26} gf={G26} glat=None",
    ],
    "backward/single/lat1/par0/all": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 p NfbInputGrads(p,p,p,p,p) 0)",
        "-> len=4 gc=None gf=None glat=32 inputs=background:6x3,dir_z:6,expression:76,ray_directions:6x3,ray_origins:6x3",
    ],
    "backward/single/lat1/par0/empty": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 p NfbInputGrads(0,0,0,0,0) 0)",
        "-> len=4 gc=None gf=None glat=32 inputs=",
    ],
    "backward/single/lat1/par0/expr": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 p NfbInputGrads(0,0,0,0,p) 0)",
        "-> len=4 gc=None gf=None glat=32 inputs=expression:76",
    ],
    "backward/single/lat1/par0/none": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} 0 0 p 0 0)",
        "-> len=3 gc=None gf=None glat=32",
    ],
    "backward/single/lat1/par1/all": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} p NfbInputGrads(p,p,p,p,p) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=32 inputs=background:6x3,dir_z:6,expression:76,ray_directions:6x3,ray_origins:6x3",
    ],
    "backward/single/lat1/par1/empty": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} p NfbInputGrads(0,0,0,0,0) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=32 inputs=",
    ],
    "backward/single/lat1/par1/expr": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} p NfbInputGrads(0,0,0,0,p) 0)",
        f"-> len=4 gc={G26} gf={G26} glat=32 inputs=expression:76",
    ],
    "backward/single/lat1/par1/none": [
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,p,p,0,0,p) {P26} {P26} {G26} {G26} p 0 0)",
        f"-> len=3 gc={G26} gf={G26} glat=32",
    ],
    "backward_into/frames": [
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,0,p,0,0,0) {P26} {P26} {G26} {G26} p 0 0 0)",
    ],
    "backward_into/single": [
        f"nfb_render_backward(0 NfbOutGrads(p,0,0,p,0,0,0) {P26} {P26} {G26} {G26} p 0)",
    ],
    "render/frames/eval": [
        "nfb_set_frames(0 p p 3 0)",
        "nfb_render_forward_frames(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) p NfbSampling(4,2,1,0.1,0,0,0,p,p) 0 NfbOutputs(p,p,p,p,p,p,p) 0)",
    ],
    "render/frames/train": [
        "nfb_set_frames(0 p p 3 0)",
        "nfb_render_forward_frames_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) p NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
    ],
    "render/single/eval": [
        "nfb_set_frame(0 p p 0)",
        "nfb_render_forward(0 NfbRays(p,p,6,0,0,0,0.2,0.8,p,p) NfbSampling(4,2,1,0.1,0,0,0,p,p) 0 NfbOutputs(p,p,p,p,p,p,p) 0 0)",
    ],
    "render/single/eval_coarse_only": [
        "nfb_set_frame(0 p p 0)",
        "nfb_render_forward(0 NfbRays(p,p,6,0,0,0,0.2,0.8,p,p) NfbSampling(4,0,1,0.1,0,0,0,p,0) 0 NfbOutputs(p,p,p,0,0,0,p) 0 0)",
    ],
    "render/single/train": [
        "nfb_set_frame(0 p p 0)",
        "nfb_render_forward_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,p,p) NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
    ],
    "render_camera/nf0": [
        "nfb_render_forward(0 NfbRays(0,0,6,2,3,0,0.2,0.8,0,p) NfbSampling(4,0,0,0,0,0,0,p,0) 0 NfbOutputs(p,p,p,0,0,0,p) 0 0)",
    ],
    "render_camera/nf2": [
        "nfb_render_forward(0 NfbRays(0,0,6,2,3,0,0.2,0.8,0,p) NfbSampling(4,2,0,0,0,0,0,p,p) 0 NfbOutputs(p,p,p,p,p,p,p) 0 0)",
    ],
    "render_frame_host": [
        "nfb_render_frame_host(0 c_float[12] c_double[4] 2 3 0 2 0.2 0.8 p p p NfbSampling(4,2,0,0,0,0,0,p,p) p 0)",
    ],
    "render_frames/frozen": [
        f"nfb_load_weights(0 0 {P26} 0)",
        f"nfb_load_weights(0 1 {P26} 0)",
        "nfb_set_frames(0 p p 3 0)",
        "nfb_render_forward_frames_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) p NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,0,p,0,0,p) {P26} {P26} 0 0 p p NfbInputGrads(p,p,0,p,0) 0)",
    ],
    "render_frames/frozen_fixed_latent": [
        f"nfb_load_weights(0 0 {P26} 0)",
        f"nfb_load_weights(0 1 {P26} 0)",
        "nfb_set_frames(0 p p 3 0)",
        "nfb_render_forward_frames_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) p NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,0,p,0,0,p) {P26} {P26} 0 0 0 p NfbInputGrads(p,p,0,p,0) 0)",
    ],
    "render_frames/trainable": [
        f"nfb_load_weights(0 0 {P26} 0)",
        f"nfb_load_weights(0 1 {P26} 0)",
        "nfb_set_frames(0 p p 3 0)",
        "nfb_render_forward_frames_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) p NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,0,p,0,0,p) {P26} {P26} {G26} {G26} 0 0 NfbInputGrads(0,0,0,0,0) 0)",
    ],
    "run_one_iter/eval": [
        f"nfb_load_weights(0 0 {P26} 0)",
        f"nfb_load_weights(0 1 {P26} 0)",
        "nfb_set_frame(0 p p 0)",
        "nfb_render_forward(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) NfbSampling(4,2,0,0,0,0,0,p,p) 0 NfbOutputs(p,p,p,p,p,p,p) 0 0)",
    ],
    "run_one_iter/frozen": [
        f"nfb_load_weights(0 0 {P26} 0)",
        f"nfb_load_weights(0 1 {P26} 0)",
        "nfb_set_frame(0 p p 0)",
        "nfb_render_forward_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,0,p,0,0,p) {P26} {P26} 0 0 p NfbInputGrads(p,p,0,p,p) 0)",
    ],
    "run_one_iter/frozen_fixed_latent": [
        f"nfb_load_weights(0 0 {P26} 0)",
        f"nfb_load_weights(0 1 {P26} 0)",
        "nfb_set_frame(0 p p 0)",
        "nfb_render_forward_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,0,p,0,0,p) {P26} {P26} 0 0 p NfbInputGrads(p,p,0,p,p) 0)",
    ],
    "run_one_iter/trainable": [
        f"nfb_load_weights(0 0 {P26} 0)",
        f"nfb_load_weights(0 1 {P26} 0)",
        "nfb_set_frame(0 p p 0)",
        "nfb_render_forward_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
        f"nfb_render_backward_ex(0 NfbOutGrads(p,0,0,p,0,0,p) {P26} {P26} {G26} {G26} p NfbInputGrads(0,0,0,0,0) 0)",
    ],
    "trainer/images_k1": [
        "nfb_set_frame(0 p p 0)",
        "nfb_render_forward_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
        "nfb_loss_mse_grad(0 p p p 6 6 p p p 0)",
        f"nfb_render_backward(0 NfbOutGrads(p,0,0,p,0,0,0) {P26} {P26} {G26} {G26} p 0)",
        "nfb_latent_rows_grad(0 p p 1 p 4 p 0 0)",
    ],
    "trainer/images_k3": [
        "nfb_set_frames(0 p p 3 0)",
        "nfb_render_forward_frames_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) p NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
        "nfb_loss_mse_grad(0 p p p 6 6 p p p 0)",
        f"nfb_render_backward_frames(0 NfbOutGrads(p,0,0,p,0,0,0) {P26} {P26} {G26} {G26} p 0 0 0)",
        "nfb_latent_rows_grad(0 p p 3 p 4 p 0.00166667 0)",
    ],
    "trainer/step": [
        "nfb_set_frame(0 p p 0)",
        "nfb_render_forward_train(0 NfbRays(p,p,6,0,0,0,0.2,0.8,0,p) NfbSampling(4,2,1,0.1,0,0,0,p,p) NfbNoise(p,p,p,p) NfbOutputs(p,p,p,p,p,p,p) 0)",
        "nfb_loss_mse_grad(0 p p p 6 6 p p p 0)",
        f"nfb_render_backward(0 NfbOutGrads(p,0,0,p,0,0,0) {P26} {P26} {G26} {G26} p 0)",
        "nfb_adam_step_dev(0 p p p p 1137792 p 0)",
        f"nfb_repack(0 {P26} {P26} 0)",
        "row=2 iter=1",
    ],
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_library_calls(rec, case):
    assert trace(rec, case) == EXPECTED[case]
