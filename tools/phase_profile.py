"""Phase-cycle profile of the render kernels (NfbDebug.prof).  Usage: python tools/phase_profile.py [fast|exact] [H W]

Needs a library with the timers compiled in: `python 4d-facial-avatars_b200/build.py --timers` (lib/libnfb_timers.so, picked
up here unless NFB_LIB is set)."""
import os
import sys

_timers = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "4d-facial-avatars_b200", "lib", "libnfb_timers.so")
if "NFB_LIB" not in os.environ and os.path.exists(_timers):
    os.environ["NFB_LIB"] = _timers

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "4d-facial-avatars_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import nerface_oracle as O  # noqa: E402
import nerf  # noqa: E402
from nerf import _engine  # noqa: E402

prec = "exact" if "exact" in sys.argv else "fast"
nums = [int(a) for a in sys.argv[1:] if a.isdigit()]
H, W = (nums + [256, 256])[:2]
dev = torch.device("cuda", 0)
fr = O.synthetic_frame(0, H, W)
mk = lambda: nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)  # noqa: E731
mc, mf = mk(), mk()
mc.load_state_dict(O.random_init_params(100)); mf.load_state_dict(O.random_init_params(101))
mc, mf = mc.to(dev), mf.to(dev)
eng = _engine.renderer_for(dev)
eng.sync_weights(mc, mf)
eng.set_frame(fr["expr"].to(dev), fr["latent"].to(dev))
bg = fr["bg"].reshape(-1, 3).to(dev)
for _ in range(2):
    eng.render_camera(fr["pose"], fr["intrinsics"], H, W, 0, H, 0.2, 0.8, 64, 128, background=bg, precision=prec)
prof = torch.zeros(64, dtype=torch.int64, device=dev)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
eng.render_camera(fr["pose"], fr["intrinsics"], H, W, 0, H, 0.2, 0.8, 64, 128, background=bg, precision=prec, prof=prof)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1)
c = prof.cpu().tolist()
ctas = min(132, H * W // 2)
units = H * W / 2
tiles = units * 4
names = {0: "ray setup", 1: "dir term", 2: "prologue (z+PE)", 3: "end-of-pass barrier", 4: "composite", 5: "cdf", 6: "inverse-cdf", 7: "sort",
         39: "loop", 41: "producer: wait free slot", 40: "producer: issue", 44: "mma: issue", 45: "mma: wait A operand", 46: "mma: wait weights"}
names[47] = "mma: wait A operand (half 1)"
for s in range(10):
    names[10 + s] = f"wait MMA step {s} half 0"
    names[20 + s] = f"epilogue step {s} half 0"
    names[48 + s] = f"epilogue step {s} half 1"
for s in range(8):
    names[30 + s] = f"wait MMA step {s}{'+' if s == 7 else ''} half 1"
row_total = sum(c[i] for i in list(range(0, 8)) + list(range(10, 40)) + list(range(48, 58)))
print(f"{prec} {H}x{W}: {ms:.2f} ms, {H*W/ms*1e3:.3e} rays/s; row-warp observer total {row_total/ctas/1e6:.2f} Mcycles per CTA")
print(f"{'phase':28s} {'cycles/tile':>12s} {'share':>7s}")
for i in sorted(names):
    if c[i]:
        share = c[i] / row_total if (i < 40 or i >= 48) else c[i] / sum(c[40:48])
        print(f"{names[i]:28s} {c[i]/tiles:12.0f} {100*share:6.1f}%")
