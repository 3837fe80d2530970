"""Phase-cycle profile of the render kernels (NfbDebug.prof).  Usage: python tools/phase_profile.py [fast|exact] [H W [NC NF]]

Needs a library with the timers compiled in: `python 4d-facial-avatars_b200/build.py --timers` (lib/libnfb_timers.so, picked
up here unless NFB_LIB is set).  The observers are the first thread of each row warpgroup of every CTA (warpgroup w's laps at
slot + 20 w) and the first thread of the ray warps (slots 40..59); their cycles are summed over CTAs and reported per tile
(MLP phases, one column per row warpgroup), per unit of work for the row warps' wait for the ray warps, and per unit for the
ray warps' per-ray stages.  "wait MMAs" includes issuing them and releasing the weight slots."""
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
H, W, NC, NF = (nums + [256, 256, 64, 128][len(nums):])[:4]
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
    eng.render_camera(fr["pose"], fr["intrinsics"], H, W, 0, H, 0.2, 0.8, NC, NF, background=bg, precision=prec)
prof = torch.zeros(64, dtype=torch.int64, device=dev)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
eng.render_camera(fr["pose"], fr["intrinsics"], H, W, 0, H, 0.2, 0.8, NC, NF, background=bg, precision=prec, prof=prof)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1)
c = prof.cpu().tolist()

# the kernel's work decomposition (TileGeom::make in csrc/nfb_layout.h): R rays per unit, tiles_c + tiles_f 128-row tiles per unit
R = 2 if 2 * (NC + NF) <= 512 else 1
tiles_per_unit = -(-R * NC // 128) + (-(-R * (NC + NF) // 128) if NF > 0 else 0)
units = -(-H * W // R)
ctas = min(torch.cuda.get_device_properties(dev).multi_processor_count, units)
tiles = units * tiles_per_unit
per_tile = {2: "prologue (z + PE)", 15: "ping-pong wait", 10: "wait weights (wait_full)", 11: "wait MMAs", 12: "epilogue",
            14: "end-of-MLP barrier", 13: "post-processing"}
per_unit = {16: "wait for ray warps"}
# the ray warps' observer (lane 0 of warp 1, slots 40..59): the per-ray stages of a unit, beside the row warps' tiles
RAY = 40  # nfb_render_common.cuh: kProfRay
per_unit_ray = {0: "wait coarse tiles", 1: "composite coarse", 2: "cdf", 3: "inverse-cdf", 4: "wait fine tiles",
                5: "composite fine", 6: "sort", 7: "ray setup + dir terms"}
WG = 20  # slot stride between the two row warpgroups' observers (nfb_render_common.cuh: kProfWgStride)
total = [sum(c[i + WG * w] for i in list(per_tile) + list(per_unit)) for w in (0, 1)]
total_ray = sum(c[RAY + i] for i in per_unit_ray)
print(f"{prec} {H}x{W} {NC}c+{NF}f: {ms:.2f} ms, {H*W/ms*1e3:.3e} rays/s; {R} rays/unit, {tiles_per_unit} tiles/unit, "
      f"{tiles/ctas:.0f} tiles per CTA; observers {total[0]/ctas/1e6:.2f} / {total[1]/ctas/1e6:.2f} Mcycles per CTA")
share = lambda v, w: 100 * v / total[w] if total[w] else 0.0  # noqa: E731
print(f"{'phase':28s} {'wg0 cycles/tile':>16s} {'share':>7s} {'wg1 cycles/tile':>16s} {'share':>7s}")
for i, name in per_tile.items():
    print(f"{name:28s} " + " ".join(f"{c[i + WG * w] / tiles:16.0f} {share(c[i + WG * w], w):6.1f}%" for w in (0, 1)))
print(f"{'phase':28s} {'wg0 cycles/unit':>16s} {'share':>7s} {'wg1 cycles/unit':>16s} {'share':>7s}")
for i, name in per_unit.items():
    print(f"{name:28s} " + " ".join(f"{c[i + WG * w] / units:16.0f} {share(c[i + WG * w], w):6.1f}%" for w in (0, 1)))
print(f"{'ray warps':28s} {'cycles/unit':>16s} {'share':>7s}   (observer {total_ray / ctas / 1e6:.2f} Mcycles per CTA)")
for i, name in per_unit_ray.items():
    print(f"{name:28s} {c[RAY + i] / units:16.0f} {100 * c[RAY + i] / total_ray if total_ray else 0.0:6.1f}%")
