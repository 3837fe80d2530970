// nfb_render_common.cuh — device code of the render kernel (nfb_render.cu): per-ray constants, the positional encoding's
// sin/cos, and the per-ray compositing.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include "nfb_ptx.cuh"

namespace nfb {

constexpr int kRayFloats = 40;  // o[3] d[3] dnorm valid bg[3] gidx PEd[24] dz frame pad[2]
struct RayP {  // per-ray constants in shared memory (kRayFloats floats)
  float o[3], d[3];
  float dnorm;
  int valid;
  float bg[3];
  int gidx;
  float ped[24];
  float dz;
  int frame;  // multi-frame kernels only: the ray's row of the frame table
  float pad[2];
};
static_assert(sizeof(RayP) == kRayFloats * 4, "RayP size");

// ------------------------------------------------------------------------------------------------
// sin/cos of y for the positional encoding.  The reference evaluates torch.sin(x * 2^k) in FP32
// (nerf_helpers.py:231-233); x * 2^k is exact, so both variants see the same argument.
//   exact: libdevice sinf/cosf (<= 2 ulp).
//   fast : two-constant Cody-Waite reduction to [-pi, pi] + MUFU.SIN/COS (abs err ~5e-7), well below the
//          FP16 rounding (2.4e-4) the value then receives.
template <bool EXACT>
__device__ __forceinline__ void pe_sincos(float y, float& s, float& c) {
  if constexpr (EXACT) {
    sincosf(y, &s, &c);
  } else {
    const float n = rintf(y * 0.15915494309189535f);
    float r = fmaf(-n, 6.2831854820251465f, y);
    r = fmaf(-n, -1.7484555e-7f, r);
    s = __sinf(r);
    c = __cosf(r);
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------
// Compositing of one ray by one warp (volume_rendering_utils.py:7-75).  Samples are lane-blocked.  `pre`
// holds what the step-9 epilogue prepared per sample: (colour r, g, b, sigma) with colour = sigmoid(rgb raw)
// — or the raw background colour on the last sample (:29-33) — and sigma = relu(raw + noise) (+1e-6 on the
// last sample, :52-53).  Returns w of the last sample; lane 0 writes rgb[3], disp, acc.
__device__ __forceinline__ float composite_ray(const float4* __restrict__ pre, const float* __restrict__ z, float* __restrict__ wbuf,
                                               int S, float dnorm, bool white_bkgd, float* out_rgb, float* out_disp,
                                               float* out_acc, int lane) {
  const int per = (S + 31) >> 5;
  const int i0 = lane * per;
  // pass 1: alpha per sample (kept in wbuf), product of (1 - alpha + 1e-10) over this lane's block
  float prod = 1.f;
  for (int j = 0; j < per; ++j) {
    const int i = i0 + j;
    if (i < S) {
      float delta = (i < S - 1) ? __fsub_rn(z[i + 1], z[i]) : 1e10f;
      delta = __fmul_rn(delta, dnorm);
      const float alpha = __fsub_rn(1.f, expf(-__fmul_rn(pre[i].w, delta)));
      wbuf[i] = alpha;
      prod *= __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f);
    }
  }
  // exclusive multiplicative scan over lanes
  float incl = prod;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl *= t;
  }
  float T = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) T = 1.f;
  // pass 2: weights and weighted sums
  float r = 0.f, g = 0.f, b = 0.f, depth = 0.f, acc = 0.f, wl = 0.f;
  for (int j = 0; j < per; ++j) {
    const int i = i0 + j;
    if (i < S) {
      const float alpha = wbuf[i];
      const float w = __fmul_rn(alpha, T);
      T *= __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f);
      wbuf[i] = w;
      const float4 q = pre[i];
      r = fmaf(w, q.x, r); g = fmaf(w, q.y, g); b = fmaf(w, q.z, b);
      depth = fmaf(w, z[i], depth);
      acc += w;
      if (i == S - 1) wl = w;
    }
  }
  r = warp_sum(r); g = warp_sum(g); b = warp_sum(b);
  depth = warp_sum(depth); acc = warp_sum(acc); wl = warp_sum(wl);
  if (lane == 0 && out_rgb) {
    if (white_bkgd) { r += 1.f - acc; g += 1.f - acc; b += 1.f - acc; }
    out_rgb[0] = r; out_rgb[1] = g; out_rgb[2] = b;
    *out_disp = 1.f / fmax_nan(1e-10f, depth / acc);
    *out_acc = acc;
  }
  return wl;
}


// Optional phase timers (NfbDebug.prof): cycles of one observer thread per role, summed over CTAs.  Compiled in only with
// -DNFB_TIMERS=1 (tools/phase_profile.py builds such a library): even disabled at run time they cost registers in the
// hot loops.
#ifndef NFB_TIMERS
#define NFB_TIMERS 0
#endif
constexpr int kProfWgStride = 20;  // render kernel: row warpgroup w's observer writes its laps at slot + 20 w (slots < 40)
constexpr int kProfRay = 40;       // ... and the ray warps' observer at slot + 40 (slots 40..59)
#if NFB_TIMERS
struct PhaseTimer {
  unsigned long long* dst;
  long long t0;
  __device__ __forceinline__ PhaseTimer(unsigned long long* d, bool on) : dst(on ? d : nullptr), t0(0) {
    if (dst) t0 = clock64();
  }
  __device__ __forceinline__ void lap(int slot) {
    if (dst) {
      const long long t1 = clock64();
      atomicAdd(dst + slot, (unsigned long long)(t1 - t0));
      t0 = t1;
    }
  }
};
#else
struct PhaseTimer {
  __device__ __forceinline__ PhaseTimer(unsigned long long*, bool) {}
  __device__ __forceinline__ void lap(int) {}
};
#endif

}  // namespace nfb
