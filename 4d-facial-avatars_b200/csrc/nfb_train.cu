// nfb_train.cu — backward of the render path as hand-written sm_90a kernels.
//
// The reference has no hand-written backward: `loss.backward()` (train_transformed_rays.py:389) runs torch.autograd over
// the unfused graph of train_utils.py:36-162 / volume_rendering_utils.py:7-75 / models.py:236-261.  SURVEY.md §8 (a''')
// derives what that computes; this file implements it in four stages, all on the caller's stream:
//
//   1. composite_bwd_kernel   G = dL/d(rgb, disp, acc, w_last) per ray  ->  dL/d(rgb_raw, sigma_raw) per sample.
//                             Re-evaluates the compositing of both passes from what the training forward saved (depths,
//                             colours, ReLU input of sigma) with a division-free reverse recurrence for the transmittance
//                             term.  Also yields per-ray d fc_rgb.bias / d sigma-bias sums and the max |gradient| for the scale.
//   2. chain_kernel           dX chain of the MLP per 128-row tile on wgmma: 9 steps with transposed weight streams,
//                             same machinery as the forward kernel (register accumulators, shared-memory activations
//                             overwritten in place, the bulk-copy ring of nfb_pipeline.cuh).  The epilogue applies the saved ReLU masks and
//                             writes every dY as a transposed FP16 image into the tile record.
//   3. dw_kernel              dW[n,k] = sum_rows dY[row,n] X[row,k] for every layer: both operands are bulk-copied from
//                             the tile records (K-major images whose K axis is the sample row) and multiplied on wgmma
//                             (M=128 output features x N input features per job, FP32 accumulation in registers over all
//                             tiles of the CTA), then stored as that CTA's partial.  One launch for both networks; the job
//                             groups are laid out for L2 sharing of the input images.
//   3b. grad_reduce_kernel    adds the partials into the FP32 accumulators in ascending part order, and the compositing
//                             backward's per-ray bias sums in a fixed order: no floating-point atomics, so the backward
//                             repeats bit for bit (include/nfb.h).
//   4. finalize_kernel        un-folds the kernel's parametrisation (fc_feat pre-multiplied into fc_alpha / layers_dir.0,
//                             conditioning columns folded into biases) by the chain rule and writes the 24 used parameter
//                             gradients of each network in the reference's state_dict layout, plus d latent_code.
//
// Gradients are carried in FP16 with one power-of-two loss scale per backward call (max |d raw| -> 2^10), FP32 accumulate.
// Exact-grad mode (NFB_PREC_EXACT_GRAD) runs the *_x3 instantiations of stages 2, 3, 5 and the per-frame sums: every FP16
// operand is hi + lo (records 2 MiB apart, nfb_layout.h rec_stride), multiplied as hi.hi + hi.lo + lo.hi.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "nfb_internal.h"
#include "nfb_layout.h"
#include "nfb_pipeline.cuh"
#include "nfb_ptx.cuh"
#include "nfb_save.cuh"

namespace nfb {

// ================================================================================================
// 1. compositing backward (SIMT; one thread per (pass, ray))
// ================================================================================================
// One WARP per (ray, pass); samples are lane-blocked (lane l owns samples [l*per, (l+1)*per)).  The forward product of
// (1 - alpha + 1e-10) and the reverse affine recurrence  C_{i-1} = dLdw_i alpha_i + omega_i C_i  are both scans: in-lane
// sequential, across lanes a shuffle scan (of products / of composed affine maps).
// kInputs: also the per-ray terms of the input gradients, from values the sweep already has:
//   ray_dn[pass][g]     = dL/d|d| through the sample spacings  = sum_i dsig_i sigma_i / |d|   (delta_i = dz_i |d|)
//   ray_bg[pass][g][3]  = w_{S-1} G_rgb (the background replaces the colour of the last sample)
template <bool kInputs>
__global__ void __launch_bounds__(256) composite_bwd_kernel(const CompBwdParams q) {
  const int lane = threadIdx.x & 31;
  const int idx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int npass = q.geom.passes(), n_rays = q.geom.n_rays;
  if (idx >= npass * n_rays) return;  // whole warps
  const int pass = idx / n_rays;
  const int g = idx - pass * n_rays;
  const int S = q.geom.samples(pass);
  const float* __restrict__ z = (pass ? q.z_f : q.z_c) + (size_t)g * S;
  const float4* __restrict__ raw = reinterpret_cast<const float4*>(pass ? q.raw_f : q.raw_c) + (size_t)g * S;
  const float dn = q.dnorm[g];
  float G0 = 0.f, G1 = 0.f, G2 = 0.f;
  if (q.g_rgb[pass]) { G0 = q.g_rgb[pass][3 * g]; G1 = q.g_rgb[pass][3 * g + 1]; G2 = q.g_rgb[pass][3 * g + 2]; }
  const float gdisp = q.g_disp[pass] ? q.g_disp[pass][g] : 0.f;
  float g_acc = q.g_acc[pass] ? q.g_acc[pass][g] : 0.f;
  const float gwl = (pass == npass - 1 && q.g_wlast) ? q.g_wlast[g] : 0.f;
  constexpr int kPer = 16;  // S <= 512
  const int per = (S + 31) >> 5;
  const int i0 = lane * per;

  // ---- forward: alpha, e = exp(-sigma delta) per sample; transmittance in front of this lane's block
  float e_[kPer], zl[kPer];
  float prod = 1.f;
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    const int i = i0 + j;
    e_[j] = 1.f; zl[j] = 0.f;
    if (j < per && i < S) {
      zl[j] = z[i];
      const float delta = ((i < S - 1) ? (z[i + 1] - zl[j]) : 1e10f) * dn;
      const float sig = relu_nan(raw[i].w) + (i == S - 1 ? 1e-6f : 0.f);  // a NaN input stays NaN, as in the forward
      e_[j] = expf(-sig * delta);
      prod *= ((1.f - (1.f - e_[j])) + 1e-10f);
    }
  }
  float incl = prod;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl *= t;
  }
  float T0 = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) T0 = 1.f;
  float depth = 0.f, acc = 0.f;
  {
    float T = T0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      if (j < per && i0 + j < S) {
        const float alpha = 1.f - e_[j];
        const float w = alpha * T;
        depth = fmaf(w, zl[j], depth);
        acc += w;
        T *= (1.f - alpha) + 1e-10f;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    depth += __shfl_xor_sync(0xffffffffu, depth, o);
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
  }
  // disp = 1 / max(1e-10, depth / acc)  (volume_rendering_utils.py:69); rgb += 1 - acc with a white background (:71-72).
  // A NaN depth / acc passes (torch.max keeps it, so its gradient is NaN); only the clamped branch has no gradient.
  float g_depth = 0.f;
  if (gdisp != 0.f) {
    const float qv = depth / acc;
    if (!(qv <= 1e-10f)) {
      const float dq = -gdisp / (qv * qv);
      g_depth = dq / acc;
      g_acc += -dq * depth / (acc * acc);
    }
  }
  if (q.white_bkgd) g_acc -= (G0 + G1 + G2);

  // ---- reverse sweep.  With omega_i = 1 - alpha_i + 1e-10 and C_i = sum_{k>i} dLdw_k alpha_k prod_{i<j<k} omega_j:
  //   dL/d alpha_i = T_i (dLdw_i - C_i),   C_{i-1} = dLdw_i alpha_i + omega_i C_i      (no division by omega).
  // A lane's block maps the C entering at its top sample to the C leaving below its first: C_out = A + B C_in.
  float A = 0.f, B = 1.f;
#pragma unroll
  for (int j = kPer - 1; j >= 0; --j) {
    const int i = i0 + j;
    if (j < per && i < S) {
      const float4 r4 = raw[i];
      const float dLdw = G0 * r4.x + G1 * r4.y + G2 * r4.z + g_acc + g_depth * zl[j] + (i == S - 1 ? gwl : 0.f);
      const float om = e_[j] + 1e-10f;
      A = fmaf(om, A, dLdw * (1.f - e_[j]));
      B *= om;
    }
  }
  // suffix composition over lanes 31 .. l+1 -> the C entering this lane (exclusive, from above)
  float SA = A, SB = B;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float ta = __shfl_down_sync(0xffffffffu, SA, o), tb = __shfl_down_sync(0xffffffffu, SB, o);
    if (lane + o < 32) { SA = fmaf(SB, ta, SA); SB *= tb; }  // this (lower) block applied AFTER the higher ones: A + B (ta + tb C)
  }
  float C = __shfl_down_sync(0xffffffffu, SA, 1);  // composed map of all higher lanes applied to C = 0
  if (lane == 31) C = 0.f;

  const TileGeom::RayRows rows = q.geom.ray_rows(pass, g);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f, amax = 0.f;
  float gdn = 0.f;  // kInputs: sum of dsig_i sigma_i over this lane's samples
  // transmittance in front of each sample of this block, walking down from the block's end
  float Tj[kPer];
  {
    float T = T0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      Tj[j] = T;
      if (j < per && i0 + j < S) T *= (1.f - (1.f - e_[j])) + 1e-10f;
    }
  }
#pragma unroll
  for (int j = kPer - 1; j >= 0; --j) {
    const int i = i0 + j;
    if (j < per && i < S) {
      const float4 r4 = raw[i];
      const float delta = ((i < S - 1) ? (z[i + 1] - zl[j]) : 1e10f) * dn;
      const float e = e_[j];
      const float alpha = 1.f - e;
      const float Ti = Tj[j];
      const float w = alpha * Ti;
      const float dLdw = G0 * r4.x + G1 * r4.y + G2 * r4.z + g_acc + g_depth * zl[j] + (i == S - 1 ? gwl : 0.f);
      const float dalpha = Ti * (dLdw - C);
      const float dsig = dalpha * (delta * e);  // d alpha / d sigma = delta exp(-sigma delta); (1e10 * 0) stays 0
      float4 d;
      // ReLU (the +1e-6 on the last sample is an additive constant); a NaN input passes its gradient, as torch's does
      d.w = (r4.w <= 0.f) ? 0.f : dsig;
      if constexpr (kInputs) gdn = fmaf(dsig, relu_nan(r4.w) + (i == S - 1 ? 1e-6f : 0.f), gdn);
      if (q.has_bg && i == S - 1) {
        d.x = d.y = d.z = 0.f;                  // background colour is data (train_background=False)
        if constexpr (kInputs) {
          float* bgo = q.ray_bg + ((size_t)pass * n_rays + g) * 3;
          bgo[0] = w * G0; bgo[1] = w * G1; bgo[2] = w * G2;
        }
      } else {
        d.x = w * G0 * r4.x * (1.f - r4.x);     // sigmoid
        d.y = w * G1 * r4.y * (1.f - r4.y);
        d.z = w * G2 * r4.z * (1.f - r4.z);
      }
      C = fmaf(e + 1e-10f, C, dLdw * alpha);
      reinterpret_cast<float4*>(q.draw)[rows.slot(i)] = d;
      s0 += d.x; s1 += d.y; s2 += d.z; s3 += d.w;
      amax = fmaxf(amax, fmaxf(fmaxf(fabsf(d.x), fabsf(d.y)), fmaxf(fabsf(d.z), fabsf(d.w))));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o); s3 += __shfl_xor_sync(0xffffffffu, s3, o);
    const float t = __shfl_xor_sync(0xffffffffu, amax, o);
    amax = (t != t || amax != amax) ? __int_as_float(0x7fc00000) : fmaxf(amax, t);
    if constexpr (kInputs) gdn += __shfl_xor_sync(0xffffffffu, gdn, o);
  }
  if constexpr (kInputs) {
    if (lane == 0) q.ray_dn[(size_t)pass * n_rays + g] = gdn / dn;
  }
  if (lane == 0) {
    reinterpret_cast<float4*>(q.bsum)[(size_t)pass * n_rays + g] = make_float4(s0, s1, s2, s3);  // summed by grad_reduce_kernel
    if (amax == amax && amax < 3.0e38f) atomicMax(q.absmax, __float_as_uint(amax));  // a max: independent of the order
  }
}

// scal[0] = loss scale (power of two bringing max |d raw| to about 2^10), scal[1] = 1 / scale.
__global__ void scale_kernel(const unsigned int* __restrict__ absmax, float* __restrict__ scal) {
  const float m = __uint_as_float(*absmax);
  int e = 0;
  if (m > 0.f) {
    e = 10 - (int)ceilf(log2f(m));
    e = max(-100, min(100, e));
  }
  scal[0] = exp2f((float)e);
  scal[1] = exp2f((float)-e);
}

// ================================================================================================
// 2. dX chain kernel
// ================================================================================================
namespace chain {

// Roles as in the forward kernel (nfb_pipeline.cuh): warp 0 streams the transposed weights (kBwdStream, written by
// repack_kernel in nfb_pack.cu), warpgroups 1 and 2 compute rows [64w, 64w+64) of the tile on wgmma with register
// accumulators; their epilogue applies the saved ReLU mask, writes the FP16 result in place into the shared-memory activation
// buffer (A operand of the next step) and as the transposed dY image into the tile record.
// X3 (exact-grad mode, chain_x3_kernel): every operand is hi + lo.  The activation buffer and the d raw operand get a lo copy,
// the producer streams each unit's hi weights then its lo weights (wstream_lo) into two ring slots, and each unit is
// hi.hi + lo.hi (first slot) + hi.lo (second slot); the epilogue writes dY as hi and lo, in shared memory and in the record.
// 64 KB ring + 128 KB activations + 32 KB operand = 224 KB: the trade exact mode's forward makes (one slot per hi/lo unit).
template <bool X3>
struct Smem {
  static constexpr int kNumSlots = X3 ? 2 : 4;
  using WeightRing = Ring<kNumSlots, kMaxUnitBytes>;
  static constexpr int kOffRing = 0;
  static constexpr int kOffAct = kOffRing + kNumSlots * kMaxUnitBytes;  // 4 K atoms x [128 rows x 128 B]
  static constexpr int kOffActLo = kOffAct + 4 * kTileM * 128;          // X3: the lo halves
  static constexpr int kOffOp = kOffActLo + (X3 ? 4 * kTileM * 128 : 0);  // d raw operand: [128 rows x 64 k] FP16, swizzled (k < 4 used)
  static constexpr int kOffOpLo = kOffOp + kTileM * 128;                // X3: its lo half
  static constexpr int kOffBars = kOffOpLo + (X3 ? kTileM * 128 : 0);
  static constexpr int kSmemBytes = kOffBars + 2 * kNumSlots * 8;
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB per-CTA shared memory limit");
};
static_assert(Smem<false>::kOffOp == 4 * kMaxUnitBytes + 4 * kTileM * 128, "the FP16 chain's map");

constexpr int kTileUnits = prog_units(kBwdStream);  // 28
__constant__ ProgTable c_prog = make_prog(kBwdStream);

// Epilogue of one 128-column accumulator half: masked gradient -> FP16, in place into the activation buffer and into the
// record image of dY(L).  X3: also its lo half, into act_lo and the lo record.
template <bool X3>
__device__ __forceinline__ void bwd_epi_half(const float (&acc)[64], int L, int c_base, const uint32_t* masks, uint8_t* act,
                                             uint8_t* act_lo, uint8_t* rec, int r0) {
  const int lane = threadIdx.x & 31, c = lane & 3;
  const int W = rec_width(L);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int R = r0 + 8 * hh;
    uint4 m = make_uint4(0u, 0u, 0u, 0u);
    if (masks) m = *reinterpret_cast<const uint4*>(masks + (L * 128 + R) * 8 + (c_base >> 5));
    const uint32_t mw[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int cc = 8 * j + 2 * c;  // column inside the half
      const uint32_t bits = mw[cc >> 5] >> (cc & 31);
      const float a0 = (bits & 1u) ? acc[4 * j + 2 * hh] : 0.f;
      const float a1 = (bits & 2u) ? acc[4 * j + 2 * hh + 1] : 0.f;
      const uint32_t h = pack_f16x2_inf(a0, a1);  // an overflow stays visible (non-finite gradients)
      const int col = c_base + cc;
      *reinterpret_cast<uint32_t*>(act + (col >> 6) * (kTileM * 128) + sw128_offset(R, col & 63)) = h;
      if (rec) {
        uint8_t* img = rec + rec_dy_off(L);
        *reinterpret_cast<uint16_t*>(img + img_offset(W, col, R)) = (uint16_t)(h & 0xFFFFu);
        *reinterpret_cast<uint16_t*>(img + img_offset(W, col + 1, R)) = (uint16_t)(h >> 16);
      }
      if constexpr (X3) {  // an inf hi leaves a non-finite lo: the overflow stays visible in hi + lo
        const float2 hf = unpack_f16x2(h);
        const uint32_t l = pack_f16x2_inf(a0 - hf.x, a1 - hf.y);
        *reinterpret_cast<uint32_t*>(act_lo + (col >> 6) * (kTileM * 128) + sw128_offset(R, col & 63)) = l;
        if (rec) {
          uint8_t* img = rec + kRecBytes + rec_dy_off(L);
          *reinterpret_cast<uint16_t*>(img + img_offset(W, col, R)) = (uint16_t)(l & 0xFFFFu);
          *reinterpret_cast<uint16_t*>(img + img_offset(W, col + 1, R)) = (uint16_t)(l >> 16);
        }
      }
    }
  }
}

template <bool X3>
__device__ __forceinline__ void chain_body(const ChainParams& p) {
  using M = Smem<X3>;
  constexpr int kOffRing = M::kOffRing, kOffAct = M::kOffAct, kOffOp = M::kOffOp, kOffBars = M::kOffBars;
  constexpr int NPART = X3 ? 2 : 1;
  constexpr size_t kRecStride = rec_stride(X3);
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t smem_base = smem_base_aligned(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  typename M::WeightRing ring(smem_base + kOffRing, smem_base + kOffBars);
  if (threadIdx.x == 0) ring.init();
  for (int i = threadIdx.x; i < NPART * kTileM * 128 / 16; i += kThreads)  // operand chunks 1..7 of every row stay zero (X3: both halves)
    reinterpret_cast<uint4*>(smem + kOffOp)[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();

  const int n_iter = (p.geom.n_units - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int tpu = p.geom.tiles_per_unit();
  const int n_tiles_cta = n_iter * tpu;

  if (warp < 4) {
    // ============================== weight producer ==============================
    reg_dec<kRegsLight>();
    if (warp == 0) {
      for (int j = 0; j < n_tiles_cta; ++j) {
        const uint8_t* base = p.wstream[p.geom.net_of(j % tpu)];
        const uint8_t* base_lo = X3 ? p.wstream_lo[p.geom.net_of(j % tpu)] : nullptr;
        for (int i = 0; i < kTileUnits; ++i) {
          const uint32_t w = c_prog.e[i].w;
          ring.produce(base + ((w & 0xFFFFFu) << 4), (w >> 20) * 128u);
          if constexpr (X3) ring.produce(base_lo + ((w & 0xFFFFFu) << 4), (w >> 20) * 128u);  // the unit's lo weights
        }
      }
    }
  } else {
    // ============================== row warpgroups ==============================
    reg_inc<kRegsRow>();
    const int q = warp & 3;
    const int row = q * 32 + lane;
    const int ch = (warp - 4) >> 2;  // == warpgroup
    const int wg = ch;
    const int r0 = 64 * wg + 16 * q + (lane >> 2);
    const float scale = p.scal[0];
    uint8_t* act = smem + kOffAct;

    for (int j = 0; j < n_tiles_cta; ++j) {
      const int unit = blockIdx.x + (j / tpu) * gridDim.x;
      const bool real = unit < p.geom.n_units;
      const size_t gt = p.geom.global_tile(unit, j % tpu);
      uint8_t* rec = real ? p.rec + gt * kRecStride : nullptr;
      // d raw of tile j -> FP16 operand row in shared memory (+ its transposed image for the weight-gradient kernel)
      if (ch == 0) {
        float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
        if (real) d = reinterpret_cast<const float4*>(p.draw)[gt * 128 + row];
        const uint32_t h01 = pack_f16x2_inf(d.x * scale, d.y * scale), h23 = pack_f16x2_inf(d.z * scale, d.w * scale);
        *reinterpret_cast<uint4*>(smem + kOffOp + row * 128 + ((0 ^ (row & 7)) << 4)) = make_uint4(h01, h23, 0u, 0u);
        if (real) {
          uint8_t* img = rec + kRecDRaw + img_row_base(16, row);
          const uint32_t cr = (uint32_t)((row & 63) >> 3);
          *reinterpret_cast<uint16_t*>(img + 0 * 128 + ((cr ^ 0u) << 4)) = (uint16_t)(h01 & 0xFFFFu);
          *reinterpret_cast<uint16_t*>(img + 1 * 128 + ((cr ^ 1u) << 4)) = (uint16_t)(h01 >> 16);
          *reinterpret_cast<uint16_t*>(img + 2 * 128 + ((cr ^ 2u) << 4)) = (uint16_t)(h23 & 0xFFFFu);
          *reinterpret_cast<uint16_t*>(img + 3 * 128 + ((cr ^ 3u) << 4)) = (uint16_t)(h23 >> 16);
        }
        if constexpr (X3) {  // the lo half of the scaled d raw: operand row and record image
          const float2 f01 = unpack_f16x2(h01), f23 = unpack_f16x2(h23);
          const uint32_t l01 = pack_f16x2_inf(d.x * scale - f01.x, d.y * scale - f01.y);
          const uint32_t l23 = pack_f16x2_inf(d.z * scale - f23.x, d.w * scale - f23.y);
          *reinterpret_cast<uint4*>(smem + M::kOffOpLo + row * 128 + ((0 ^ (row & 7)) << 4)) = make_uint4(l01, l23, 0u, 0u);
          if (real) {
            uint8_t* img = rec + kRecBytes + kRecDRaw + img_row_base(16, row);
            const uint32_t cr = (uint32_t)((row & 63) >> 3);
            *reinterpret_cast<uint16_t*>(img + 0 * 128 + ((cr ^ 0u) << 4)) = (uint16_t)(l01 & 0xFFFFu);
            *reinterpret_cast<uint16_t*>(img + 1 * 128 + ((cr ^ 1u) << 4)) = (uint16_t)(l01 >> 16);
            *reinterpret_cast<uint16_t*>(img + 2 * 128 + ((cr ^ 2u) << 4)) = (uint16_t)(l23 & 0xFFFFu);
            *reinterpret_cast<uint16_t*>(img + 3 * 128 + ((cr ^ 3u) << 4)) = (uint16_t)(l23 >> 16);
          }
        }
      } else if (real) {  // rows 4..15 of the image are zero
        uint8_t* img = rec + kRecDRaw + img_row_base(16, row);
        const uint32_t cr = (uint32_t)((row & 63) >> 3);
#pragma unroll
        for (int k = 4; k < 16; ++k) *reinterpret_cast<uint16_t*>(img + k * 128 + ((cr ^ (uint32_t)(k & 7)) << 4)) = 0;
        if constexpr (X3) {
#pragma unroll
          for (int k = 4; k < 16; ++k) *reinterpret_cast<uint16_t*>(img + kRecBytes + k * 128 + ((cr ^ (uint32_t)(k & 7)) << 4)) = 0;
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(kRowBarrier, kRowThreads);  // operand of tile j in place

      const uint32_t* masks = rec ? reinterpret_cast<const uint32_t*>(rec + kRecMask) : nullptr;
      int prog = 0;
      for (int s = 0; s < kBwdSteps; ++s) {
        const StepInfo si = bwd_step_info(s);
        const bool two = si.nh1 > 0;
        float acc0[64], acc1[64];
        for (int u = 0; u < si.k_atoms; ++u, ++prog) {
          const ProgEntry e = c_prog.e[prog];
          const uint32_t a = ((e.z & kUnitFromOperand) ? smem_base + kOffOp : smem_base + kOffAct + e.y * (kTileM * 128)) + 64 * wg * 128;
          const uint64_t ad = wgmma_desc_sw128(a);
          // X3: the lo half of the A operand, at the same place in the lo buffers
          const uint64_t al = X3 ? wgmma_desc_sw128(a + ((e.z & kUnitFromOperand) ? M::kOffOpLo - kOffOp : M::kOffActLo - kOffAct)) : 0;
#pragma unroll
          for (int part = 0; part < NPART; ++part) {  // X3: the unit's hi weights (hi.hi + lo.hi), then its lo weights (hi.lo)
            const uint32_t b = ring.wait_full();
            const uint64_t b0 = wgmma_desc_sw128(b), b1 = wgmma_desc_sw128(b + 128 * 128);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
              const uint32_t accf = (u | part | ks) ? 1u : 0u;
              wgmma_n128(acc0, ad + (uint64_t)(ks * 2), b0 + (uint64_t)(ks * 2), accf);
              if (two) wgmma_n128(acc1, ad + (uint64_t)(ks * 2), b1 + (uint64_t)(ks * 2), accf);
              if (X3 && part == 0) {
                wgmma_n128(acc0, al + (uint64_t)(ks * 2), b0 + (uint64_t)(ks * 2), 1u);
                if (two) wgmma_n128(acc1, al + (uint64_t)(ks * 2), b1 + (uint64_t)(ks * 2), 1u);
              }
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(acc0);
            reg_fence(acc1);
            ring.release();
          }
        }
        const int L = 8 - s;  // forward layer whose pre-activation gradient this step produces
        bwd_epi_half<X3>(acc0, L, 0, masks, act, smem + M::kOffActLo, rec, r0);
        if (two) bwd_epi_half<X3>(acc1, L, 128, masks, act, smem + M::kOffActLo, rec, r0);
        fence_proxy_async_smem();
        named_bar_sync(2 + wg, 128);
      }
      named_bar_sync(kRowBarrier, kRowThreads);  // the operand buffer is free for the next tile
    }
  }
}

__global__ void __launch_bounds__(kThreads, 1) chain_kernel(const __grid_constant__ ChainParams p) { chain_body<false>(p); }
// exact-grad mode: hi + lo operands end to end (a kernel of its own, so chain_kernel keeps its name and code)
__global__ void __launch_bounds__(kThreads, 1) chain_x3_kernel(const __grid_constant__ ChainParams p) { chain_body<true>(p); }

}  // namespace chain

// ================================================================================================
// 3. weight-gradient kernel
// ================================================================================================
namespace dw {

// Roles (nfb_pipeline.cuh): warp 0 producer, warpgroups 1 and 2 = output features [64w, 64w+64) of the job's 128 on wgmma,
// FP32 accumulators in registers over all tiles of the CTA, then stored (plain stores, one writer per element) into the
// CTA's partial slot, which grad_reduce_kernel adds into the accumulators in global memory.
constexpr int kStages = 4;
constexpr int kStageBytes = 16384 + 32768;       // one r-atom (64 sample rows): A [128 features x 128 B], B [<=256 features x 128 B]
using StageRing = Ring<kStages, kStageBytes>;
constexpr int kOffOnes = kStages * kStageBytes;  // [16 rows x 64 r]: row 0 = 1.0 (bias = column sums of dY)
constexpr int kOffBars = kOffOnes + 2048;
constexpr int kSmemBytes = kOffBars + 2 * kStages * 8;

struct Job {
  int a_off, a_rows, a_half;  // A image (M side): record offset, features in the image, which 128-feature half
  int b_off, b_rows;          // B image (N side): record offset, features (= MMA N)
  int bias_layer;             // >= 0: also accumulate column sums of A into the bias of this layer
  int out_off, out_ld, out_row0;
};
// Jobs are dealt to kGroups groups of CTAs; within a group every CTA runs the group's jobs over its own share of the tiles (fewer
// accumulator drains and partials than every CTA running every job).  The kernel streams each job's two images of every tile
// once, so the groups are balanced by BYTES per tile (172..200 KB each), and groups 2q / 2q+1 are the two 128-feature output
// halves of the SAME layers in the SAME order: they run on neighbouring CTAs over the same tiles at the same time, so the B
// image both need (the layer's whole input, 2/3 of a job's bytes) comes from HBM once and from L2 the second time.
constexpr int kNumJobs = 21;
constexpr int kGroups = 8;
struct JobTable { Job j[kNumJobs]; int group_begin[kGroups + 1]; };
constexpr Job half_job(int dy_layer, int h, int b_off, int b_rows, int bias_layer, int out_off) {
  return Job{rec_dy_off(dy_layer), 256, h, b_off, b_rows, bias_layer, out_off, b_rows, 128 * h};
}
constexpr JobTable make_jobs() {
  JobTable t{};
  int i = 0, g = 0;
  for (int h = 0; h < 2; ++h) {  // groups 0, 1: layers_xyz.1, .2
    t.group_begin[g++] = i;
    t.j[i++] = half_job(1, h, rec_x_off(0), 256, 1, kAcc1);
    t.j[i++] = half_job(2, h, rec_x_off(1), 256, 2, kAcc2);
  }
  for (int h = 0; h < 2; ++h) {  // groups 2, 3: layers_xyz.4, .5
    t.group_begin[g++] = i;
    t.j[i++] = half_job(4, h, rec_x_off(3), 256, 4, kAcc4);
    t.j[i++] = half_job(5, h, rec_x_off(4), 256, 5, kAcc5);
  }
  for (int h = 0; h < 2; ++h) {  // groups 4, 5: the skip layer (hidden part, then its PE part) and layers_xyz.0 (dY0 x PE)
    t.group_begin[g++] = i;
    t.j[i++] = half_job(3, h, rec_x_off(2), 256, -1, kAcc3b);
    t.j[i++] = half_job(3, h, kRecPE, 64, 3, kAcc3a);
    t.j[i++] = half_job(0, h, kRecPE, 64, 0, kAcc0);
  }
  t.group_begin[g++] = i;          // group 6: everything that reads dY6 or h5
  t.j[i++] = Job{rec_dy_off(6), 128, 0, rec_x_off(5), 256, 6, kAcc6, 256, 0};     // d M1
  t.j[i++] = Job{rec_dy_off(6), 128, 0, kRecPEd, 32, -1, kAcc6d, 32, 0};          // d layers_dir.0[:, 256:280]
  t.j[i++] = Job{rec_x_off(5), 256, 0, kRecDRaw, 16, -1, kAccSig, 16, 0};         // h5^T . d raw, first half
  t.group_begin[g++] = i;          // group 7: its second half and the rest of the direction branch
  t.j[i++] = Job{rec_x_off(5), 256, 1, kRecDRaw, 16, -1, kAccSig, 16, 128};
  t.j[i++] = Job{rec_dy_off(7), 128, 0, rec_x_off(6), 128, 7, kAcc7, 128, 0};
  t.j[i++] = Job{rec_dy_off(8), 128, 0, rec_x_off(7), 128, 8, kAcc8, 128, 0};
  t.j[i++] = Job{rec_x_off(8), 128, 0, kRecDRaw, 16, -1, kAcc9, 16, 0};           // g2^T . d raw
  t.group_begin[g] = i;
  return t;
}
static_assert(make_jobs().group_begin[kGroups] == kNumJobs, "job table");
static_assert(make_jobs().group_begin[5] - make_jobs().group_begin[4] == 3 && make_jobs().j[make_jobs().group_begin[4] + 1].b_off == kRecPE &&
                  make_jobs().j[make_jobs().group_begin[5] + 2].b_off == kRecPE && make_jobs().group_begin[6] - make_jobs().group_begin[5] == 3,
              "the PE-only weight-gradient launch runs jobs 1 and 2 of groups 4 and 5");
static_assert(make_jobs().j[make_jobs().group_begin[4] + 1].b_rows == 64 && make_jobs().j[make_jobs().group_begin[4] + 2].b_rows == 64 &&
                  make_jobs().j[make_jobs().group_begin[5] + 1].b_rows == 64 && make_jobs().j[make_jobs().group_begin[5] + 2].b_rows == 64,
              "dw_kernel<true> compiles run_job for the 64-row PE image only");
__constant__ JobTable c_jobs = make_jobs();

// Partial slots.  A part of the full launch writes every accumulator below kAccBRaw exactly once (the groups' output blocks tile
// it), so its slot mirrors that range.  A part of the PE-only launch writes four blocks only; its slot packs them as
// [dW0 | dW3a | db0 | db3] instead of reserving kAccFloats.
constexpr int kPeSlotFloats = 2 * 256 * 64 + 2 * 256;
__host__ __device__ constexpr int pe_slot_off(int a) {  // accumulator offset inside one of the four blocks -> slot offset
  return a < kAcc1 ? a : a < kAccB ? a - kAcc3a + 16384 : a < acc_bias_off(1) ? a - kAccB + 32768 : a - acc_bias_off(3) + 33024;
}
__host__ __device__ constexpr int pe_slot_to_acc(int e) {
  return e < 16384 ? e : e < 32768 ? kAcc3a + (e - 16384) : e < 33024 ? kAccB + (e - 32768) : acc_bias_off(3) + (e - 33024);
}
static_assert(pe_slot_off(kAcc3a) == 16384 && pe_slot_off(acc_bias_off(0)) == 32768 && pe_slot_off(acc_bias_off(3)) == 33024 &&
                  pe_slot_to_acc(pe_slot_off(acc_bias_off(3) + 255)) == acc_bias_off(3) + 255 && pe_slot_to_acc(32767) == kAcc3a + 16383,
              "PE-only slot layout");
static_assert(kAccBRaw % 4 == 0 && kPeSlotFloats % 4 == 0 && kAcc3a % 4 == 0 && kAccB % 4 == 0 && acc_bias_off(3) % 4 == 0,
              "grad_reduce_kernel adds float4s");

template <int N> __device__ __forceinline__ void mma_n(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t accf) {
  if constexpr (N == 16) wgmma_n16(d, a, b, accf);
  else if constexpr (N == 32) wgmma_n32(d, a, b, accf);
  else if constexpr (N == 64) wgmma_n64(d, a, b, accf);
  else wgmma_n128(d, a, b, accf);
}

// kPeOnly (input-gradient-only backward): only the four jobs that read the PE image — dW0, dW3a and with them the column sums
// db0, db3 that d latent and d expression need — i.e. groups 4 and 5 without their first (hidden-part) job.
constexpr int kPeGroup = 4, kPeGroups = 2;

// One job over the CTA's tiles j0..j1 for this warpgroup's 64 output features: NB = N of the B image (<= 128 per accumulator;
// 256 runs as two 128-column halves).  X3 (exact-grad mode, dw_x3_kernel): the records are the 2 MiB hi/lo ones and every
// r-atom takes three stages, (A hi, B hi), (A hi, B lo), (A lo, B hi), with the same MMAs on each; the bias column sums take
// A hi (first stage) and A lo (third) against the ones row.  The result and the bias column sums go to the CTA's partial
// slot; where exactly is worked out only after the tile loop, from the parameter block, so no address stays live in
// registers across it.
template <bool kPeOnly, bool X3, int NB>
__device__ __forceinline__ void run_job(const DwParams& p, const Job& J, int j0, int j1, uint32_t smem_base, StageRing& ring,
                                        int wg, int lane) {
  constexpr int NA = NB > 128 ? 128 : NB;
  constexpr int NH = NB > 128 ? 2 : 1;
  constexpr int NPART = X3 ? 3 : 1;
  float acc[NH][NA / 2];
  float accb[8];
  const bool bias = J.bias_layer >= 0;
  const uint64_t ones = wgmma_desc_sw128(smem_base + kOffOnes);
  for (int j = j0; j < j1; ++j) {
    for (int a = 0; a < 2; ++a) {
#pragma unroll
      for (int part = 0; part < NPART; ++part) {
        const uint32_t sa = ring.wait_full(), sb = sa + 16384;
        const uint64_t ad = wgmma_desc_sw128(sa + 64 * wg * 128);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint32_t accf = ((j - j0) | a | part | ks) ? 1u : 0u;
#pragma unroll
          for (int h = 0; h < NH; ++h) mma_n<NA>(acc[h], ad + (uint64_t)(ks * 2), wgmma_desc_sw128(sb + h * 16384) + (uint64_t)(ks * 2), accf);
          if (bias && part != 1) wgmma_n16(accb, ad + (uint64_t)(ks * 2), ones + (uint64_t)(ks * 2), accf);  // A hi, A lo
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int h = 0; h < NH; ++h) reg_fence(acc[h]);
        reg_fence(accb);
        ring.release();
      }
    }
  }
  constexpr int kG = kPeOnly ? kPeGroups : kGroups;
  float* slot = p.ws + (size_t)(blockIdx.x / kG) * p.ws_stride;  // this (network, part)'s partial
  const int bias_acc = bias ? acc_bias_off(J.bias_layer) : 0;
  const int out_off = kPeOnly ? pe_slot_off(J.out_off) : J.out_off, bias_off = kPeOnly ? pe_slot_off(bias_acc) : bias_acc;
  const float inv = p.scal[1];
  const int c = lane & 3, r0 = 64 * wg + 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int R = r0 + 8 * hh;
    float* out = slot + out_off + (size_t)(J.out_row0 + R) * J.out_ld;
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int jj = 0; jj < NA / 8; ++jj) {
        const int col = h * 128 + 8 * jj + 2 * c;
        *reinterpret_cast<float2*>(out + col) = make_float2(acc[h][4 * jj + 2 * hh] * inv, acc[h][4 * jj + 2 * hh + 1] * inv);
      }
    if (bias && c == 0) slot[bias_off + J.out_row0 + R] = accb[2 * hh] * inv;
  }
}

template <bool kPeOnly, bool X3>
__device__ __forceinline__ void dw_body(const DwParams& p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t smem_base = smem_base_aligned(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // this CTA: network x job group (blockIdx.x % kGroups) x a contiguous share of the network's tiles
  constexpr int kG = kPeOnly ? kPeGroups : kGroups;
  const int group = (kPeOnly ? kPeGroup : 0) + (int)blockIdx.x % kG;
  int part = (int)blockIdx.x / kG;
  const int net = (part >= p.parts[0]) ? 1 : 0;
  if (net) part -= p.parts[0];
  const int parts = p.parts[net];
  const int t_cnt = p.geom.tile_count(net);
  const int total = p.geom.n_units * t_cnt;
  const int per = (total + parts - 1) / parts;
  const int j0 = part * per;
  const int j1 = min(total, j0 + per);
  if (part >= parts || j0 >= j1) return;  // uniform for the whole CTA
  const int job0 = c_jobs.group_begin[group] + (kPeOnly ? 1 : 0), job1 = c_jobs.group_begin[group + 1];

  StageRing ring(smem_base, smem_base + kOffBars);
  if (threadIdx.x == 0) ring.init();
  for (int i = threadIdx.x; i < 2048 / 4; i += kThreads)  // row 0 (first 128 bytes) = FP16 ones, rows 1..15 = 0
    reinterpret_cast<uint32_t*>(smem + kOffOnes)[i] = (i < 32) ? 0x3C003C00u : 0u;
  fence_proxy_async_smem();
  __syncthreads();

  auto tile_rec = [&](int j) -> const uint8_t* {
    const int u = j / t_cnt, t = j - u * t_cnt;
    return p.rec + p.geom.global_tile(u, net, t) * rec_stride(X3);
  };

  if (warp < 4) {
    // ============================== producer ==============================
    reg_dec<kRegsLight>();
    if (warp == 0) {
      for (int job = job0; job < job1; ++job) {
        const Job J = c_jobs.j[job];
        const uint32_t b_bytes = (uint32_t)J.b_rows * 128u;
        for (int j = j0; j < j1; ++j) {
          const uint8_t* rec = tile_rec(j);
          for (int a = 0; a < 2; ++a) {  // one stage = the A and the B image of one r-atom (X3: three stages, lo at +kRecBytes)
            const uint8_t* A = rec + J.a_off + a * J.a_rows * 128 + J.a_half * 16384;
            const uint8_t* B = rec + J.b_off + a * J.b_rows * 128;
            ring.produce(A, 16384, 16384, B, b_bytes);
            if constexpr (X3) {
              ring.produce(A, 16384, 16384, B + kRecBytes, b_bytes);
              ring.produce(A + kRecBytes, 16384, 16384, B, b_bytes);
            }
          }
        }
      }
    }
  } else {
    // ============================== MMA + epilogue warpgroups ==============================
    reg_inc<kRegsRow>();
    const int wg = (warp - 4) >> 2;
    for (int job = job0; job < job1; ++job) {
      const Job J = c_jobs.j[job];
      if constexpr (kPeOnly) {  // both PE jobs multiply by the 64-row PE image: only that shape is compiled in
        run_job<kPeOnly, X3, 64>(p, J, j0, j1, smem_base, ring, wg, lane);
        continue;
      }
      switch (J.b_rows) {
        case 16: run_job<kPeOnly, X3, 16>(p, J, j0, j1, smem_base, ring, wg, lane); break;
        case 32: run_job<kPeOnly, X3, 32>(p, J, j0, j1, smem_base, ring, wg, lane); break;
        case 64: run_job<kPeOnly, X3, 64>(p, J, j0, j1, smem_base, ring, wg, lane); break;
        case 128: run_job<kPeOnly, X3, 128>(p, J, j0, j1, smem_base, ring, wg, lane); break;
        default: run_job<kPeOnly, X3, 256>(p, J, j0, j1, smem_base, ring, wg, lane); break;
      }
    }
  }
}

template <bool kPeOnly>
__global__ void __launch_bounds__(kThreads, 1) dw_kernel(const __grid_constant__ DwParams p) { dw_body<kPeOnly, false>(p); }
// exact-grad mode: hi + lo records (a kernel of its own, so dw_kernel keeps its name)
template <bool kPeOnly>
__global__ void __launch_bounds__(kThreads, 1) dw_x3_kernel(const __grid_constant__ DwParams p) { dw_body<kPeOnly, true>(p); }

}  // namespace dw

// ================================================================================================
// 3b. fixed-order reduction of the partials
// ================================================================================================
struct ReduceParams {
  float* acc[2];
  const float* ws;          // the weight-gradient partials (DwParams::ws)
  int stride;               // floats per slot
  int first1, filled[2];    // network i's partials, in part order: slots [0, filled[0]) and [first1, first1 + filled[1])
  int net0, nets;           // the networks that have partials: [net0, net0 + nets)
  int pe_only;              // slots in the compact PE-only layout
  int dw_blocks;            // blocks [0, dw_blocks) add the partials; block dw_blocks + pass sums bsum[pass]
  const float* bsum;        // [pass][n_rays][4] (CompBwdParams::bsum)
  int n_rays;
};
constexpr int kBsumThreads = 256;
__global__ void __launch_bounds__(256) grad_reduce_kernel(const ReduceParams r) {
  if ((int)blockIdx.x >= r.dw_blocks) {
    // d b_rgb, d b_sigma of pass `pass`: thread t sums rays t, t + 256, ... in order, then a fixed tree over the threads
    __shared__ float4 red[kBsumThreads];
    const int pass = (int)blockIdx.x - r.dw_blocks;
    const float4* b = reinterpret_cast<const float4*>(r.bsum) + (size_t)pass * r.n_rays;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int g = threadIdx.x; g < r.n_rays; g += kBsumThreads) {
      const float4 t = b[g];
      s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
    }
    red[threadIdx.x] = s;
    __syncthreads();
#pragma unroll
    for (int h = kBsumThreads / 2; h > 0; h >>= 1) {
      if ((int)threadIdx.x < h) {
        const float4 t = red[threadIdx.x + h];
        float4& u = red[threadIdx.x];
        u.x += t.x; u.y += t.y; u.z += t.z; u.w += t.w;
      }
      __syncthreads();
    }
    if (threadIdx.x < 4) {
      const float4 t = red[0];
      (pass ? r.acc[1] : r.acc[0])[kAccBRaw + threadIdx.x] += threadIdx.x == 0 ? t.x : threadIdx.x == 1 ? t.y : threadIdx.x == 2 ? t.z : t.w;
    }
    return;
  }
  // acc += p_0 + p_1 + ... one float4 per thread, strictly left to right: ((acc + p_0) + p_1) + ...
  const int nv = r.stride >> 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < r.nets * nv; i += r.dw_blocks * blockDim.x) {
    const int net = r.net0 + (i >= nv ? 1 : 0), v = i >= nv ? i - nv : i;
    const int n = net ? r.filled[1] : r.filled[0];  // (no dynamic index into the parameter block: no local copy)
    float4* a = reinterpret_cast<float4*>((net ? r.acc[1] : r.acc[0]) + (r.pe_only ? dw::pe_slot_to_acc(4 * v) : 4 * v));
    const float4* p = reinterpret_cast<const float4*>(r.ws + (size_t)(net ? r.first1 : 0) * r.stride) + v;
    float4 s = *a;
#pragma unroll 4
    for (int k = 0; k < n; ++k) {
      const float4 t = p[(size_t)k * nv];
      s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
    }
    *a = s;
  }
}

// ================================================================================================
// 4. finalize: accumulators (folded parametrisation) -> reference parameter gradients
// ================================================================================================
struct FinArgs {
  const float* p[26];  // FP32 master parameters (device)
  float* g[26];        // gradient outputs (device; layers_dir.3.* may be null)
  const float* acc;    // this network's accumulators
  const float* cond;   // [108] = [expression / 3 ; latent]
};
__host__ __device__ __forceinline__ int fin_numel(int t) {
  switch (t) {
    case 0: return 256 * 171;
    case 6: return 256 * 427;
    case 2: case 4: case 8: case 10: case 12: return 65536;
    case 1: case 3: case 5: case 7: case 9: case 11: case 13: case 14: return 256;
    case 15: return 1;
    case 16: return 128 * 280;
    case 18: case 20: return 128 * 128;
    case 17: case 19: case 21: return 128;
    case 24: return 3 * 128;
    case 25: return 3;
    default: return 0;  // layers_dir.3.*: unused by the forward (models.py:257) -> no gradient
  }
}
// ONE launch finishes both networks: blockIdx.y = network; blockIdx.x walks the 26 tensors back to back in 256-element blocks
// (2.2 k blocks per network instead of a 427 x 26 grid that is mostly empty); the last block of network 0 computes d latent.
// The two blocks after the last tensor of network 0 compute d latent and d expression.
struct FinAll { FinArgs net[2]; int nets; float* latent_out; float* expr_out; };
__device__ __forceinline__ int fin_blocks(int t) { return (fin_numel(t) + 255) >> 8; }
__device__ void latent_grad_block(const FinAll& f);
__device__ void expr_grad_block(const FinAll& f);
__global__ void __launch_bounds__(256) finalize_kernel(const FinAll f) {
  const FinArgs& a = f.net[blockIdx.y];
  int b = blockIdx.x, t = 0;
  while (t < 26 && b >= fin_blocks(t)) { b -= fin_blocks(t); ++t; }
  if (t == 26) {  // the blocks after the last tensor
    if (blockIdx.y == 0 && b == 0 && f.latent_out) latent_grad_block(f);
    if (blockIdx.y == 0 && b == 1 && f.expr_out) expr_grad_block(f);
    return;
  }
  const int e = b * 256 + threadIdx.x;
  if (e >= fin_numel(t) || a.g[t] == nullptr) return;
  const float* acc = a.acc;
  const float* b6 = acc + acc_bias_off(6);
  const float dbs = acc[kAccBRaw + 3];  // d (fc_alpha.bias + wa . bf)
  float v = 0.f;
  switch (t) {
    case 0: {
      const int n = e / 171, k = e - n * 171;
      v = (k < kDimXyz) ? acc[kAcc0 + n * 64 + k] : acc[acc_bias_off(0) + n] * a.cond[k - kDimXyz];
      break;
    }
    case 6: {
      const int n = e / 427, k = e - n * 427;
      v = (k < kDimXyz) ? acc[kAcc3a + n * 64 + k]
          : (k < kDimXyz + kDimCond) ? acc[acc_bias_off(3) + n] * a.cond[k - kDimXyz]
                                     : acc[kAcc3b + n * 256 + (k - kDimXyz - kDimCond)];
      break;
    }
    case 1: v = acc[acc_bias_off(0) + e]; break;
    case 2: v = acc[kAcc1 + e]; break;
    case 3: v = acc[acc_bias_off(1) + e]; break;
    case 4: v = acc[kAcc2 + e]; break;
    case 5: v = acc[acc_bias_off(2) + e]; break;
    case 7: v = acc[acc_bias_off(3) + e]; break;
    case 8: v = acc[kAcc4 + e]; break;
    case 9: v = acc[acc_bias_off(4) + e]; break;
    case 10: v = acc[kAcc5 + e]; break;
    case 11: v = acc[acc_bias_off(5) + e]; break;
    case 12: {  // fc_feat.weight[j][k] = sum_i Wd0[i][j] dM1[i][k] + wa[j] dm2[k]
      const int j = e >> 8, k = e & 255;
      float s = a.p[14][j] * acc[kAccSig + k * 16 + 3];
      for (int i = 0; i < 128; ++i) s = fmaf(a.p[16][i * 280 + j], acc[kAcc6 + i * 256 + k], s);
      v = s;
      break;
    }
    case 13: {  // fc_feat.bias[j] = sum_i Wd0[i][j] db6[i] + wa[j] dbs
      float s = a.p[14][e] * dbs;
      for (int i = 0; i < 128; ++i) s = fmaf(a.p[16][i * 280 + e], b6[i], s);
      v = s;
      break;
    }
    case 14: return;  // fc_alpha.weight: 256 dot products of length 256 -> fin_dir0_kernel (one warp each, coalesced)
    case 15: v = dbs; break;
    case 16: {  // layers_dir.0.weight[i][j]: j < 256: sum_k dM1[i][k] Wf[j][k] + db6[i] bf[j]; else direction columns
      const int i = e / 280, j = e - i * 280;
      if (j < 256) return;  // written by fin_dir0_kernel (one warp per element, coalesced along k)
      v = acc[kAcc6d + i * 32 + (j - 256)];
      break;
    }
    case 17: v = b6[e]; break;
    case 18: v = acc[kAcc7 + e]; break;
    case 19: v = acc[acc_bias_off(7) + e]; break;
    case 20: v = acc[kAcc8 + e]; break;
    case 21: v = acc[acc_bias_off(8) + e]; break;
    case 24: { const int n = e >> 7, k = e & 127; v = acc[kAcc9 + k * 16 + n]; break; }
    case 25: v = acc[kAccBRaw + e]; break;
    default: break;
  }
  a.g[t][e] = v;
}

// layers_dir.0.weight[i][j], j < 256:  sum_k dM1[i][k] Wf[j][k] + db6[i] bf[j].  One warp per output element, lanes along k.
__global__ void fin_dir0_kernel(const FinAll f) {
  const FinArgs& a = f.net[blockIdx.y];
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= 128 * 256) {  // fc_alpha.weight[0][j] = sum_k dm2[k] Wf[j][k] + dbs bf[j]
    const int j = w - 128 * 256;
    if (j >= 256 || a.g[14] == nullptr) return;
    const float* wf = a.p[12] + j * 256;
    float s = 0.f;
#pragma unroll
    for (int k = lane; k < 256; k += 32) s = fmaf(a.acc[kAccSig + k * 16 + 3], wf[k], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) a.g[14][j] = s + a.acc[kAccBRaw + 3] * a.p[13][j];
    return;
  }
  const int i = w >> 8, j = w & 255;
  const float* dm1 = a.acc + kAcc6 + i * 256;
  const float* wf = a.p[12] + j * 256;
  float s = 0.f;
#pragma unroll
  for (int k = lane; k < 256; k += 32) s = fmaf(dm1[k], wf[k], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) a.g[16][i * 280 + j] = s + a.acc[acc_bias_off(6) + i] * a.p[13][j];
}

// d latent[j] = sum over networks, n of W0[n][139 + j] db0[n] + W3[n][139 + j] db3[n]
__device__ void latent_grad_block(const FinAll& f) {  // one block of 256 threads: thread = (n-chunk of 32 rows, j)
  __shared__ float part[8][kDimLatent];
  const int j = threadIdx.x & 31, c = threadIdx.x >> 5;
  float s = 0.f;
  for (int net = 0; net < f.nets; ++net) {
    const float* b0 = f.net[net].acc + acc_bias_off(0);
    const float* b3 = f.net[net].acc + acc_bias_off(3);
    const float* w0 = f.net[net].p[0];
    const float* w3 = f.net[net].p[6];
    for (int n = c * 32; n < c * 32 + 32; ++n) {
      s = fmaf(w0[n * 171 + kDimXyz + kDimExpr + j], b0[n], s);
      s = fmaf(w3[(size_t)n * 427 + kDimXyz + kDimExpr + j], b3[n], s);
    }
  }
  part[c][j] = s;
  __syncthreads();
  if (c == 0) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += part[k][j];
    f.latent_out[j] = t;
  }
}

// d expression[j] = (1/3) sum over networks, n of W0[n][63 + j] db0[n] + W3[n][63 + j] db3[n]  (cond = [expression / 3 ; latent]).
// One block of 256 threads: thread = (n-chunk of 64 rows, j); 76 of every 128 threads work.
__device__ void expr_grad_block(const FinAll& f) {
  __shared__ float part[2][kDimExpr];
  const int j = threadIdx.x & 127, c = threadIdx.x >> 7;  // c in {0, 1}: rows [128c, 128c + 128)
  float s = 0.f;
  if (j < kDimExpr) {
    for (int net = 0; net < f.nets; ++net) {
      const float* b0 = f.net[net].acc + acc_bias_off(0);
      const float* b3 = f.net[net].acc + acc_bias_off(3);
      const float* w0 = f.net[net].p[0];
      const float* w3 = f.net[net].p[6];
      for (int n = c * 128; n < c * 128 + 128; ++n) {
        s = fmaf(w0[n * 171 + kDimXyz + j], b0[n], s);
        s = fmaf(w3[(size_t)n * 427 + kDimXyz + j], b3[n], s);
      }
    }
    part[c][j] = s;
  }
  __syncthreads();
  if (c == 0 && j < kDimExpr) f.expr_out[j] = (part[0][j] + part[1][j]) * (1.f / 3.f);
}

// Input-gradient-only backward: the latent and expression blocks of finalize_kernel alone.
__global__ void __launch_bounds__(256) cond_grad_kernel(const FinAll f) {
  if (blockIdx.x == 0 && f.latent_out) latent_grad_block(f);
  if (blockIdx.x == 1 && f.expr_out) expr_grad_block(f);
}

// ================================================================================================
// 4b. multi-frame conditioning (nfb_render_backward_frames)
// ================================================================================================
// Per-frame bias sums db0_f, db3_f = the sums of dY0, dY3 over the sample rows of frame f's rays, in a fixed order and without
// atomics: per ray (samples ascending) from the dY images the dX chain left in the tile records, then per frame over the rays in
// ascending order, added to the running sums of earlier chunks.
// raysum_kernel: block = (ray, pass), thread = column (0..255: dY0, 256..511: dY3).
// X3 (raysum_x3_kernel, exact-grad mode): each dY is hi + lo of the 2 MiB record.
template <bool X3>
__device__ __forceinline__ float rec_dy(const uint8_t* img, int off) {
  float v = __half2float(*reinterpret_cast<const __half*>(img + off));
  if constexpr (X3) v += __half2float(*reinterpret_cast<const __half*>(img + kRecBytes + off));  // exact in FP32
  return v;
}
template <bool X3>
__device__ __forceinline__ void raysum_body(const FrameSumParams& p) {
  const int g = blockIdx.x, pass = blockIdx.y, t = threadIdx.x;
  const int L = t < 256 ? 0 : 3, n = t & 255;
  const TileGeom::RayRows rows = p.geom.ray_rows(pass, g);
  float s = 0.f;
  for (int i = 0; i < rows.S; ++i) {
    const size_t slot = rows.slot(i);
    const uint8_t* img = p.rec + (slot >> 7) * rec_stride(X3) + rec_dy_off(L);
    s += rec_dy<X3>(img, img_offset(256, n, (int)(slot & 127)));
  }
  p.raysum[((size_t)pass * p.geom.n_rays + g) * kFrameRows + t] = s * p.scal[1];
}
__global__ void __launch_bounds__(kFrameRows) raysum_kernel(const FrameSumParams p) { raysum_body<false>(p); }
__global__ void __launch_bounds__(kFrameRows) raysum_x3_kernel(const FrameSumParams p) { raysum_body<true>(p); }
// framesum_kernel: block = (frame, pass), thread = column.  Per batch of 512 rays the block first compacts the frame's rays into a
// list (ballot + warp prefix: ascending ray order, no atomics), then every thread adds its column over that list.  A block reads
// each frame slot once (n / 512 steps) and sums only its own frame's rays, so the launch costs O(F n / 512 + 512 n), not O(F n 512).
__global__ void __launch_bounds__(kFrameRows) framesum_kernel(const FrameSumParams p) {
  constexpr int kWarps = kFrameRows / 32;
  __shared__ int list[kFrameRows];
  __shared__ int wcount[kWarps];
  const int f = blockIdx.x, pass = blockIdx.y, t = threadIdx.x, n = p.geom.n_rays, lane = t & 31, w = t >> 5;
  const float* rs = p.raysum + (size_t)pass * n * kFrameRows + t;
  float s = 0.f;
  for (int b = 0; b < n; b += kFrameRows) {
    const bool hit = b + t < n && p.frame[b + t] == f;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) wcount[w] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
    for (int i = 0; i < kWarps; ++i) {
      const int c = wcount[i];
      before += i < w ? c : 0;
      total += c;
    }
    if (hit) list[before + __popc(m & ((1u << lane) - 1u))] = b + t;
    __syncthreads();
    for (int i = 0; i < total; ++i) s += rs[(size_t)list[i] * kFrameRows];
    __syncthreads();
  }
  float* out = p.fsum + ((size_t)f * 2 + pass) * kFrameRows + t;
  *out = *out + s;
}

// From the per-frame sums, blockIdx.y selects the work:
//   y = 0: block f = frame f's d latent [32] and d expression [76] (the sums latent_grad_block / expr_grad_block form from the totals)
//   y = 1 + net: the conditioning columns of network net, W0[:, 63:171] and W3[:, 63:171]: sum_f db_f[n] c_f[j], frames ascending
struct FramesGradArgs {
  const float* p[2][2];  // [net] = {layers_xyz.0.weight, layers_xyz.3.weight}
  float* g[2][2];        // [net] = their gradients (null: no parameter gradients)
  const float *fsum, *fcond;
  int n_frames, nets;
  float *latent_out, *expr_out;
};
__global__ void __launch_bounds__(256) frames_grad_kernel(const FramesGradArgs a) {
  const int t = threadIdx.x;
  if (blockIdx.y == 0) {
    const int f = blockIdx.x;
    if (f >= a.n_frames) return;
    __shared__ float part[2][128];
    // thread = (half c of the 256 rows, j < 108 of [expression ; latent]), then the two halves in a fixed order
    const int j = t & 127, c = t >> 7;
    float s = 0.f;
    if (j < kDimCond)
      for (int net = 0; net < a.nets; ++net) {
        const float* b0 = a.fsum + ((size_t)f * 2 + net) * kFrameRows;
        const float* b3 = b0 + 256;
        const float* w0 = a.p[net][0];
        const float* w3 = a.p[net][1];
        for (int n = c * 128; n < c * 128 + 128; ++n) {
          s = fmaf(w0[n * 171 + kDimXyz + j], b0[n], s);
          s = fmaf(w3[(size_t)n * 427 + kDimXyz + j], b3[n], s);
        }
      }
    part[c][j] = s;
    __syncthreads();
    if (c == 0 && j < kDimCond) {
      const float v = part[0][j] + part[1][j];
      if (j < kDimExpr) { if (a.expr_out) a.expr_out[(size_t)f * kDimExpr + j] = v * (1.f / 3.f); }
      else if (a.latent_out) a.latent_out[(size_t)f * kDimLatent + j - kDimExpr] = v;
    }
    return;
  }
  const int net = blockIdx.y - 1;
  const int e = blockIdx.x * 256 + t;  // (layer L of {0, 3}, row n, column j)
  if (net >= a.nets || e >= 2 * 256 * kDimCond || !a.g[net][0]) return;
  const int L = e / (256 * kDimCond), r = e - L * 256 * kDimCond, n = r / kDimCond, j = r - n * kDimCond;
  float v = 0.f;
  for (int f = 0; f < a.n_frames; ++f)
    v = fmaf(a.fsum[((size_t)f * 2 + net) * kFrameRows + 256 * L + n], a.fcond[(size_t)f * kDimCond + j], v);
  if (L == 0) a.g[net][0][n * 171 + kDimXyz + j] = v;
  else a.g[net][1][(size_t)n * 427 + kDimXyz + j] = v;
}

// ================================================================================================
// 5. input gradients (rays, direction, background; nfb_render_backward_ex)
// ================================================================================================
// Per sample row of every tile (after the dX chain, which left dY0, dY3 and dY6 in the tile record):
//   dPE  = W0[:, :63]^T dY0 + W3[:, :63]^T dY3,   dPEd[6j], dPEd[6j+3] = Wd0[:, 256+6j]^T dY6, Wd0[:, 259+6j]^T dY6
//   dp   = dPE[0:3] + sum_j 2^j (cos(2^j p) dPE[3+6j:6+6j] - sin(2^j p) dPE[6+6j:9+6j])        p = o + d z
//   dv0  = sum_j 2^j (cos(2^j v0) dPEd[6j] - sin(2^j v0) dPEd[6j+3])                          v0 = dir_z or d.z
// written as one float4 (dp, dv0) per row.  SIMT with the FP32 master columns in shared memory: thread = (row, quarter of the
// 64 PE columns); a warp is 32 rows of one quarter, so every weight load is a broadcast.  The chain and weight-gradient kernels
// are untouched by this (their parameter-only code stays as it is); the cost is one extra pass over 160 KB of each record.
namespace ing {
constexpr int kThreadsRow = 512;
constexpr int kOffW3 = 256 * 64 * 4;
constexpr int kOffWd = 2 * kOffW3;              // [128][8]: the v0 columns sin/cos of the 4 frequencies
constexpr int kOffRed = kOffWd + 128 * 8 * 4;   // [4][128] float4
constexpr int kSmemBytes = kOffRed + 4 * 128 * 16;

// X3 (row_x3_kernel, exact-grad mode): dY0, dY3 and dY6 are hi + lo of the 2 MiB record.
template <bool X3>
__device__ __forceinline__ void row_body(const InGradRowParams& p) {
  extern __shared__ __align__(16) uint8_t smem[];
  float* w0s = reinterpret_cast<float*>(smem);
  float* w3s = reinterpret_cast<float*>(smem + kOffW3);
  float* wds = reinterpret_cast<float*>(smem + kOffWd);
  float4* red = reinterpret_cast<float4*>(smem + kOffRed);
  const int net = (int)blockIdx.x >= p.parts[0] ? 1 : 0;
  const int part = (int)blockIdx.x - (net ? p.parts[0] : 0);
  const int parts = p.parts[net];
  for (int i = threadIdx.x; i < 256 * 64; i += kThreadsRow) {
    const int n = i >> 6, k = i & 63;
    w0s[i] = k < kDimXyz ? p.w0[net][n * 171 + k] : 0.f;
    w3s[i] = k < kDimXyz ? p.w3[net][(size_t)n * 427 + k] : 0.f;
  }
  for (int i = threadIdx.x; i < 128 * 8; i += kThreadsRow) {
    const int n = i >> 3, c = i & 7;
    wds[i] = p.wd0[net][n * 280 + 256 + 6 * (c >> 1) + 3 * (c & 1)];
  }
  __syncthreads();
  const int row = threadIdx.x & 127, kq = threadIdx.x >> 7;
  const float inv = p.scal[1];
  const int t_cnt = p.geom.tile_count(net);
  const int S = p.geom.samples(net);
  const float* zp = net ? p.z_f : p.z_c;
  const int total = p.geom.n_units * t_cnt;
  for (int j = part; j < total; j += parts) {
    const int unit = j / t_cnt, tl = j - unit * t_cnt;
    const size_t gt = p.geom.global_tile(unit, net, tl);
    const uint8_t* rec = p.rec + gt * rec_stride(X3);
    float acc[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) acc[k] = 0.f;
#pragma unroll 1
    for (int L = 0; L < 2; ++L) {
      const uint8_t* img = rec + rec_dy_off(3 * L);
      const float* ws = (L ? w3s : w0s) + 16 * kq;
#pragma unroll 4
      for (int n = 0; n < 256; ++n) {
        const float dy = rec_dy<X3>(img, img_offset(256, n, row));
        const float4* w4 = reinterpret_cast<const float4*>(ws + n * 64);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 w = w4[q];
          acc[4 * q] = fmaf(w.x, dy, acc[4 * q]); acc[4 * q + 1] = fmaf(w.y, dy, acc[4 * q + 1]);
          acc[4 * q + 2] = fmaf(w.z, dy, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(w.w, dy, acc[4 * q + 3]);
        }
      }
    }
    float ds = 0.f, dc = 0.f;  // dPEd of sin / cos of frequency kq
    {
      const uint8_t* img = rec + rec_dy_off(6);
#pragma unroll 4
      for (int n = 0; n < 128; ++n) {
        const float dy = rec_dy<X3>(img, img_offset(128, n, row));
        ds = fmaf(wds[n * 8 + 2 * kq], dy, ds);
        dc = fmaf(wds[n * 8 + 2 * kq + 1], dy, dc);
      }
    }
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    const TileGeom::Row rw = p.geom.row(net, tl, row);
    const int g = p.geom.ray_index(unit, rw.ray);
    if (rw.used && g < p.geom.n_rays) {
      const float z = zp[(size_t)g * S + rw.sample];
      const float* ray = p.ray + 7 * (size_t)g;
      // p = o + d z rounded twice, exactly as the forward encoded it (one fused rounding moves p by an ulp at times, and the
      // 2^9 frequency turns that into a phase error)
      const float px = __fadd_rn(ray[0], __fmul_rn(ray[3], z)), py = __fadd_rn(ray[1], __fmul_rn(ray[4], z)),
                  pz = __fadd_rn(ray[2], __fmul_rn(ray[5], z));
#pragma unroll
      for (int kk = 0; kk < 16; ++kk) {
        const int k = 16 * kq + kk;
        if (k >= kDimXyz) continue;
        const float a = acc[kk];
        if (k < 3) {
          if (k == 0) r.x += a; else if (k == 1) r.y += a; else r.z += a;
          continue;
        }
        const int kp = k - 3, fj = kp / 6, wi = kp - 6 * fj, comp = wi % 3;
        const float f = (float)(1 << fj);
        const float x = f * (comp == 0 ? px : comp == 1 ? py : pz);
        const float v = f * a * (wi < 3 ? cosf(x) : -sinf(x));
        if (comp == 0) r.x += v; else if (comp == 1) r.y += v; else r.z += v;
      }
      const float f = (float)(1 << kq), x = f * ray[6];
      r.w = f * (cosf(x) * ds - sinf(x) * dc);
    }
    red[kq * 128 + row] = r;
    __syncthreads();
    if (kq == 0) {
      float4 s = red[row];
#pragma unroll
      for (int q = 1; q < 4; ++q) {
        const float4 t = red[q * 128 + row];
        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
      }
      s.x *= inv; s.y *= inv; s.z *= inv; s.w *= inv;
      reinterpret_cast<float4*>(p.out)[gt * 128 + row] = s;
    }
    __syncthreads();
  }
}
__global__ void __launch_bounds__(kThreadsRow, 1) row_kernel(const InGradRowParams p) { row_body<false>(p); }
__global__ void __launch_bounds__(kThreadsRow, 1) row_x3_kernel(const InGradRowParams p) { row_body<true>(p); }

// One warp per ray: sums the row float4s of both passes (lane-strided over the samples, then a butterfly: deterministic, no
// atomics), d o += dp, d d += z dp, and adds the |d| term of the compositing and the background term.
__global__ void __launch_bounds__(256) ray_kernel(const InGradRayParams p) {
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= p.geom.n_rays) return;  // whole warps
  const int npass = p.geom.passes();
  float so0 = 0.f, so1 = 0.f, so2 = 0.f, sd0 = 0.f, sd1 = 0.f, sd2 = 0.f, sv = 0.f;
  if (p.rows) {
    for (int pass = 0; pass < npass; ++pass) {
      const int S = p.geom.samples(pass);
      const float* z = (pass ? p.z_f : p.z_c) + (size_t)g * S;
      const TileGeom::RayRows rows = p.geom.ray_rows(pass, g);
      for (int i = lane; i < S; i += 32) {
        const float4 v = reinterpret_cast<const float4*>(p.rows)[rows.slot(i)];
        const float zi = z[i];
        so0 += v.x; so1 += v.y; so2 += v.z;
        sd0 = fmaf(zi, v.x, sd0); sd1 = fmaf(zi, v.y, sd1); sd2 = fmaf(zi, v.z, sd2);
        sv += v.w;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      so0 += __shfl_xor_sync(0xffffffffu, so0, o); so1 += __shfl_xor_sync(0xffffffffu, so1, o);
      so2 += __shfl_xor_sync(0xffffffffu, so2, o); sd0 += __shfl_xor_sync(0xffffffffu, sd0, o);
      sd1 += __shfl_xor_sync(0xffffffffu, sd1, o); sd2 += __shfl_xor_sync(0xffffffffu, sd2, o);
      sv += __shfl_xor_sync(0xffffffffu, sv, o);
    }
  }
  if (lane != 0) return;
  if (p.g_o) { p.g_o[3 * g] = so0; p.g_o[3 * g + 1] = so1; p.g_o[3 * g + 2] = so2; }
  if (p.g_d) {
    float gdn = p.ray_dn[g];
    if (npass == 2) gdn += p.ray_dn[p.geom.n_rays + g];
    const float* ray = p.ray + 7 * (size_t)g;
    const float dx = ray[3], dy = ray[4], dz = ray[5];
    const float s = gdn / p.dnorm[g];
    p.g_d[3 * g] = fmaf(s, dx, sd0);
    p.g_d[3 * g + 1] = fmaf(s, dy, sd1);
    p.g_d[3 * g + 2] = fmaf(s, dz, sd2) + (p.has_dir_z ? 0.f : sv);
  }
  if (p.g_dir_z) p.g_dir_z[g] = sv;
  if (p.g_bg) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float b = p.ray_bg[3 * g + c];
      if (npass == 2) b += p.ray_bg[3 * ((size_t)p.geom.n_rays + g) + c];
      p.g_bg[3 * g + c] = b;
    }
  }
}
}  // namespace ing

// ================================================================================================
// host-side launchers
// ================================================================================================
int debug_jobs_dw(int index, uint32_t* out) {
  constexpr dw::JobTable t = dw::make_jobs();
  if (index < 0) return dw::kNumJobs;
  if (index >= dw::kNumJobs) return -1;
  const dw::Job& j = t.j[index];
  const int v[9] = {j.a_off, j.a_rows, j.a_half, j.b_off, j.b_rows, j.bias_layer, j.out_off, j.out_ld, j.out_row0};
  for (int i = 0; i < 9; ++i) out[i] = (uint32_t)v[i];
  int g = 0;
  while (g + 1 < dw::kGroups && t.group_begin[g + 1] <= index) ++g;
  out[9] = (uint32_t)g;
  return 10;
}

cudaError_t train_kernels_setup() {
  const cudaError_t e[8] = {
      cudaFuncSetAttribute(chain::chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, chain::Smem<false>::kSmemBytes),
      cudaFuncSetAttribute(chain::chain_x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, chain::Smem<true>::kSmemBytes),
      cudaFuncSetAttribute(dw::dw_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, dw::kSmemBytes),
      cudaFuncSetAttribute(dw::dw_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, dw::kSmemBytes),
      cudaFuncSetAttribute(dw::dw_x3_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, dw::kSmemBytes),
      cudaFuncSetAttribute(dw::dw_x3_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, dw::kSmemBytes),
      cudaFuncSetAttribute(ing::row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ing::kSmemBytes),
      cudaFuncSetAttribute(ing::row_x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ing::kSmemBytes)};
  for (const cudaError_t x : e)
    if (x != cudaSuccess) return x;
  return cudaSuccess;
}

cudaError_t launch_composite_bwd(const CompBwdParams& q, float* scal, cudaStream_t st, long long* launches) {
  const int n = q.geom.passes() * q.geom.n_rays;
  if (q.ray_dn) composite_bwd_kernel<true><<<(n + 7) / 8, 256, 0, st>>>(q);  // one warp per (ray, pass)
  else composite_bwd_kernel<false><<<(n + 7) / 8, 256, 0, st>>>(q);
  ++*launches;
  scale_kernel<<<1, 1, 0, st>>>(q.absmax, scal);
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_chain(const ChainParams& p, int num_sms, cudaStream_t st, long long* launches, bool hilo) {
  const int grid = p.geom.n_units < num_sms ? p.geom.n_units : num_sms;
  if (grid <= 0) return cudaSuccess;
  if (hilo) chain::chain_x3_kernel<<<grid, kThreads, chain::Smem<true>::kSmemBytes, st>>>(p);
  else chain::chain_kernel<<<grid, kThreads, chain::Smem<false>::kSmemBytes, st>>>(p);
  ++*launches;
  return cudaGetLastError();
}

// CTAs per job group for the two networks: `num_sms / kGroups` parts split in proportion to the networks' tile counts
// (64c + 64f: 1 : 2 -> 6 + 12 on 148 SMs, 171 tiles per CTA either way), at least one part per non-empty network, never more
// parts than tiles.  Host logic, exposed to the tests through nfb_debug_schedule(4, ...).
void dw_split(int num_sms, long long tot0, long long tot1, int* parts0, int* parts1) {
  int parts = num_sms / dw::kGroups;
  if (parts < 1) parts = 1;
  if (tot0 > 0 && tot1 > 0 && parts < 2) parts = 2;  // CTAs are independent: more CTAs than SMs only serialises them
  int p0 = tot1 <= 0 ? (tot0 > 0 ? parts : 0) : (tot0 <= 0 ? 0 : (int)((parts * tot0 + (tot0 + tot1) / 2) / (tot0 + tot1)));
  if (tot0 > 0 && p0 < 1) p0 = 1;
  if (tot1 > 0 && p0 > parts - 1) p0 = parts - 1;
  int p1 = tot1 > 0 ? parts - p0 : 0;
  if (p0 > tot0) p0 = (int)tot0;
  if (p1 > tot1) p1 = (int)tot1;
  *parts0 = p0;
  *parts1 = p1;
}
int debug_dw_split(uint32_t* io) {  // in: num_sms, tiles of network 0, tiles of network 1; out: parts0, parts1, groups
  int p0 = 0, p1 = 0;
  dw_split((int)io[0], (long long)io[1], (long long)io[2], &p0, &p1);
  io[0] = (uint32_t)p0; io[1] = (uint32_t)p1; io[2] = (uint32_t)dw::kGroups;
  return 3;
}

// CTAs dw_split gives a launch (PE-only: two job groups, so num_sms / 2 CTAs per group).
static int dw_split_sms(int num_sms, bool pe_only) { return pe_only ? num_sms * dw::kGroups / dw::kPeGroups : num_sms; }

size_t dw_workspace_floats(int num_sms) {  // the most parts dw_split deals out (both networks), times the slot size
  auto most = [](int sms) { const int parts = sms / dw::kGroups; return (size_t)(parts < 2 ? 2 : parts); };
  const size_t full = most(dw_split_sms(num_sms, false)) * kAccBRaw, pe = most(dw_split_sms(num_sms, true)) * dw::kPeSlotFloats;
  return full > pe ? full : pe;
}

cudaError_t launch_dw(DwParams& p, int num_sms, cudaStream_t st, long long* launches, bool pe_only, bool hilo) {
  p.parts[0] = p.parts[1] = 0;
  p.ws_stride = pe_only ? dw::kPeSlotFloats : kAccBRaw;
  const long long tot0 = (long long)p.geom.n_units * p.geom.tiles_c, tot1 = (long long)p.geom.n_units * p.geom.tiles_f;
  if (tot0 + tot1 <= 0) return cudaSuccess;
  dw_split(dw_split_sms(num_sms, pe_only), tot0, tot1, &p.parts[0], &p.parts[1]);
  if (p.parts[0] + p.parts[1] < 1) return cudaSuccess;
  const int blocks = (p.parts[0] + p.parts[1]) * (pe_only ? dw::kPeGroups : dw::kGroups);
  if (hilo) {
    if (pe_only) dw::dw_x3_kernel<true><<<blocks, kThreads, dw::kSmemBytes, st>>>(p);
    else dw::dw_x3_kernel<false><<<blocks, kThreads, dw::kSmemBytes, st>>>(p);
  } else {
    if (pe_only) dw::dw_kernel<true><<<blocks, kThreads, dw::kSmemBytes, st>>>(p);
    else dw::dw_kernel<false><<<blocks, kThreads, dw::kSmemBytes, st>>>(p);
  }
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_grad_reduce(const DwParams* d, bool pe_only, const float* bsum, int n_rays, int npass, float* const acc[2], int num_sms,
                               cudaStream_t st, long long* launches) {
  ReduceParams r = {};
  r.acc[0] = acc[0]; r.acc[1] = acc[1];
  r.bsum = bsum; r.n_rays = n_rays;
  r.pe_only = pe_only ? 1 : 0;
  r.stride = pe_only ? dw::kPeSlotFloats : kAccBRaw;
  if (d) {
    r.ws = d->ws;
    r.stride = d->ws_stride;
    for (int net = 0; net < 2; ++net) {  // the parts dw_kernel gave tiles: the leading ones (j0 = part * per)
      const long long total = (long long)d->geom.n_units * d->geom.tile_count(net);
      const int parts = d->parts[net];
      if (parts > 0 && total > 0) {
        const long long per = (total + parts - 1) / parts;
        r.filled[net] = (int)((total + per - 1) / per);
      }
    }
    r.first1 = d->parts[0];
    r.net0 = r.filled[0] > 0 ? 0 : 1;
    r.nets = (r.filled[0] > 0) + (r.filled[1] > 0);
  }
  const int work = r.nets * (r.stride / 4);  // one thread per float4 of every network that has partials
  int blocks = (work + 255) / 256;
  if (blocks > 8 * num_sms) blocks = 8 * num_sms;
  r.dw_blocks = blocks;
  const int grid = blocks + (n_rays > 0 ? npass : 0);
  if (grid == 0) return cudaSuccess;
  grad_reduce_kernel<<<grid, 256, 0, st>>>(r);
  ++*launches;
  return cudaGetLastError();
}

// Chain rule through the folds for one or both networks + d latent, two launches in all.
cudaError_t launch_finalize_all(const float* const params_c[26], float* const grads_c[26], const float* acc_c,
                                const float* const params_f[26], float* const grads_f[26], const float* acc_f, const float* cond,
                                float* latent_out, cudaStream_t st, long long* launches, float* expr_out) {
  FinAll f;
  f.nets = params_f ? 2 : 1;
  f.latent_out = latent_out;
  f.expr_out = expr_out;
  for (int i = 0; i < 26; ++i) {
    f.net[0].p[i] = params_c[i]; f.net[0].g[i] = grads_c ? grads_c[i] : nullptr;
    f.net[1].p[i] = params_f ? params_f[i] : nullptr; f.net[1].g[i] = (params_f && grads_f) ? grads_f[i] : nullptr;
  }
  f.net[0].acc = acc_c; f.net[1].acc = acc_f;
  f.net[0].cond = f.net[1].cond = cond;
  if (!grads_c) {  // input gradients only: no parameter gradient, only the latent / expression blocks
    if (!latent_out && !expr_out) return cudaSuccess;
    cond_grad_kernel<<<2, 256, 0, st>>>(f);
    ++*launches;
    return cudaGetLastError();
  }
  int blocks = expr_out ? 2 : 1;  // + the latent (and expression) blocks
  for (int t = 0; t < 26; ++t) blocks += (fin_numel(t) + 255) / 256;
  finalize_kernel<<<dim3(blocks, f.nets), 256, 0, st>>>(f);
  ++*launches;
  fin_dir0_kernel<<<dim3((128 * 256 + 256) * 32 / 256, f.nets), 256, 0, st>>>(f);
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_frame_sums(const FrameSumParams& p, cudaStream_t st, long long* launches, bool hilo) {
  if (p.geom.n_rays <= 0) return cudaSuccess;
  if (hilo) raysum_x3_kernel<<<dim3(p.geom.n_rays, p.geom.passes()), kFrameRows, 0, st>>>(p);
  else raysum_kernel<<<dim3(p.geom.n_rays, p.geom.passes()), kFrameRows, 0, st>>>(p);
  ++*launches;
  framesum_kernel<<<dim3(p.n_frames, p.geom.passes()), kFrameRows, 0, st>>>(p);
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_frames_grad(const float* const params_c[26], float* const grads_c[26], const float* const params_f[26],
                               float* const grads_f[26], const float* fsum, const float* fcond, int n_frames, float* latent_out,
                               float* expr_out, cudaStream_t st, long long* launches) {
  FramesGradArgs a = {};
  a.nets = params_f ? 2 : 1;
  const float* const* ps[2] = {params_c, params_f};
  float* const* gs[2] = {grads_c, grads_f};
  for (int n = 0; n < a.nets; ++n) {
    a.p[n][0] = ps[n][0]; a.p[n][1] = ps[n][6];
    if (gs[n]) { a.g[n][0] = gs[n][0]; a.g[n][1] = gs[n][6]; }
  }
  a.fsum = fsum; a.fcond = fcond; a.n_frames = n_frames; a.latent_out = latent_out; a.expr_out = expr_out;
  const int col_blocks = grads_c ? (2 * 256 * kDimCond + 255) / 256 : 0;
  const int bx = n_frames > col_blocks ? n_frames : col_blocks;
  if (bx <= 0) return cudaSuccess;
  frames_grad_kernel<<<dim3(bx, grads_c ? 1 + a.nets : 1), 256, 0, st>>>(a);
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_input_grads(const InGradRowParams& r_in, const InGradRayParams& q_in, int num_sms, cudaStream_t st, long long* launches,
                               bool hilo) {
  InGradRayParams q = q_in;
  if (q.g_o || q.g_d || q.g_dir_z) {
    InGradRowParams r = r_in;
    const long long tot0 = (long long)r.geom.n_units * r.geom.tiles_c, tot1 = (long long)r.geom.n_units * r.geom.tiles_f;
    dw_split(num_sms * dw::kGroups, tot0, tot1, &r.parts[0], &r.parts[1]);  // num_sms CTAs, split by tile counts
    if (hilo) ing::row_x3_kernel<<<r.parts[0] + r.parts[1], ing::kThreadsRow, ing::kSmemBytes, st>>>(r);
    else ing::row_kernel<<<r.parts[0] + r.parts[1], ing::kThreadsRow, ing::kSmemBytes, st>>>(r);
    ++*launches;
    q.rows = r.out;
  } else {
    q.rows = nullptr;
  }
  ing::ray_kernel<<<(q.geom.n_rays + 7) / 8, 256, 0, st>>>(q);  // one warp per ray
  ++*launches;
  return cudaGetLastError();
}

}  // namespace nfb
