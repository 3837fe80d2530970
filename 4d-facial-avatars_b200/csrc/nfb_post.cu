// nfb_post.cu — the steps either side of the render path (SURVEY.md §8f ranks 3, 4), as kernels on the caller's stream:
//
//   * frame products (after the path): the 8-bit images eval_transformed_rays.py writes per frame — cast_to_image (:184-192:
//     clamp, x255, truncate), torch_normal_map (:84-119: back-project the disparity map, cross product of the forward differences,
//     normalise, x0.5+0.5, clean with the last-sample weights: > 0.22 -> 1 and a (1-w) n + w blend, x255, truncate) and
//     cast_to_disparity_image (:195-198: min/max normalise).  The FP32 operation order of the torch expressions is kept (every
//     torch op rounds once; torch.cross contracts a1*b2 - a2*b1 into fma(a1, b2, -(a2*b1)) on both of its back ends; torch's CPU
//     and CUDA back ends differ in two roundings — selectable, see ProductArgs), so the bytes equal the reference function's.
//     Also at the edges (tests/test_frame_products_gpu.py, every pixel): NaN of either sign, +-inf, +-0, subnormal and constant
//     disparities, w_last at the FP32 neighbours of 0.22, rgb outside [0, 1], frames from 2x2 to past one grid-stride sweep.
//     NaN and +-inf become the byte the reference's host-side conversion gives (to_u8).
//   * ray sampler (before the path): see the second half of this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "nfb_internal.h"

namespace nfb {

__device__ __forceinline__ uint32_t float_order_key(float f) {  // monotone float -> uint32 map (for atomic min / max)
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_from_key(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

struct ProductArgs {
  const float* rgb;     // [H, W, 3] or null
  const float* disp;    // [H, W] or null
  const float* w_last;  // [H, W] or null
  int H, W;
  float fx, fy, cx, cy; // cx = intrinsics[2] * rows, cy = intrinsics[3] * cols, rounded to FP32 like the torch scalars
  uint8_t* rgb_u8;      // [H, W, 3] or null
  uint8_t* normals_u8;  // [H - 1, W - 1, 3] or null
  uint32_t* minmax;     // [2] ordered keys of min / max disparity (null: no disparity image requested)
  // Where torch's two back ends round differently (measured on this image, torch 2.11): the CUDA back end divides a tensor by a
  // host scalar as a multiplication by the scalar's reciprocal (".../ fx"), taken in double and rounded to FP32 — not the
  // reciprocal of the FP32 fx, which differs when fx is not an FP32 — and sums the three squared components as (x2 + z2) + y2;
  // the CPU back end divides by the FP32 fx and sums (x2 + y2) + z2.
  int like_cpu;
  float inv_fx, inv_fy;
};

// point of pixel (r, c): (((c - cx) * d) / fx, -(((r - cy) * d) / fy), d)
__device__ __forceinline__ void back_project(const ProductArgs& a, int r, int c, float d, float& x, float& y) {
  const float u = __fmul_rn(__fsub_rn((float)c, a.cx), d), v = __fmul_rn(__fsub_rn((float)r, a.cy), d);
  x = a.like_cpu ? __fdiv_rn(u, a.fx) : __fmul_rn(u, a.inv_fx);
  y = -(a.like_cpu ? __fdiv_rn(v, a.fy) : __fmul_rn(v, a.inv_fy));
}
__device__ __forceinline__ float cross_term(float a1, float b2, float a2, float b1) { return __fmaf_rn(a1, b2, -__fmul_rn(a2, b1)); }
// numpy astype('uint8') / torch .byte() as an x86-64 host computes them: truncate to int32 (cvttss2si: NaN, +-inf and values
// outside the int32 range give 0x80000000), keep the low byte.  A value in [0, 256) truncates.  NaN (0/0: the normal of a
// degenerate patch, any NaN disparity or colour) gives 0, and so does +-inf (a normal whose squared components underflow to a
// zero length while a component does not) — where the device's saturating conversion would give 255 for +inf.
__device__ __forceinline__ uint8_t to_u8(float v) {
  return fabsf(v) < 2147483648.f ? (uint8_t)__float2int_rz(v) : (uint8_t)0;
}

__global__ void __launch_bounds__(256) frame_products_kernel(const ProductArgs a) {
  const int n = a.H * a.W;
  uint32_t kmin = 0xFFFFFFFFu, kmax = 0u;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int r = i / a.W, c = i - r * a.W;
    if (a.rgb_u8) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float v = fminf(fmaxf(a.rgb[3 * i + k], 0.f), 1.f);
        a.rgb_u8[3 * i + k] = to_u8(__fmul_rn(v, 255.f));
      }
    }
    if (a.minmax) {
      const uint32_t k = float_order_key(a.disp[i]);
      kmin = min(kmin, k);
      kmax = max(kmax, k);
    }
    if (a.normals_u8 && r < a.H - 1 && c < a.W - 1) {
      const float d00 = a.disp[i], d01 = a.disp[i + 1], d10 = a.disp[i + a.W];
      float x00, y00, x01, y01, x10, y10;
      back_project(a, r, c, d00, x00, y00);
      back_project(a, r, c + 1, d01, x01, y01);
      back_project(a, r + 1, c, d10, x10, y10);
      // dy = column difference, dx = row difference; normals = cross(dy, dx)
      const float a0 = __fsub_rn(x01, x00), a1 = __fsub_rn(y01, y00), a2 = __fsub_rn(d01, d00);
      const float b0 = __fsub_rn(x10, x00), b1 = __fsub_rn(y10, y00), b2 = __fsub_rn(d10, d00);
      float nrm[3] = {cross_term(a1, b2, a2, b1), cross_term(a2, b0, a0, b2), cross_term(a0, b1, a1, b0)};
      const float q0 = __fmul_rn(nrm[0], nrm[0]), q1 = __fmul_rn(nrm[1], nrm[1]), q2 = __fmul_rn(nrm[2], nrm[2]);
      const float len = __fsqrt_rn(a.like_cpu ? __fadd_rn(__fadd_rn(q0, q1), q2) : __fadd_rn(__fadd_rn(q0, q2), q1));
      const float m = a.w_last ? a.w_last[i] : 0.f;
      uint8_t* out = a.normals_u8 + 3 * ((size_t)r * (a.W - 1) + c);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        float v = __fadd_rn(__fmul_rn(__fdiv_rn(nrm[k], len), 0.5f), 0.5f);
        if (a.w_last) {
          if (m > 0.22f) v = 1.0f;
          v = __fadd_rn(__fmul_rn(__fsub_rn(1.f, m), v), m);
        }
        out[k] = to_u8(__fmul_rn(v, 255.f));
      }
    }
  }
  if (a.minmax) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
      kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
    }
    if ((threadIdx.x & 31) == 0) {
      atomicMin(a.minmax, kmin);
      atomicMax(a.minmax + 1, kmax);
    }
  }
}

// cast_to_disparity_image: ((d - min) / (max - min)).clamp(0, 1) * 255, truncated
__global__ void __launch_bounds__(256) disparity_image_kernel(const float* __restrict__ disp, int n, const uint32_t* __restrict__ minmax,
                                                              uint8_t* __restrict__ out) {
  const float lo = float_from_key(minmax[0]), hi = float_from_key(minmax[1]);
  const float range = __fsub_rn(hi, lo);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float v = __fdiv_rn(__fsub_rn(disp[i], lo), range);
    v = fminf(fmaxf(v, 0.f), 1.f);
    out[i] = to_u8(__fmul_rn(v, 255.f));
  }
}

cudaError_t launch_frame_products(const float* rgb, const float* disp, const float* w_last, const double intr[4], int H, int W,
                                  uint8_t* rgb_u8, uint8_t* normals_u8, uint8_t* disp_u8, uint32_t* minmax_scratch, int like_torch_cpu,
                                  cudaStream_t st, long long* launches) {
  ProductArgs a;
  a.like_cpu = like_torch_cpu;
  a.inv_fx = (float)(1.0 / intr[0]);
  a.inv_fy = (float)(1.0 / intr[1]);
  a.rgb = rgb; a.disp = disp; a.w_last = w_last; a.H = H; a.W = W;
  a.fx = (float)intr[0]; a.fy = (float)intr[1];
  a.cx = (float)(intr[2] * (double)H);  // the reference multiplies by depthmap.shape[0] for x and shape[1] for y (square frames)
  a.cy = (float)(intr[3] * (double)W);
  a.rgb_u8 = rgb_u8; a.normals_u8 = normals_u8;
  a.minmax = disp_u8 ? minmax_scratch : nullptr;
  if (disp_u8) {
    const uint32_t init[2] = {0xFFFFFFFFu, 0u};
    cudaError_t e = cudaMemcpyAsync(minmax_scratch, init, sizeof(init), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
  }
  const int n = H * W;
  int blocks = (n + 255) / 256;
  if (blocks > 148 * 8) blocks = 148 * 8;
  frame_products_kernel<<<blocks, 256, 0, st>>>(a);
  ++*launches;
  if (disp_u8) {
    disparity_image_kernel<<<blocks, 256, 0, st>>>(disp, n, minmax_scratch, disp_u8);
    ++*launches;
  }
  return cudaGetLastError();
}

}  // namespace nfb

// ================================================================================================
// Ray sampler (before the path): np.random.choice(H * W, size, replace=False, p=importance map) of
// train_transformed_rays.py:319-321 with bit-identical indices given the same uniform draws, then the gathers of :323-331
// (ray origin / direction, target colour, background colour) including the reference's index quirk: flat index k addresses the
// PROBABILITY map row-major (k = row * W + col) but the PIXEL (row = k % H, col = k / H) — coords is built from a transposed
// meshgrid (:303-316) — so the box of probable pixels is the transposed bounding box.
// One thread block does the whole selection of one image: the cdf is never materialised (nfb_sampler.h evaluates any entry
// exactly).  sample_rays_kernel selects for one image; sample_images_kernel for K images of a training step, one block each.
// ================================================================================================
#include "nfb_sampler.h"

namespace nfb {

constexpr int kSmpThreads = 1024;

// One image's selection, run by one thread block of kSmpThreads threads.
struct SelectArgs {
  smp::Map map;
  const double* draws;   // consumed like RandomState.rand: round r takes (size - n_found) values
  int size, max_rounds;
  long long* found;      // [size] selected flat indices in selection order
  smp::Run* runs;
  smp::Seg* segs;
  int* first_pos;        // [H * W] scratch, all INT_MAX before and after
};
struct SelectState { int n_found, rounds, consumed; };

// numpy's choice loop (nfb_sampler.h) from `resume` ({n_found, rounds, consumed}; null: from the start) until `size` indices are
// found or max_rounds rounds ran.  Every thread of the block returns the same state.
__device__ __forceinline__ SelectState select_pixels(const SelectArgs& a, const int* resume) {
  __shared__ long long sorted[kSmpMax];
  __shared__ long long cand[kSmpMax];
  __shared__ int warp_sums[kSmpThreads / 32];
  __shared__ double total_s;
  __shared__ int n_runs_s, n_segs_s, n_found_s, consumed_s;
  const int tid = threadIdx.x;
  const long long N = (long long)a.map.H * a.map.W;
  if (tid == 0) { n_found_s = resume ? resume[0] : 0; consumed_s = resume ? resume[2] : 0; }
  __syncthreads();
  int rounds = 0;
  while (rounds < a.max_rounds && n_found_s < a.size) {
    const int n_found = n_found_s, m = a.size - n_found, consumed = consumed_s;
    // ---- ascending copy of the indices found so far (their probability is zero from now on): bitonic sort, padded
    for (int i = tid; i < kSmpMax; i += kSmpThreads) sorted[i] = i < n_found ? a.found[i] : 0x7FFFFFFFFFFFFFFFLL;
    __syncthreads();
    for (int kk = 2; kk <= kSmpMax; kk <<= 1)
      for (int jj = kk >> 1; jj > 0; jj >>= 1) {
        const int i = 2 * tid - (tid & (jj - 1)), l = i + jj;
        const bool up = (i & kk) == 0;
        const long long x = sorted[i], y = sorted[l];
        if ((x > y) == up) { sorted[i] = y; sorted[l] = x; }
        __syncthreads();
      }
    // ---- tables of the sequential cumsum with those entries zeroed (serial in the running sum: one thread)
    if (tid == 0) {
      int nr, ns;
      total_s = smp::build_tables(a.map, sorted, n_found, a.runs, nr, a.segs, ns);
      n_runs_s = nr;
      n_segs_s = ns;
      __threadfence_block();
    }
    __syncthreads();
    // more segments than the table holds: the selection ends short here, before any search reads an unwritten segment.  No map
    // of at most kMaxRuns runs gets here (nfb_sampler.h bounds its segments); this keeps the reads inside the tables regardless.
    if (n_segs_s > smp::kMaxSegs) break;
    const double total = total_s;
    const int n_runs = n_runs_s;
    // ---- searchsorted(cdf / cdf[-1], x, side='right') for this round's draws; first occurrence of every value wins
    for (int j = tid; j < kSmpMax; j += kSmpThreads) {
      long long c = -1;
      if (j < m) {
        c = smp::search_right(a.draws[consumed + j], total, N, a.runs, n_runs, a.segs, sorted, n_found);
        if (c >= N) c = N - 1;  // x < 1 = cdf[-1]: cannot happen; keeps the scratch index in range
        atomicMin(a.first_pos + c, j);
      }
      cand[j] = c;
    }
    __syncthreads();
    // ---- keep flags, exclusive scan in draw order, append
    int keep[2], local = 0;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int j = 2 * tid + e;
      keep[e] = (j < m && a.first_pos[cand[j]] == j) ? 1 : 0;
      local += keep[e];
    }
    int incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if ((tid & 31) >= o) incl += t;
    }
    if ((tid & 31) == 31) warp_sums[tid >> 5] = incl;
    __syncthreads();
    if (tid < 32) {
      int w = warp_sums[tid];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, o);
        if (tid >= o) w += t;
      }
      warp_sums[tid] = w;
    }
    __syncthreads();
    int pos = n_found + incl - local + ((tid >> 5) ? warp_sums[(tid >> 5) - 1] : 0);
    const int added = warp_sums[kSmpThreads / 32 - 1];
#pragma unroll
    for (int e = 0; e < 2; ++e)
      if (keep[e]) a.found[pos++] = cand[2 * tid + e];
    __syncthreads();
    for (int j = tid; j < m; j += kSmpThreads) a.first_pos[cand[j]] = 0x7FFFFFFF;  // leave the scratch clean
    if (tid == 0) { n_found_s = n_found + added; consumed_s = consumed + m; }
    ++rounds;
    __syncthreads();
  }
  const SelectState r = {n_found_s, rounds, consumed_s};
  __syncthreads();  // every thread has read the state before a later call may reset it
  return r;
}

// Where the gathers of one image go (any output may be null).
struct GatherArgs {
  const float* pose;        // [12] camera-to-world 3x4
  float fx, fy, wcx, hcy;
  int H, W;
  const float* image;       // [H, W, 3]
  const float* background;  // [H, W, 3]
  float *ray_o, *ray_d, *target, *bg_out;  // [count, 3] each
  int* pixel_rc;            // [count, 2]
  long long* indices;       // [count]
  int* frame;               // [count] <- frame_value
  int frame_value;
};

// Gathers (train_transformed_rays.py:323-331) into output slots [0, count): slot i takes found[i] while i < n_found and
// found[i % n_found] after (an incomplete selection repeats its first pixels).
__device__ __forceinline__ void gather_pixels(const GatherArgs& a, const long long* found, int n_found, int count) {
  const int H = a.H, W = a.W;
  for (int i = threadIdx.x; i < count; i += kSmpThreads) {
    const long long k = found[i < n_found ? i : i % n_found];
    const int row = (int)(k % H), col = (int)(k / H);  // coords[k]: the transposed-meshgrid quirk
    if (a.pixel_rc) { a.pixel_rc[2 * i] = row; a.pixel_rc[2 * i + 1] = col; }
    if (a.indices) a.indices[i] = k;
    if (a.frame) a.frame[i] = a.frame_value;
    if (a.ray_d) {  // get_ray_bundle (nerf_helpers.py:111-122) at pixel (row, col), same FP32 operation order as the render kernels
      float cx, cy;
      smp::camera_dir(row, col, a.fx, a.fy, a.wcx, a.hcy, cx, cy);
      for (int q = 0; q < 3; ++q)
        a.ray_d[3 * i + q] = __fadd_rn(__fadd_rn(__fmul_rn(cx, a.pose[4 * q]), __fmul_rn(cy, a.pose[4 * q + 1])), __fmul_rn(-1.f, a.pose[4 * q + 2]));
      if (a.ray_o) for (int q = 0; q < 3; ++q) a.ray_o[3 * i + q] = a.pose[4 * q + 3];
    }
    const size_t px = smp::pixel_index(row, col, W) * 3;
    if (a.target) for (int q = 0; q < 3; ++q) a.target[3 * i + q] = a.image[px + q];
    if (a.bg_out) for (int q = 0; q < 3; ++q) a.bg_out[3 * i + q] = a.background[px + q];
  }
}

__global__ void __launch_bounds__(kSmpThreads, 1) sample_rays_kernel(const SampleArgs a) {
  const SelectArgs s = {a.map, a.draws, a.size, a.max_rounds, a.found, a.runs, a.segs, a.first_pos};
  const SelectState r = select_pixels(s, a.state);
  if (threadIdx.x == 0) { a.state[0] = r.n_found; a.state[1] += r.rounds; a.state[2] = r.consumed; }
  GatherArgs g = {};
  g.pose = a.pose; g.fx = a.fx; g.fy = a.fy; g.wcx = a.wcx; g.hcy = a.hcy; g.H = a.map.H; g.W = a.map.W;
  g.image = a.image; g.background = a.background;
  g.ray_o = a.ray_o; g.ray_d = a.ray_d; g.target = a.target; g.bg_out = a.bg_out; g.pixel_rc = a.pixel_rc;
  gather_pixels(g, a.found, r.n_found, r.n_found);
}

// Several images in one launch, block k = image image_index[k] (see ImageSampleArgs).  Everything per step comes from device
// memory, so a captured launch samples whatever images the index table names at replay.
__global__ void __launch_bounds__(kSmpThreads, 1) sample_images_kernel(const ImageSampleArgs a) {
  const int k = blockIdx.x, tid = threadIdx.x, n = a.size;
  const int img = a.image_index[k];
  const size_t slot = (size_t)k * n;
  bool ok = img >= 0 && img < a.n_images;
  smp::Map m = {};
  if (ok) {
    const RayMapRec r = a.maps[img];
    m.H = r.H; m.W = r.W; m.b0 = r.bbox[0]; m.b1 = r.bbox[1]; m.b2 = r.bbox[2]; m.b3 = r.bbox[3]; m.q_out = r.q_out; m.q_in = r.q_in;
    // a map the selection cannot follow reads nothing: the batch's shape, a box inside the frame, positive weights, room for its runs
    ok = m.H == a.H && m.W == a.W && m.b0 >= 0 && m.b1 <= m.H && m.b2 >= 0 && m.b3 <= m.W && m.q_out > 0.0 && m.q_in > 0.0 &&
         smp::num_runs(m) <= smp::kMaxRuns;
  }
  if (!ok) {  // out-of-range index: NaN rays and rows, frame slot K (out of range for nfb_set_frames of K frames: renders NaN)
    const float nan = __int_as_float(0x7FC00000);
    for (int i = tid; i < n; i += kSmpThreads) {
      for (int q = 0; q < 3; ++q) {
        if (a.ray_o) a.ray_o[3 * (slot + i) + q] = nan;
        if (a.ray_d) a.ray_d[3 * (slot + i) + q] = nan;
        if (a.target) a.target[3 * (slot + i) + q] = nan;
        if (a.bg_out) a.bg_out[3 * (slot + i) + q] = nan;
      }
      if (a.pixel_rc) { a.pixel_rc[2 * (slot + i)] = -1; a.pixel_rc[2 * (slot + i) + 1] = -1; }
      if (a.indices) a.indices[slot + i] = -1;
      if (a.frame) a.frame[slot + i] = a.K;
    }
    if (a.expr_out) for (int i = tid; i < kDimExpr; i += kSmpThreads) a.expr_out[(size_t)k * kDimExpr + i] = nan;
    if (a.latent_out) for (int i = tid; i < kDimLatent; i += kSmpThreads) a.latent_out[(size_t)k * kDimLatent + i] = nan;
    if (tid == 0 && a.state) { a.state[3 * k] = 0; a.state[3 * k + 1] = 0; a.state[3 * k + 2] = 0; }
    return;
  }
  const size_t hw = (size_t)a.H * a.W;
  const SelectArgs s = {m, a.draws + (size_t)k * a.max_rounds * n, n, a.max_rounds, a.found + slot, a.runs + (size_t)k * smp::kMaxRuns,
                        a.segs + (size_t)k * smp::kMaxSegs, a.first_pos + k * hw};
  const SelectState r = select_pixels(s, nullptr);
  if (tid == 0) {
    if (a.state) { a.state[3 * k] = r.n_found; a.state[3 * k + 1] = r.rounds; a.state[3 * k + 2] = r.consumed; }
    if (a.shortfall) a.shortfall[k] += n - r.n_found;  // slot k is this block's alone: no atomic
  }
  GatherArgs g = {};
  g.pose = a.poses + 12 * (size_t)img; g.fx = a.fx; g.fy = a.fy; g.wcx = a.wcx; g.hcy = a.hcy; g.H = a.H; g.W = a.W;
  g.image = a.images + 3 * hw * img; g.background = a.background;
  auto at3 = [&](float* p) { return p ? p + 3 * slot : nullptr; };
  g.ray_o = at3(a.ray_o); g.ray_d = at3(a.ray_d); g.target = at3(a.target); g.bg_out = at3(a.bg_out);
  g.pixel_rc = a.pixel_rc ? a.pixel_rc + 2 * slot : nullptr;
  g.indices = a.indices ? a.indices + slot : nullptr;
  g.frame = a.frame ? a.frame + slot : nullptr;
  g.frame_value = k;
  gather_pixels(g, a.found + slot, r.n_found, r.n_found > 0 ? n : 0);  // nothing selected: nothing to repeat
  // the conditioning rows nfb_set_frames reads: frame k = (expressions[img], latent_table[img])
  if (a.expr_out) for (int i = tid; i < kDimExpr; i += kSmpThreads) a.expr_out[(size_t)k * kDimExpr + i] = a.expr_table[(size_t)img * kDimExpr + i];
  if (a.latent_out)
    for (int i = tid; i < kDimLatent; i += kSmpThreads) a.latent_out[(size_t)k * kDimLatent + i] = a.latent_table[(size_t)img * kDimLatent + i];
}

__global__ void fill_int_kernel(int* p, long long n, int v) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

cudaError_t launch_fill_int(int* p, long long n, int v, cudaStream_t st, long long* launches) {
  fill_int_kernel<<<296, 256, 0, st>>>(p, n, v);
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_sample_rays(const SampleArgs& a, cudaStream_t st, long long* launches) {
  sample_rays_kernel<<<1, kSmpThreads, 0, st>>>(a);
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_sample_images(const ImageSampleArgs& a, cudaStream_t st, long long* launches) {
  sample_images_kernel<<<a.K, kSmpThreads, 0, st>>>(a);
  ++*launches;
  return cudaGetLastError();
}

}  // namespace nfb
