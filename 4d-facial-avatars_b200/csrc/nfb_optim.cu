// nfb_optim.cu — the training step's tail as two launches (SURVEY.md §8f rank 2): the loss of
// train_transformed_rays.py:355-389 (mse(rgb_coarse) + mse(rgb_fine); the latent-code regulariser joins in the optimizer
// kernel) as a gradient w.r.t. the rendered colours, and torch.optim.Adam (:391, YAML optimizer block) over ONE flat FP32
// bucket holding both networks and the latent-code table, with optimizer.zero_grad() fused in.  The FP32 -> kernel-layout
// re-pack that follows is fold_feat_kernel + repack_kernel (nfb_pack.cu), two more launches.
#include <cuda_runtime.h>

#include <cstddef>

#include "../../include/nfb.h"
#include "nfb_internal.h"
#include "nfb_layout.h"

namespace nfb {

// d/d rgb of  mean((rgb - target)^2)  taken over n_total * 3 elements (n_total = the GLOBAL batch when the rays of this call
// are one shard of it: a SUM all-reduce of the parameter gradients then yields the single-process gradient).
// loss[0] += sum((rgb_c - t)^2) / (3 n_total), loss[1] likewise for the fine pass (each call adds its shard's share).
// ONE block: the partial sums meet in a fixed order (thread-strided, warp butterfly, warps in order) with no atomics, so the loss
// repeats bit for bit.  A training batch is a few thousand rays: a handful of elements per thread.
constexpr int kLossThreads = 1024;
__global__ void __launch_bounds__(kLossThreads) loss_grad_kernel(const float* __restrict__ rgb_c, const float* __restrict__ rgb_f,
                                                                 const float* __restrict__ target, int n_elems, float inv_count,
                                                                 float* __restrict__ g_c, float* __restrict__ g_f, float* __restrict__ loss) {
  __shared__ float part[2][kLossThreads / 32];
  float sc = 0.f, sf = 0.f;
  for (int i = threadIdx.x; i < n_elems; i += kLossThreads) {
    const float t = target[i];
    const float dc = rgb_c[i] - t;
    g_c[i] = 2.f * dc * inv_count;
    sc = fmaf(dc, dc, sc);
    if (rgb_f) {
      const float df = rgb_f[i] - t;
      g_f[i] = 2.f * df * inv_count;
      sf = fmaf(df, df, sf);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sc += __shfl_xor_sync(0xffffffffu, sc, o);
    sf += __shfl_xor_sync(0xffffffffu, sf, o);
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { part[0][w] = sc; part[1][w] = sf; }
  __syncthreads();
  if (threadIdx.x < 2) {
    float s = 0.f;
    for (int k = 0; k < kLossThreads / 32; ++k) s += part[threadIdx.x][k];
    loss[threadIdx.x] += s * inv_count;
  }
}

// torch.optim.Adam (no weight decay, no amsgrad), element-wise over the flat bucket, same operation order as torch's
// single-tensor implementation:  m.lerp_(g, 1 - b1);  v.mul_(b2).addcmul_(g, g, 1 - b2);
// denom = sqrt(v) / sqrt(1 - b2^t) + eps;  p -= (lr / (1 - b1^t)) * m / denom.   Gradients are zeroed after use.
// Latent-code regulariser (train_transformed_rays.py:369-372,386: 10 * 0.0005 * ||latent||_2 on the frame's row of the
// table): its gradient reg_w * l / ||l|| (0 at l == 0, as torch.norm's backward gives) is added to that row's gradient here,
// after any all-reduce, so every rank adds it exactly once.
// The element-wise update both Adam kernels run over [0, n), grid-strided, from this step's scalars: one body, so the host-scalar
// and the device-state entries cannot drift apart.
__device__ __forceinline__ void adam_update(float* __restrict__ P, float* __restrict__ G, float* __restrict__ M, float* __restrict__ V,
                                            long long n, float lr_over_bc1, float sqrt_bc2, float b1, float b2, float eps, float gs,
                                            long long reg_off, float reg_w) {
  __shared__ float reg_inv_norm;
  if (reg_off >= 0) {  // every block that touches the row needs 1 / ||l||: 32 values, recomputed per block (cheap, uniform)
    if (threadIdx.x < 32) {
      const float l = P[reg_off + threadIdx.x];
      float s = l * l;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (threadIdx.x == 0) reg_inv_norm = s > 0.f ? rsqrtf(s) : 0.f;
    }
    __syncthreads();
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float g = G[i] * gs;
    const float p = P[i];
    if (reg_off >= 0 && i >= reg_off && i < reg_off + kDimLatent) g = fmaf(reg_w * reg_inv_norm, p, g);
    float m = M[i], v = V[i];
    m = fmaf(g - m, 1.f - b1, m);
    v = fmaf(g * g, 1.f - b2, v * b2);
    const float denom = sqrtf(v) / sqrt_bc2 + eps;
    P[i] = p - lr_over_bc1 * (m / denom);
    M[i] = m;
    V[i] = v;
    G[i] = 0.f;
  }
}

struct AdamArgs {
  float* p; float* g; float* m; float* v;
  long long n;
  float lr_over_bc1, sqrt_bc2, b1, b2, eps, grad_scale;
  long long reg_off;   // float offset of the regularised 32-vector inside the bucket; < 0: none
  float reg_w;
};
__global__ void __launch_bounds__(256) adam_kernel(const AdamArgs a) {
  adam_update(a.p, a.g, a.m, a.v, a.n, a.lr_over_bc1, a.sqrt_bc2, a.b1, a.b2, a.eps, a.grad_scale, a.reg_off, a.reg_w);
}

// Graph-capturable variant: the step counter, the learning-rate schedule and the regularised row live in DEVICE memory, so one
// captured CUDA graph replays every iteration, and eager steps can share the same state.  adam_prepare_kernel (1 thread) advances
// the step and derives this step's scalars: the reference's schedule in float64 on the caller's double constants, the bias
// corrections from the FP32 betas the moments are formed with; adam_dev_kernel runs adam_update on them.
struct AdamDevState {  // mirrors NfbAdamDev (include/nfb.h)
  int step, pad;
  double lr0, decay_factor, decay_steps;
  float b1, b2, eps, grad_scale, reg_w;
  long long table_off;       // float offset of the latent table in the bucket (< 0: no regulariser)
  const long long* row;      // device pointer to the current row index (null or < 0: no regulariser)
  float lr_over_bc1, sqrt_bc2;
  long long reg_off;
};
static_assert(sizeof(AdamDevState) == sizeof(NfbAdamDev) && offsetof(AdamDevState, lr0) == offsetof(NfbAdamDev, lr0) &&
                  offsetof(AdamDevState, b1) == offsetof(NfbAdamDev, beta1) && offsetof(AdamDevState, table_off) == offsetof(NfbAdamDev, table_offset) &&
                  offsetof(AdamDevState, lr_over_bc1) == offsetof(NfbAdamDev, lr_over_bc1) && offsetof(AdamDevState, reg_off) == offsetof(NfbAdamDev, reg_offset),
              "NfbAdamDev mirror");
__global__ void adam_prepare_kernel(AdamDevState* st) {
  const int step = ++st->step;  // 1-based number of the step being taken
  const int i = step - 1;       // the reference's loop index (train_transformed_rays.py:393-399: lr set AFTER step i)
  const double lr = (i <= 0) ? st->lr0 : st->lr0 * pow(st->decay_factor, (double)(i - 1) / st->decay_steps);
  const double bc1 = 1.0 - pow((double)st->b1, (double)step), bc2 = 1.0 - pow((double)st->b2, (double)step);
  st->lr_over_bc1 = (float)(lr / bc1);
  st->sqrt_bc2 = (float)sqrt(bc2);
  const long long row = st->row ? st->row[0] : -1;
  st->reg_off = (st->table_off >= 0 && row >= 0) ? st->table_off + (long long)kDimLatent * row : -1;
}
__global__ void __launch_bounds__(256) adam_dev_kernel(float* __restrict__ P, float* __restrict__ G, float* __restrict__ M, float* __restrict__ V,
                                                       long long n, const AdamDevState* __restrict__ st) {
  adam_update(P, G, M, V, n, st->lr_over_bc1, st->sqrt_bc2, st->b1, st->b2, st->eps, st->grad_scale, st->reg_off, st->reg_w);
}
cudaError_t launch_adam_dev(float* p, float* g, float* m, float* v, long long n, void* dev_state, cudaStream_t st, long long* launches) {
  AdamDevState* s = static_cast<AdamDevState*>(dev_state);
  adam_prepare_kernel<<<1, 1, 0, st>>>(s);
  ++*launches;
  long long blocks = (n + 255) / 256;
  if (blocks > 148 * 8) blocks = 148 * 8;
  adam_dev_kernel<<<(int)blocks, 256, 0, st>>>(p, g, m, v, n, s);
  ++*launches;
  return cudaGetLastError();
}

// The latent-table rows of the bucket gradient for one step over K images (nfb_latent_rows_grad).  ONE warp, lane c = column c of
// every row, so each element's sum runs in one fixed order with integer indexing and no atomics:
//   for k = 0..K-1:  G[img[k]][c] += grad_latents[k][c]                                   (the per-frame d latent)
//   for k = 0..K-1:  G[img[k]][c] += (reg_w * (1 / sqrt(s))) * T[img[k]][c],  s = sum_c T[img[k]][c]^2
// each a separately rounded FP32 multiply and add; s is the lanes' squares summed by the xor butterfly (offsets 16, 8, 4, 2, 1);
// the term is skipped at s == 0 (torch.norm's subgradient at 0) and for reg_w == 0.  A row named twice gets both frames'
// terms in that order; an index outside [0, n_rows) adds nothing and reads nothing.
__global__ void __launch_bounds__(32) latent_rows_kernel(const float* __restrict__ glat, const int* __restrict__ img, int K,
                                                         const float* __restrict__ table, int n_rows, float* __restrict__ tgrad, float reg_w) {
  const int c = threadIdx.x;
  for (int k = 0; k < K; ++k) {
    const int r = img[k];
    if (r < 0 || r >= n_rows) continue;
    float* g = tgrad + (size_t)r * kDimLatent + c;
    *g = __fadd_rn(*g, glat[(size_t)k * kDimLatent + c]);
  }
  if (reg_w == 0.f) return;
  for (int k = 0; k < K; ++k) {
    const int r = img[k];
    if (r < 0 || r >= n_rows) continue;
    const float l = table[(size_t)r * kDimLatent + c];
    float s = __fmul_rn(l, l);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    if (s == 0.f) continue;  // uniform: every lane holds the same s
    float* g = tgrad + (size_t)r * kDimLatent + c;
    *g = __fadd_rn(*g, __fmul_rn(__fmul_rn(reg_w, __fdiv_rn(1.f, __fsqrt_rn(s))), l));
  }
}

cudaError_t launch_latent_rows(const float* grad_latents, const int* image_index, int K, const float* table, int n_rows, float* table_grads,
                               float reg_w, cudaStream_t st, long long* launches) {
  latent_rows_kernel<<<1, kDimLatent, 0, st>>>(grad_latents, image_index, K, table, n_rows, table_grads, reg_w);
  ++*launches;
  return cudaGetLastError();
}

// The pose and expression rows of a fitting step over K images (nfb_fit_rows_grad; order: include/nfb.h).  Ray j of slot k sits
// at pixel (row, col) = pixel_rc[k * n + j] with camera direction c = (cx, cy, -1) (smp::camera_dir, the sampler's own bits),
// d = R c and o = t, so the 3x4 pose row gets dR[q] = sum_j dd_j[q] * (cx_j, cy_j, -1) and dt[q] = sum_j do_j[q].
// fit_pose_slots_kernel: block k sums slot k's rays into slots[k][12] (entry 4q + m of the row-major 3x4).  Thread t adds the
// terms of rays j = t, t + 256, ... in ascending j, each term one rounded FP32 product (dd * cx, dd * cy), a negation (-dd) or the
// value itself (do), added with one rounded FP32 add; the 256 partials then meet in a halving tree, partial[t] += partial[t + s]
// for s = 128, 64, ..., 1.  A NULL dd (do) gives zero for columns 0..2 (3).
constexpr int kFitThreads = 256;
__global__ void __launch_bounds__(kFitThreads) fit_pose_slots_kernel(const int* __restrict__ pixel_rc, const float* __restrict__ g_o,
                                                                     const float* __restrict__ g_d, int n, float fx, float fy, float wcx,
                                                                     float hcy, float* __restrict__ slots) {
  __shared__ float part[12][kFitThreads];
  const int k = blockIdx.x, t = threadIdx.x;
  float acc[12];
#pragma unroll
  for (int c = 0; c < 12; ++c) acc[c] = 0.f;
  for (int j = t; j < n; j += kFitThreads) {
    const size_t i = (size_t)k * n + j;
    if (g_d) {
      float cx, cy;
      smp::camera_dir(pixel_rc[2 * i], pixel_rc[2 * i + 1], fx, fy, wcx, hcy, cx, cy);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const float dd = g_d[3 * i + q];
        acc[4 * q] = __fadd_rn(acc[4 * q], __fmul_rn(dd, cx));
        acc[4 * q + 1] = __fadd_rn(acc[4 * q + 1], __fmul_rn(dd, cy));
        acc[4 * q + 2] = __fadd_rn(acc[4 * q + 2], -dd);
      }
    }
    if (g_o) {
#pragma unroll
      for (int q = 0; q < 3; ++q) acc[4 * q + 3] = __fadd_rn(acc[4 * q + 3], g_o[3 * i + q]);
    }
  }
#pragma unroll
  for (int c = 0; c < 12; ++c) part[c][t] = acc[c];
  __syncthreads();
  for (int s = kFitThreads / 2; s > 0; s >>= 1) {
    if (t < s) {
#pragma unroll
      for (int c = 0; c < 12; ++c) part[c][t] = __fadd_rn(part[c][t], part[c][t + s]);
    }
    __syncthreads();
  }
  if (t < 12) slots[(size_t)k * 12 + t] = part[t][0];
}

// fit_rows_kernel: one block, thread c = one column of the 12 pose columns (c < 12: slots) and the 76 expression columns
// (12 <= c < 88: grad_expressions), in ascending k:  G[img[k]][c] += term[k][c], one FP32 add each; no atomics.  An index outside
// [0, n_rows) adds nothing.  A NULL source or destination leaves its columns alone.
__global__ void __launch_bounds__(96) fit_rows_kernel(const int* __restrict__ img, int K, int n_rows, const float* __restrict__ slots,
                                                      float* __restrict__ pose_grads, const float* __restrict__ g_expr,
                                                      float* __restrict__ expr_grads) {
  const int c = threadIdx.x;
  const bool pose = c < 12 && pose_grads, expr = c >= 12 && c < 12 + kDimExpr && expr_grads;
  if (!pose && !expr) return;
  for (int k = 0; k < K; ++k) {
    const int r = img[k];
    if (r < 0 || r >= n_rows) continue;
    if (pose) {
      float* g = pose_grads + (size_t)r * 12 + c;
      *g = __fadd_rn(*g, slots[(size_t)k * 12 + c]);
    } else {
      float* g = expr_grads + (size_t)r * kDimExpr + (c - 12);
      *g = __fadd_rn(*g, g_expr[(size_t)k * kDimExpr + (c - 12)]);
    }
  }
}

cudaError_t launch_fit_rows(const int* image_index, int K, int n, int n_rows, const int* pixel_rc, const float* g_o, const float* g_d,
                            float fx, float fy, float wcx, float hcy, float* slots, float* pose_grads, const float* g_expr,
                            float* expr_grads, cudaStream_t st, long long* launches) {
  if (pose_grads) {
    fit_pose_slots_kernel<<<K, kFitThreads, 0, st>>>(pixel_rc, g_o, g_d, n, fx, fy, wcx, hcy, slots);
    ++*launches;
  }
  fit_rows_kernel<<<1, 96, 0, st>>>(image_index, K, n_rows, slots, pose_grads, g_expr, expr_grads);
  ++*launches;
  return cudaGetLastError();
}

// The learned background's rows of the bucket gradient (nfb_background_rows_grad; order: include/nfb.h).  The pixels are split
// between warps instead of the rays: warp w of the grid owns the table rows whose index is w modulo the number of warps, and walks
// ALL rays in ascending order, 32 at a time.  In each group of 32, __match_any_sync gathers the lanes whose ray falls on the same
// owned pixel, and the lowest of them adds the group's rays in ascending lane order; __syncwarp orders one group's row writes
// before the next group's reads.  So every pixel receives its rays in ascending order from one warp, whatever the batch holds
// (repeats inside a slot, pixels shared across slots, a rank's slice cutting either), with no atomics and no sort; how many warps
// run changes which warp owns a pixel, never the order of its adds.  Every warp reads every ray's pixel (8 B a ray, from L1/L2).
constexpr int kBgWarps = 8, kBgBlocks = 128;
__global__ void __launch_bounds__(kBgWarps * 32) background_rows_kernel(const int* __restrict__ pixel_rc, int n_rays, int H, int W,
                                                                         const float* __restrict__ g_render, const float* __restrict__ g_loss,
                                                                         float* __restrict__ table) {
  const int lane = threadIdx.x & 31;
  const int part = blockIdx.x * kBgWarps + (threadIdx.x >> 5), parts = gridDim.x * kBgWarps;
  for (int base = 0; base < n_rays; base += 32) {
    const int r = base + lane;
    int key = -1;
    if (r < n_rays) {
      const int row = pixel_rc[2 * (size_t)r], col = pixel_rc[2 * (size_t)r + 1];
      if (row >= 0 && row < H && col >= 0 && col < W) key = (int)smp::pixel_index(row, col, W);
    }
    const bool mine = key >= 0 && key % parts == part;
    const unsigned group = __match_any_sync(0xffffffffu, mine ? key : -2 - lane);  // lanes not owning their pixel match no one
    if (mine && lane == __ffs(group) - 1) {
      float* g = table + 3 * (size_t)key;
      float a0 = g[0], a1 = g[1], a2 = g[2];
      for (unsigned m = group; m; m &= m - 1) {
        const size_t i = 3 * (size_t)(base + __ffs(m) - 1);
        if (g_loss) {
          a0 = __fadd_rn(a0, __fadd_rn(g_render[i], g_loss[i]));
          a1 = __fadd_rn(a1, __fadd_rn(g_render[i + 1], g_loss[i + 1]));
          a2 = __fadd_rn(a2, __fadd_rn(g_render[i + 2], g_loss[i + 2]));
        } else {
          a0 = __fadd_rn(a0, g_render[i]);
          a1 = __fadd_rn(a1, g_render[i + 1]);
          a2 = __fadd_rn(a2, g_render[i + 2]);
        }
      }
      g[0] = a0; g[1] = a1; g[2] = a2;
    }
    __syncwarp();  // this group's rows are written (and visible to the warp) before the next group reads them
  }
}

cudaError_t launch_background_rows(const int* pixel_rc, int n_rays, int H, int W, const float* g_render, const float* g_loss,
                                   float* table_grads, cudaStream_t st, long long* launches) {
  if (n_rays <= 0) return cudaSuccess;
  background_rows_kernel<<<kBgBlocks, kBgWarps * 32, 0, st>>>(pixel_rc, n_rays, H, W, g_render, g_loss, table_grads);
  ++*launches;
  return cudaGetLastError();
}

// The supervised background term (nfb_loss_background_grad; order: include/nfb.h), 0.001 * mean(w_last * ||bg - target||^2) in
// the reference: per ray d = bg - t, e = (d0 d0 + d1 d1) + d2 d2, then g_bg = (2 d) (s w), g_w = s e and the loss term w e, with
// s = weight * (1 / n_total).  ONE block, the loss terms meeting in loss_grad_kernel's fixed order.
__global__ void __launch_bounds__(kLossThreads) loss_background_kernel(const float* __restrict__ bg, const float* __restrict__ target,
                                                                       const float* __restrict__ w_last, int n_rays, float s,
                                                                       float* __restrict__ g_bg, float* __restrict__ g_w,
                                                                       float* __restrict__ loss) {
  __shared__ float part[kLossThreads / 32];
  float acc = 0.f;
  for (int r = threadIdx.x; r < n_rays; r += kLossThreads) {
    const size_t i = 3 * (size_t)r;
    const float d0 = __fsub_rn(bg[i], target[i]), d1 = __fsub_rn(bg[i + 1], target[i + 1]), d2 = __fsub_rn(bg[i + 2], target[i + 2]);
    const float e = __fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2));
    const float w = w_last[r], sw = __fmul_rn(s, w);
    g_bg[i] = __fmul_rn(2.f * d0, sw);
    g_bg[i + 1] = __fmul_rn(2.f * d1, sw);
    g_bg[i + 2] = __fmul_rn(2.f * d2, sw);
    g_w[r] = __fmul_rn(s, e);
    acc = __fadd_rn(acc, __fmul_rn(w, e));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  const int wp = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) part[wp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float sum = 0.f;
    for (int k = 0; k < kLossThreads / 32; ++k) sum = __fadd_rn(sum, part[k]);
    loss[0] = __fadd_rn(loss[0], __fmul_rn(sum, s));
  }
}

cudaError_t launch_loss_background(const float* bg, const float* target, const float* w_last, int n_rays, long long n_total, float weight,
                                   float* g_bg, float* g_w, float* loss, cudaStream_t st, long long* launches) {
  if (n_rays <= 0) return cudaSuccess;
  const float s = weight * (1.f / (float)n_total);  // two FP32 roundings, as autograd's mean backward forms it on CUDA
  loss_background_kernel<<<1, kLossThreads, 0, st>>>(bg, target, w_last, n_rays, s, g_bg, g_w, loss);
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_loss_grad(const float* rgb_c, const float* rgb_f, const float* target, int n_rays, long long n_total, float* g_c,
                             float* g_f, float* loss, cudaStream_t st, long long* launches) {
  const int n = 3 * n_rays;
  if (n <= 0) return cudaSuccess;
  loss_grad_kernel<<<1, kLossThreads, 0, st>>>(rgb_c, rgb_f, target, n, 1.f / (3.f * (float)n_total), g_c, g_f, loss);
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_adam(float* p, float* g, float* m, float* v, long long n, float lr, float b1, float b2, float eps, int step,
                        float grad_scale, long long reg_off, float reg_w, cudaStream_t st, long long* launches) {
  AdamArgs a;
  a.p = p; a.g = g; a.m = m; a.v = v; a.n = n;
  const double bc1 = 1.0 - pow((double)b1, (double)step), bc2 = 1.0 - pow((double)b2, (double)step);
  a.lr_over_bc1 = (float)((double)lr / bc1);
  a.sqrt_bc2 = (float)sqrt(bc2);
  a.b1 = b1; a.b2 = b2; a.eps = eps; a.grad_scale = grad_scale;
  a.reg_off = reg_off; a.reg_w = reg_w;
  long long blocks = (n + 255) / 256;
  if (blocks > 148 * 8) blocks = 148 * 8;
  adam_kernel<<<(int)blocks, 256, 0, st>>>(a);
  ++*launches;
  return cudaGetLastError();
}

}  // namespace nfb
