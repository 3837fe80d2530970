// nfb_internal.h — what the C-ABI layer (nfb_api.cu) and the kernel files share: the handle's device buffers, the parameter
// blocks of the preparation (nfb_pack.cu), render (nfb_render.cu), training (nfb_train.cu, nfb_optim.cu) and post-processing
// (nfb_post.cu) kernels, and their launchers.  Not part of the public interface.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "nfb_layout.h"
#include "nfb_sampler.h"

namespace nfb {

// A device allocation its owner frees.  Grow-only; what it held is gone once it has grown.  Built with a counter, it adds one to
// it every time it frees a live allocation to grow (nfb_buffer_epoch: addresses taken before are stale).
template <class T>
class DevBuf {
 public:
  DevBuf() = default;
  explicit DevBuf(long long* frees) : frees_(frees) {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { cudaFree(p_); }
  T* get() const { return p_; }
  // Room for n elements: allocates anew only when there is none or less.  *grew, when asked for, says whether it did.
  cudaError_t reserve(size_t n, bool* grew = nullptr) {
    if (grew) *grew = false;
    if (p_ && cap_ >= n) return cudaSuccess;
    if (p_ && frees_) ++*frees_;
    cudaError_t e = p_ ? cudaFree(p_) : cudaSuccess;
    p_ = nullptr; cap_ = 0;
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&p_), n * sizeof(T));
    if (e != cudaSuccess) return e;
    cap_ = n;
    if (grew) *grew = true;
    return cudaSuccess;
  }

 private:
  T* p_ = nullptr;
  size_t cap_ = 0;
  long long* frees_ = nullptr;
};

// Device buffers of one loaded network.
struct NetBuffers {
  DevBuf<uint8_t> stream_x1;  // kStreamBytesX1: FP16 weights, swizzled units in execution order
  DevBuf<uint8_t> stream_x3;  // kStreamBytesX3: hi unit, lo unit, ...
  DevBuf<float> w6;           // [144,256] folded layers_dir.0 / fc_alpha
  DevBuf<float> b6;           // [144]
  DevBuf<float> bias_static;  // [kBiasFloats]
  DevBuf<float> bias_frame;   // [kBiasFloats] bias_static + per-frame fold (what the kernel reads)
  DevBuf<float> w0c;          // [256,108] conditioning columns of layers_xyz.0
  DevBuf<float> w3c;          // [256,108] conditioning columns of layers_xyz.3
  DevBuf<float> wd0b_t;       // [24,128] direction columns of layers_dir.0, transposed
  DevBuf<uint8_t> stream_bwd; // kBwdStreamBytes: transposed FP16 weights for the backward chain (nfb_train.cu)
  DevBuf<uint8_t> stream_bwd_lo;  // kBwdStreamBytes: its lo half (exact-grad mode; allocated and written from the first such forward)
  bool loaded = false;
};

// Everything the render kernel needs, passed by value (__grid_constant__).
struct RenderParams {
  // rays
  const float* o;
  const float* d;
  float pose[12];
  float fx, fy, wcx, hcy;  // intrinsics as FP32; wcx = width*cx, hcy = height*cy (rounded like torch does)
  int width, row_begin;
  float near_, far_;
  const float* dir_z;
  const float* bg;
  // sampling
  TileGeom geom;          // rays, samples per ray, and how they are cut into units and tiles
  int perturb;
  float noise_std;
  int white_bkgd;
  const float* t_coarse;  // [nc]
  const float* u_fine;    // [nf]
  const float *t_rand, *noise_c, *u_rand, *noise_f;
  // networks
  const uint8_t* wstream[2];
  const float* bias[2];
  const float* wd0b_t[2];
  // outputs
  float *rgb_c, *disp_c, *acc_c, *rgb_f, *disp_f, *acc_f, *w_last;
  // training forward (all null in evaluation): per-tile activation records (nfb_layout.h kRec*), per-ray |d|, and per
  // sample (colour or bg, ReLU input of sigma) of both passes
  uint8_t* save_rec;
  float* save_dnorm;
  float* save_ray;  // optional [n][7] = (o, d, direction-encoder input d_z or dir_z)
  float *save_raw_c, *save_raw_f;
  // debug
  float *dbg_z_c, *dbg_raw_c, *dbg_z_f, *dbg_raw_f, *dbg_act;
  int dbg_act_step;
  unsigned long long* prof;  // optional [64] phase-cycle counters (see PhaseTimer in nfb_render.cu)
  // multi-frame call (render_frames_kernel; unused by render_kernel): per-ray frame index and the folded rows of steps 0 and 3 per
  // (network, frame) — kFrameRows floats per frame, then the NaN row an out-of-range index selects (nfb_pack.cu: frames_fold_kernel)
  const int* frame;
  int n_frames;
  const float* fbias[2];
  int* save_frame;  // training forward: [n] the frame slot each ray was rendered with (n_frames when out of range)
};

// ---- training (nfb_train.cu)
struct CompBwdParams {
  TileGeom geom;
  int has_bg, white_bkgd;
  const float *z_c, *raw_c, *z_f, *raw_f, *dnorm;                       // saved by the training forward
  const float *g_rgb[2], *g_disp[2], *g_acc[2], *g_wlast;               // dL/d outputs (coarse, fine); any may be null
  float* draw;                                                          // [tiles][128][4] dL/d(rgb_raw, sigma_raw), zero-initialised
  float* bsum;                                                          // [pass][ray][4] per-ray sums of d raw (grad_reduce_kernel adds them into kAccBRaw)
  unsigned int* absmax;                                                 // max |d raw| as float bits
  float *ray_dn, *ray_bg;  // non-null: input-gradient terms per (pass, ray): dL/d|d| [2][n], w_last G_rgb [2][n][3] (with a background)
};
// Input gradients (nfb_render_backward_ex): per-row (dp, d v0) of every tile, then per-ray sums.
struct InGradRowParams {
  const uint8_t* rec;
  TileGeom geom;
  int parts[2];                       // CTAs working on network 0 / network 1
  const float *z_c, *z_f, *ray;        // ray: the training forward's [n][7] = (o, d, v0)
  const float* scal;
  const float *w0[2], *w3[2], *wd0[2];  // FP32 layers_xyz.0 / .3 / layers_dir.0 weights of the two networks
  float* out;                         // [tiles][128] float4
};
struct InGradRayParams {
  TileGeom geom;
  int has_dir_z;
  const float *rows, *z_c, *z_f, *ray, *dnorm, *ray_dn, *ray_bg;
  float *g_o, *g_d, *g_dir_z, *g_bg;  // any may be null
};
struct ChainParams {
  TileGeom geom;
  uint8_t* rec;
  const float* draw;
  const float* scal;            // [0] = loss scale, [1] = 1 / scale
  const uint8_t* wstream[2];    // backward weight streams (coarse, fine)
  const uint8_t* wstream_lo[2]; // their lo halves (the exact-grad chain only)
};
struct DwParams {  // ONE launch covers both networks: the first parts[0] * groups CTAs work on network 0, the rest on network 1
  const uint8_t* rec;
  TileGeom geom;
  int parts[2];             // CTAs per job group of network i (set by launch_dw, proportional to the tile counts)
  float* ws;                // partial sums: slot (network 0's parts, then network 1's) of ws_stride floats per part
  int ws_stride;            // set by launch_dw: kAccBRaw, or the compact PE-only slot (nfb_train.cu dw::kPeSlotFloats)
  const float* scal;
};
// Multi-frame backward (nfb_render_backward_frames): per-ray sums of dY0 and dY3 from the tile records, then per-frame sums.
struct FrameSumParams {
  const uint8_t* rec;
  TileGeom geom;
  const float* scal;
  const int* frame;  // [n] frame slot per ray, saved by the training forward
  int n_frames;
  float* raysum;     // [passes][n][kFrameRows] scratch
  float* fsum;       // [n_frames][2][kFrameRows]: += this chunk's per-frame sums (zeroed before the first chunk)
};
// host copies of the compile-time schedules (nfb_debug_schedule); index < 0: number of entries; else words written or -1
int debug_jobs_dw(int index, uint32_t* out);
int debug_dw_split(uint32_t* io);  // io: {num_sms, tiles net 0, tiles net 1} -> {parts0, parts1, groups}
cudaError_t train_kernels_setup();
cudaError_t launch_composite_bwd(const CompBwdParams& q, float* scal, cudaStream_t st, long long* launches);
// hilo (exact-grad mode, here and below): the records are 2 MiB apart and hold lo halves (nfb_layout.h rec_stride); the kernels
// multiply and sum hi + lo.
cudaError_t launch_chain(const ChainParams& p, int num_sms, cudaStream_t st, long long* launches, bool hilo = false);
// Writes one partial per (network, part) into p.ws and fills in p.parts / p.ws_stride for launch_grad_reduce.
cudaError_t launch_dw(DwParams& p, int num_sms, cudaStream_t st, long long* launches, bool pe_only = false, bool hilo = false);
size_t dw_workspace_floats(int num_sms);  // floats of DwParams::ws that either weight-gradient launch may write
// One launch: acc[net] += the partials of the weight-gradient launch `d` in ascending part order (d == nullptr: there was none),
// and acc[pass][kAccBRaw..+4] += the compositing backward's per-ray sums bsum[pass][0..n_rays) in a fixed order.
cudaError_t launch_grad_reduce(const DwParams* d, bool pe_only, const float* bsum, int n_rays, int npass, float* const acc[2], int num_sms,
                               cudaStream_t st, long long* launches);
// grads_c == nullptr: input-gradient-only backward (d latent and d expression alone, one small launch).  cond == nullptr: the
// conditioning columns of dW0 / dW3 are left to launch_frames_grad.
cudaError_t launch_finalize_all(const float* const params_c[26], float* const grads_c[26], const float* acc_c,
                                const float* const params_f[26], float* const grads_f[26], const float* acc_f, const float* cond,
                                float* latent_out, cudaStream_t st, long long* launches, float* expr_out = nullptr);
cudaError_t launch_frame_sums(const FrameSumParams& p, cudaStream_t st, long long* launches, bool hilo = false);
// d latent_f, d expression_f [n_frames][32 / 76] from the per-frame sums, and (grads_* non-null) the conditioning columns of dW0 / dW3
// as sum_f db_f (x) c_f.  One launch.
cudaError_t launch_frames_grad(const float* const params_c[26], float* const grads_c[26], const float* const params_f[26],
                               float* const grads_f[26], const float* fsum, const float* fcond, int n_frames, float* latent_out,
                               float* expr_out, cudaStream_t st, long long* launches);
cudaError_t launch_input_grads(const InGradRowParams& r, const InGradRayParams& q, int num_sms, cudaStream_t st, long long* launches,
                               bool hilo = false);

// Two launches (fold, pack): FP32 parameters of n_nets (1 or 2) networks -> forward / backward weight streams, bias block, conditioning and
// direction columns (nfb_pack.cu: repack_kernel).
cudaError_t launch_repack(NetBuffers* const nb[2], const float* const* const params[2], int n_nets, cudaStream_t st, long long* launches);
// One launch: the lo half of the backward stream of n_nets networks (stream_bwd_lo, reserved by the caller) from their x3 streams.
cudaError_t launch_bwd_lo(NetBuffers* const nb[2], int n_nets, cudaStream_t st, long long* launches);
// One launch: per-frame bias fold of the loaded networks + cond[108] = [expr / 3 ; latent].
cudaError_t launch_frame_fold(NetBuffers* const nb[2], int n_nets, const float* expr, const float* latent, float* cond,
                              cudaStream_t st, long long* launches);
// One launch: the fold of n_frames frames into table[net] ([n_frames + 1][kFrameRows], the last row NaN) + cond[n_frames][108].
cudaError_t launch_frames_fold(NetBuffers* const nb[2], int n_nets, int n_frames, const float* expr, const float* latent,
                               float* const table[2], float* cond, cudaStream_t st, long long* launches);
// Training-step tail (nfb_optim.cu): d mse / d rgb (+ loss sums), Adam over a flat bucket with zero_grad fused.
cudaError_t launch_loss_grad(const float* rgb_c, const float* rgb_f, const float* target, int n_rays, long long n_total, float* g_c,
                             float* g_f, float* loss, cudaStream_t st, long long* launches);
cudaError_t launch_adam_dev(float* p, float* g, float* m, float* v, long long n, void* dev_state, cudaStream_t st, long long* launches);
cudaError_t launch_adam(float* p, float* g, float* m, float* v, long long n, float lr, float b1, float b2, float eps, int step,
                        float grad_scale, long long reg_off, float reg_w, cudaStream_t st, long long* launches);
// precision: 0 = fast (x1), 1 = exact (x3), 2 = exact-grad (exact mode's kernels; a training forward writes the lo records too).
// num_sms = CTAs to launch at most.  p.frame set: a multi-frame call (render_frames_kernel), where p.frame and p.fbias select
// each ray's rows of steps 0 and 3.
cudaError_t launch_render(const RenderParams& p, int precision, int num_sms, cudaStream_t st, long long* launches);
cudaError_t render_kernel_setup();  // opt-in to the large dynamic shared memory size

// ---- either side of the path (nfb_post.cu)
cudaError_t launch_frame_products(const float* rgb, const float* disp, const float* w_last, const double intr[4], int H, int W,
                                  uint8_t* rgb_u8, uint8_t* normals_u8, uint8_t* disp_u8, uint32_t* minmax_scratch, int like_torch_cpu,
                                  cudaStream_t st, long long* launches);
constexpr int kSmpMax = 2048;  // rays per sampler call (num_random_rays of the shipped YAML)
struct SampleArgs {
  smp::Map map;
  const double* draws;   // uniform [0,1) doubles, consumed like RandomState.rand: round r takes (size - n_found) values
  int size, max_rounds;
  long long* found;      // [size] selected flat indices in selection order (= np.random.choice's return value)
  int* state;            // [0] n_found, [1] rounds run, [2] draws consumed  (in/out: a call may resume a partial selection)
  smp::Run* runs;
  smp::Seg* segs;
  int* first_pos;        // [H * W] scratch, all INT_MAX between calls
  // gathers (any output may be null)
  float pose[12];
  float fx, fy, wcx, hcy;
  const float* image;       // [H, W, 3]
  const float* background;  // [H, W, 3]
  float *ray_o, *ray_d, *target, *bg_out;  // [size, 3] each
  int* pixel_rc;            // [size, 2] (row, col) of the selected pixels
};

cudaError_t launch_sample_rays(const SampleArgs& a, cudaStream_t st, long long* launches);

// Training rays of K images in one launch (nfb_sample_rays_images): block k selects n = size pixels of image image_index[k] as
// sample_rays_kernel does (draws [K][max_rounds * size], block k reads its own slice) and writes rays k*size.. of the batch.
constexpr int kMaxStepImages = 64;
struct RayMapRec { int H, W; int bbox[4]; double q_out, q_in; };  // mirrors NfbRayMap (include/nfb.h)
struct ImageSampleArgs {
  // dataset (device tables; images and background may be pinned host memory)
  const RayMapRec* maps;     // [n_images]
  const float* poses;        // [n_images][12]
  const float* expr_table;   // [n_images][kDimExpr]
  const float* images;       // [n_images][H][W][3]
  const float* background;   // [H][W][3] or null
  int n_images, H, W;
  float fx, fy, wcx, hcy;
  // this step
  const int* image_index;    // [K]
  int K, size, max_rounds;
  const double* draws;       // [K][max_rounds * size]
  const float* latent_table; // [n_images][kDimLatent]
  // per-image scratch: [K][kMaxRuns], [K][kMaxSegs], [K][H * W] (all INT_MAX between calls), [K][size]
  smp::Run* runs;
  smp::Seg* segs;
  int* first_pos;
  long long* found;
  // outputs, any may be null: [K * size] rows of the batch, [K] conditioning rows, [K][3] state, [K] running shortfall
  float *ray_o, *ray_d, *target, *bg_out;
  int* pixel_rc;
  long long* indices;
  int* frame;
  float *expr_out, *latent_out;
  int* state;
  long long* shortfall;
};
cudaError_t launch_sample_images(const ImageSampleArgs& a, cudaStream_t st, long long* launches);
// One launch (nfb_optim.cu): the latent-table rows of the bucket gradient for a step over K images (order: include/nfb.h,
// nfb_latent_rows_grad).
cudaError_t launch_latent_rows(const float* grad_latents, const int* image_index, int K, const float* table, int n_rows, float* table_grads,
                               float reg_w, cudaStream_t st, long long* launches);
// One or two launches (nfb_optim.cu): the pose rows (slot sums into `slots` [K][12], then the rows) and the expression rows of a
// fitting step over K images (order: include/nfb.h, nfb_fit_rows_grad).  pose_grads NULL: the expression rows only, one launch.
cudaError_t launch_fit_rows(const int* image_index, int K, int n, int n_rows, const int* pixel_rc, const float* g_o, const float* g_d,
                            float fx, float fy, float wcx, float hcy, float* slots, float* pose_grads, const float* g_expr,
                            float* expr_grads, cudaStream_t st, long long* launches);
// One launch each (nfb_optim.cu; none for n_rays == 0): a learned background's rows of the bucket gradient, and the supervised
// background loss with its two gradients (orders: include/nfb.h, nfb_background_rows_grad / nfb_loss_background_grad).
cudaError_t launch_background_rows(const int* pixel_rc, int n_rays, int H, int W, const float* g_render, const float* g_loss,
                                   float* table_grads, cudaStream_t st, long long* launches);
cudaError_t launch_loss_background(const float* bg, const float* target, const float* w_last, int n_rays, long long n_total, float weight,
                                   float* g_bg, float* g_w, float* loss, cudaStream_t st, long long* launches);
cudaError_t launch_fill_int(int* p, long long n, int v, cudaStream_t st, long long* launches);

}  // namespace nfb
