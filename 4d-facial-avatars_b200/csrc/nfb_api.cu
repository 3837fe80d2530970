// nfb_api.cu — the C ABI declared in include/nfb.h: handle management, argument validation, and
// translation of the public structs into kernel launches.  No torch, no exceptions across the boundary.
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "../../include/nfb.h"
#include "nfb_internal.h"
#include "nfb_layout.h"

namespace {
thread_local std::string g_last_cuda_error;

int cuda_fail(cudaError_t e, const char* where) {
  g_last_cuda_error = std::string(where) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
  return NFB_ERR_CUDA;
}
#define NFB_CUDA(call)                                   \
  do {                                                   \
    cudaError_t e__ = (call);                            \
    if (e__ != cudaSuccess) return cuda_fail(e__, #call); \
  } while (0)
}  // namespace

using nfb::DevBuf;
static_assert(NFB_MAX_FRAMES == nfb::kMaxFrames, "frame bound");
static_assert(NFB_MAX_STEP_IMAGES == nfb::kMaxStepImages, "image bound");
static_assert(sizeof(NfbRayMap) == sizeof(nfb::RayMapRec) && offsetof(NfbRayMap, q_out) == offsetof(nfb::RayMapRec, q_out),
              "NfbRayMap mirror");

struct NfbHandle {
  int device = 0;
  int num_sms = 0;
  nfb::NetBuffers net[2];
  bool frame_set = false;
  // exact-grad mode: set by the first exact-grad training forward, which allocates and writes the backward stream's lo halves; from
  // then on every weight load and re-pack rewrites them (NetBuffers::stream_bwd_lo).  Fast and exact handles never pay for them.
  bool bwd_lo = false;
  long long launches = 0;
  // nfb_buffer_epoch = frees + tr.frees: the buffers a training step's launches take an address of count their re-allocations
  // into one of the two (the linspace tables count every refill for another n)
  long long frees = 0;
  // cached torch.linspace(0,1,n) tables on the device, and the n each was filled for
  DevBuf<float> lin_c, lin_f;
  int lin_c_n = 0, lin_f_n = 0;
  // staging for nfb_render_frame_host
  DevBuf<float> d_expr, d_latent, d_bg, d_out;
  // training state: what nfb_render_forward_train saved for nfb_render_backward (grow-only buffers)
  struct Train {
    long long frees = 0;
    DevBuf<uint8_t> rec{&frees};                        // per-tile activation records (nfb_layout.h kRec*)
    DevBuf<float> draw{&frees};                         // [tiles][128][4]
    DevBuf<float> z_c{&frees}, raw_c{&frees}, z_f{&frees}, raw_f{&frees}, dnorm{&frees};
    DevBuf<float> acc[2]{DevBuf<float>(&frees), DevBuf<float>(&frees)};  // kAccFloats each
    // what the backward sums in a fixed order instead of with atomics: per-ray bias sums of the compositing backward
    // ([pass][ray][4]) and one weight-gradient partial per (network, part) (nfb::dw_workspace_floats)
    DevBuf<float> bsum{&frees}, dw_ws{&frees};
    DevBuf<float> scal{&frees};                         // [0] scale, [1] 1/scale, [2] max |d raw| (bits)
    DevBuf<float> cond{&frees};                         // [108] conditioning vector of the frame the forward rendered
    nfb::TileGeom geom = {};                            // of the whole forward call
    int has_bg = 0, white_bkgd = 0;
    bool valid = false;
    // for input gradients (nfb_render_backward_ex): the forward's rays (copied unless chunked), per-row / per-ray scratch
    bool has_rays = false, has_dir_z = false;
    DevBuf<float> ray{&frees};                          // [n][7] = (o, d, v0), written by the SAVE forward
    DevBuf<float> rows{&frees};                         // [tiles][128][4]
    DevBuf<float> ray_dn{&frees}, ray_bg{&frees};
    // what the last one-launch backward of this forward left in ray_dn / ray_bg, rows and raysum / fsum (nfb_train_debug)
    bool per_ray_formed = false, rows_formed = false, frame_sums_formed = false;
    // ... and in dw_ws / bsum: the split and slot size of its weight-gradient launch (dw_parts 0, 0: none ran)
    bool bwd_formed = false, dw_pe_only = false;
    int dw_parts[2] = {0, 0}, dw_stride = 0;
    // chunked mode (the records of the whole call would exceed the memory budget): the forward only produced the outputs; the
    // backward re-runs the training forward chunk by chunk from the saved launch parameters (the caller keeps the inputs alive)
    bool chunked = false;
    nfb::RenderParams full;      // the forward call's parameters (pointers into caller memory)
    // handle-owned state `full` points at, copied at the forward: the folded per-frame biases (nfb_set_frame overwrites
    // bias_frame in place) and the linspace tables when they came from the handle's cache (a later sample count replaces it)
    DevBuf<float> bias[2]{DevBuf<float>(&frees), DevBuf<float>(&frees)};
    DevBuf<float> lin_c{&frees}, lin_f{&frees};
    int chunk_rays = 0, precision = 0;
    bool hilo = false;                   // an exact-grad forward: 2 MiB records with lo halves, the *_x3 backward kernels
    DevBuf<float> scratch_out{&frees};   // [11 * chunk_rays] outputs of the re-run forwards (discarded)
    // multi-frame forward (nfb_render_forward_frames_train): the frame table and conditioning vectors it rendered with (copied,
    // as bias / cond are), the frame slot of every ray (written by the forward), and the backward's per-ray / per-frame sums
    bool multi = false;
    int n_frames = 0;
    DevBuf<float> ftab[2]{DevBuf<float>(&frees), DevBuf<float>(&frees)}, fcond{&frees};
    DevBuf<int> frame{&frees};
    DevBuf<float> raysum{&frees}, fsum{&frees};
  } tr;
  size_t train_budget = 0;       // bytes the per-tile records of one launch may take (0: not decided yet)
  DevBuf<float> cond;            // [108] = [expression / 3 ; latent] of the current frame
  // nfb_set_frames: per network [n_frames + 1][kFrameRows] folded rows (the last NaN), and [n_frames][108] conditioning vectors;
  // independent of the single frame above
  DevBuf<float> ftab[2]{DevBuf<float>(&frees), DevBuf<float>(&frees)}, fcond{&frees};
  int n_frames = 0;
  // scratch of the steps either side of the path
  DevBuf<uint32_t> minmax;       // disparity-image min / max keys
  DevBuf<nfb::smp::Run> smp_runs;
  DevBuf<nfb::smp::Seg> smp_segs;
  DevBuf<int> smp_first;
  // nfb_sample_rays_images: per-image copies of the above, and the selected indices
  DevBuf<nfb::smp::Run> smpi_runs{&frees};
  DevBuf<nfb::smp::Seg> smpi_segs{&frees};
  DevBuf<int> smpi_first{&frees};
  DevBuf<long long> smpi_found{&frees};
  // nfb_fit_rows_grad: the per-slot pose sums [NFB_MAX_STEP_IMAGES][12] (allocated once at full size, so it never moves)
  DevBuf<float> fit_slots{&frees};
};

extern "C" {

int nfb_version(void) { return NFB_VERSION; }

const char* nfb_strerror(int status) {
  switch (status) {
    case NFB_OK: return "ok";
    case NFB_ERR_INVALID: return "invalid argument";
    case NFB_ERR_UNSUPPORTED: return "configuration not supported by the sm_90a render kernel";
    case NFB_ERR_CUDA: return "CUDA runtime error (see nfb_last_cuda_error)";
    case NFB_ERR_STATE: return "weights or per-frame conditioning not set";
    case NFB_ERR_ARCH: return "device is not compute capability 9.0 (sm_90a code only)";
    default: return "unknown status";
  }
}

const char* nfb_last_cuda_error(void) { return g_last_cuda_error.c_str(); }

int nfb_host_linspace(float* out, int n) {
  if (!out || n < 1) return NFB_ERR_INVALID;
  if (n == 1) { out[0] = 0.f; return NFB_OK; }
  // ATen's CPU linspace: symmetric evaluation about the midpoint, all in FP32.
  const float start = 0.f, end = 1.f;
  const float step = (end - start) / static_cast<float>(n - 1);
  const int halfway = n / 2;
  for (int i = 0; i < n; ++i) out[i] = (i < halfway) ? start + step * static_cast<float>(i) : end - step * static_cast<float>(n - i - 1);
  return NFB_OK;
}

static int create_impl(NfbHandle* h, const cudaDeviceProp& prop) {
  h->num_sms = prop.multiProcessorCount;
  for (int n = 0; n < 2; ++n) {
    nfb::NetBuffers& nb = h->net[n];
    NFB_CUDA(nb.stream_x1.reserve(nfb::kStreamBytesX1));
    NFB_CUDA(nb.stream_x3.reserve(nfb::kStreamBytesX3));
    NFB_CUDA(nb.w6.reserve(144 * 256));
    NFB_CUDA(nb.b6.reserve(144));
    NFB_CUDA(nb.bias_static.reserve(nfb::kBiasFloats));
    NFB_CUDA(nb.bias_frame.reserve(nfb::kBiasFloats));
    NFB_CUDA(nb.w0c.reserve(256 * nfb::kDimCond));
    NFB_CUDA(nb.w3c.reserve(256 * nfb::kDimCond));
    NFB_CUDA(nb.wd0b_t.reserve(nfb::kDimDir * 128));
    NFB_CUDA(nb.stream_bwd.reserve(nfb::kBwdStreamBytes));
    NFB_CUDA(h->tr.acc[n].reserve(nfb::kAccFloats));
  }
  NFB_CUDA(h->tr.scal.reserve(4));
  NFB_CUDA(h->tr.cond.reserve(nfb::kDimCond));
  NFB_CUDA(h->cond.reserve(nfb::kDimCond));
  NFB_CUDA(nfb::train_kernels_setup());
  NFB_CUDA(h->d_expr.reserve(nfb::kDimExpr));
  NFB_CUDA(h->d_latent.reserve(nfb::kDimLatent));
  NFB_CUDA(nfb::render_kernel_setup());
  return NFB_OK;
}


int nfb_create(const NfbModelDims* dims, int device, NfbHandle** out) {
  if (!dims || !out) return NFB_ERR_INVALID;
  if (dims->num_encoding_fn_xyz != 10 || dims->num_encoding_fn_dir != 4 || dims->include_input_xyz != 1 ||
      dims->include_input_dir != 0 || dims->dim_expression != nfb::kDimExpr || dims->dim_latent != nfb::kDimLatent)
    return NFB_ERR_UNSUPPORTED;
  NFB_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  NFB_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return NFB_ERR_ARCH;
  NfbHandle* h = new (std::nothrow) NfbHandle();
  if (!h) return NFB_ERR_INVALID;
  h->device = device;
  const int rc = create_impl(h, prop);
  if (rc != NFB_OK) {  // frees whatever was allocated before the failure
    nfb_destroy(h);
    return rc;
  }
  *out = h;
  return NFB_OK;
}

int nfb_destroy(NfbHandle* h) {
  if (!h) return NFB_ERR_INVALID;
  cudaSetDevice(h->device);
  delete h;
  return NFB_OK;
}

int nfb_load_weights(NfbHandle* h, int which, const float* const params[26], void* stream) {
  if (!h || !params || (which != NFB_NET_COARSE && which != NFB_NET_FINE)) return NFB_ERR_INVALID;
  for (int i = 0; i < 26; ++i)
    if (!params[i]) return NFB_ERR_INVALID;
  NFB_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  nfb::NetBuffers& nb = h->net[which];
  nfb::NetBuffers* const nbs[2] = {&nb, nullptr};
  const float* const* const ps[2] = {params, nullptr};
  NFB_CUDA(nfb::launch_repack(nbs, ps, 1, st, &h->launches));  // forward streams, transposed backward stream, bias / column blocks
  if (h->bwd_lo) NFB_CUDA(nfb::launch_bwd_lo(nbs, 1, st, &h->launches));
  nb.loaded = true;
  h->frame_set = false;  // folded biases are stale
  h->n_frames = 0;
  return NFB_OK;
}

int nfb_repack(NfbHandle* h, const float* const params_coarse[26], const float* const params_fine[26], void* stream) {
  if (!h || !params_coarse) return NFB_ERR_INVALID;
  for (int i = 0; i < 26; ++i)
    if (!params_coarse[i] || (params_fine && !params_fine[i])) return NFB_ERR_INVALID;
  NFB_CUDA(cudaSetDevice(h->device));
  nfb::NetBuffers* const nbs[2] = {&h->net[0], &h->net[1]};
  const float* const* const ps[2] = {params_coarse, params_fine};
  NFB_CUDA(nfb::launch_repack(nbs, ps, params_fine ? 2 : 1, static_cast<cudaStream_t>(stream), &h->launches));
  if (h->bwd_lo) NFB_CUDA(nfb::launch_bwd_lo(nbs, params_fine ? 2 : 1, static_cast<cudaStream_t>(stream), &h->launches));
  h->net[0].loaded = true;
  if (params_fine) h->net[1].loaded = true;
  h->frame_set = false;  // folded biases are stale
  h->n_frames = 0;
  return NFB_OK;
}

int nfb_loss_mse_grad(NfbHandle* h, const float* rgb_coarse, const float* rgb_fine, const float* target, int n_rays,
                      long long n_total, float* grad_rgb_coarse, float* grad_rgb_fine, float* loss, void* stream) {
  if (!h || !rgb_coarse || !target || !grad_rgb_coarse || !loss || n_rays < 0 || n_total < n_rays || n_total <= 0) return NFB_ERR_INVALID;
  if (rgb_fine && !grad_rgb_fine) return NFB_ERR_INVALID;
  NFB_CUDA(cudaSetDevice(h->device));
  NFB_CUDA(nfb::launch_loss_grad(rgb_coarse, rgb_fine, target, n_rays, n_total, grad_rgb_coarse, grad_rgb_fine, loss,
                                 static_cast<cudaStream_t>(stream), &h->launches));
  return NFB_OK;
}

int nfb_adam_step(NfbHandle* h, float* params, float* grads, float* exp_avg, float* exp_avg_sq, long long n, const NfbAdam* hp,
                  void* stream) {
  if (!h || !params || !grads || !exp_avg || !exp_avg_sq || !hp || n <= 0 || hp->step < 1) return NFB_ERR_INVALID;
  // the regularised row must not straddle two 256-float chunks (one thread block each): its norm is taken per block
  if (hp->reg_offset >= 0 && (hp->reg_offset + nfb::kDimLatent > n || hp->reg_offset % nfb::kDimLatent != 0)) return NFB_ERR_INVALID;
  NFB_CUDA(cudaSetDevice(h->device));
  NFB_CUDA(nfb::launch_adam(params, grads, exp_avg, exp_avg_sq, n, hp->lr, hp->beta1, hp->beta2, hp->eps, hp->step, hp->grad_scale,
                            hp->reg_offset, hp->reg_weight, static_cast<cudaStream_t>(stream), &h->launches));
  return NFB_OK;
}

int nfb_adam_step_dev(NfbHandle* h, float* params, float* grads, float* exp_avg, float* exp_avg_sq, long long n, NfbAdamDev* dev_state,
                      void* stream) {
  if (!h || !params || !grads || !exp_avg || !exp_avg_sq || !dev_state || n <= 0) return NFB_ERR_INVALID;
  NFB_CUDA(cudaSetDevice(h->device));
  NFB_CUDA(nfb::launch_adam_dev(params, grads, exp_avg, exp_avg_sq, n, dev_state, static_cast<cudaStream_t>(stream), &h->launches));
  return NFB_OK;
}

int nfb_set_frame(NfbHandle* h, const float* expression, const float* latent, void* stream) {
  if (!h || !expression || !latent) return NFB_ERR_INVALID;
  if (!h->net[0].loaded) return NFB_ERR_STATE;
  NFB_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  nfb::NetBuffers* const nbs[2] = {&h->net[0], &h->net[1]};
  NFB_CUDA(nfb::launch_frame_fold(nbs, h->net[1].loaded ? 2 : 1, expression, latent, h->cond.get(), st, &h->launches));
  h->frame_set = true;
  return NFB_OK;
}

int nfb_set_frames(NfbHandle* h, const float* expressions, const float* latents, int n_frames, void* stream) {
  if (!h || !expressions || !latents || n_frames < 1) return NFB_ERR_INVALID;
  if (n_frames > NFB_MAX_FRAMES) return NFB_ERR_UNSUPPORTED;
  if (!h->net[0].loaded) return NFB_ERR_STATE;
  NFB_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nets = h->net[1].loaded ? 2 : 1;
  for (int n = 0; n < nets; ++n) NFB_CUDA(h->ftab[n].reserve((size_t)(n_frames + 1) * nfb::kFrameRows));
  NFB_CUDA(h->fcond.reserve((size_t)n_frames * nfb::kDimCond));
  nfb::NetBuffers* const nbs[2] = {&h->net[0], &h->net[1]};
  float* const tab[2] = {h->ftab[0].get(), h->ftab[1].get()};
  h->n_frames = 0;
  NFB_CUDA(nfb::launch_frames_fold(nbs, nets, n_frames, expressions, latents, tab, h->fcond.get(), st, &h->launches));
  h->n_frames = n_frames;
  return NFB_OK;
}

static int ensure_linspace(DevBuf<float>& buf, int* cached_n, int n, long long* frees, cudaStream_t st) {
  if (*cached_n == n && buf.get()) return NFB_OK;
  std::vector<float> host(n);
  nfb_host_linspace(host.data(), n);
  if (*cached_n) ++*frees;  // a table a graph may have captured now holds other values
  *cached_n = 0;
  NFB_CUDA(buf.reserve((size_t)n));
  // pageable source: the runtime stages it before returning, so `host` may die afterwards
  NFB_CUDA(cudaMemcpyAsync(buf.get(), host.data(), n * sizeof(float), cudaMemcpyHostToDevice, st));
  *cached_n = n;
  return NFB_OK;
}

// Memory the per-tile activation records of ONE training launch may take: NFB_TRAIN_MEM_MB, else 60 % of the device memory that
// is free when first asked (at least 1 GiB).  A call that needs more is processed in ray chunks (see NfbHandle::Train::chunked).
static size_t train_budget(NfbHandle* h) {
  if (const char* e = std::getenv("NFB_TRAIN_MEM_MB")) {  // read on every call: tests switch it within one process
    const size_t mb = (size_t)std::strtoull(e, nullptr, 10);
    if (mb) return mb << 20;
  }
  if (h->train_budget) return h->train_budget;
  size_t budget = 0;
  {
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) budget = free_b / 10 * 6;
  }
  if (budget < ((size_t)1 << 30)) budget = (size_t)1 << 30;
  return h->train_budget = budget;
}

// (Re)size the buffers a training launch of geometry g and its backward write.
static int ensure_train_buffers(NfbHandle::Train& tr, const nfb::TileGeom& g, int num_sms) {
  const size_t n = (size_t)g.n_rays, tiles = g.tiles();
  NFB_CUDA(tr.rec.reserve(tiles * nfb::rec_stride(tr.hilo)));
  NFB_CUDA(tr.draw.reserve(tiles * 512));
  NFB_CUDA(tr.bsum.reserve(8 * n));
  NFB_CUDA(tr.dw_ws.reserve(nfb::dw_workspace_floats(num_sms)));
  NFB_CUDA(tr.z_c.reserve(n * g.samples(0)));
  NFB_CUDA(tr.raw_c.reserve(n * g.samples(0) * 4));
  NFB_CUDA(tr.dnorm.reserve(n));
  NFB_CUDA(tr.ray.reserve(7 * n));
  if (tr.multi) {
    NFB_CUDA(tr.frame.reserve(n));
    NFB_CUDA(tr.raysum.reserve(2 * n * nfb::kFrameRows));
  }
  if (g.passes() == 2) {
    NFB_CUDA(tr.z_f.reserve(n * g.samples(1)));
    NFB_CUDA(tr.raw_f.reserve(n * g.samples(1) * 4));
  }
  return NFB_OK;
}

// A training forward (a whole one, or one chunk of it re-run by the backward) saves what the backward reads into tr's buffers.
static void set_save_slots(nfb::RenderParams& p, NfbHandle::Train& tr) {
  p.save_rec = tr.rec.get(); p.save_dnorm = tr.dnorm.get(); p.save_raw_c = tr.raw_c.get(); p.save_raw_f = tr.raw_f.get();
  p.dbg_z_c = tr.z_c.get(); p.dbg_z_f = tr.z_f.get();
  p.save_ray = tr.ray.get();  // the rays, for input gradients (the backward does not read the caller's buffers)
  if (tr.multi) p.save_frame = tr.frame.get();
}

// frame_index non-null: a multi-frame call (the frame table of nfb_set_frames instead of the frame of nfb_set_frame).
static int render_impl(NfbHandle* h, const NfbRays* rays, const NfbSampling* sm, const NfbNoise* noise, const NfbOutputs* out,
                       const NfbDebug* dbg, void* stream, bool train, const int32_t* frame_index = nullptr) {
  if (!h || !rays || !sm || !out) return NFB_ERR_INVALID;
  const bool multi = frame_index != nullptr;
  if (rays->n_rays < 0) return NFB_ERR_INVALID;
  if ((rays->o == nullptr) != (rays->d == nullptr)) return NFB_ERR_INVALID;
  if (!rays->o && (rays->width <= 0 || rays->height <= 0)) return NFB_ERR_INVALID;
  const int nc = sm->num_coarse, nf = sm->num_fine;
  if (nc < 3 || nf < 0 || nc + nf > 512) return NFB_ERR_UNSUPPORTED;
  if (sm->lindisp) return NFB_ERR_UNSUPPORTED;
  if (sm->precision != NFB_PREC_FAST && sm->precision != NFB_PREC_EXACT && sm->precision != NFB_PREC_EXACT_GRAD) return NFB_ERR_INVALID;
  if (multi && !rays->o) return NFB_ERR_UNSUPPORTED;  // in-kernel ray generation is one pose per call
  if (!h->net[0].loaded || (nf > 0 && !h->net[1].loaded) || (multi ? h->n_frames < 1 : !h->frame_set)) return NFB_ERR_STATE;
  if (!out->rgb_coarse || !out->disp_coarse || !out->acc_coarse) return NFB_ERR_INVALID;
  if (nf > 0 && (!out->rgb_fine || !out->disp_fine || !out->acc_fine)) return NFB_ERR_INVALID;
  if (sm->perturb && (!noise || !noise->t_rand || (nf > 0 && !noise->u))) return NFB_ERR_INVALID;
  if (sm->noise_std > 0.f && (!noise || !noise->sigma_noise_c || (nf > 0 && !noise->sigma_noise_f))) return NFB_ERR_INVALID;
  if (rays->n_rays == 0) return NFB_OK;
  NFB_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  nfb::RenderParams p;
  std::memset(&p, 0, sizeof(p));
  p.o = rays->o; p.d = rays->d;
  for (int i = 0; i < 12; ++i) p.pose[i] = rays->pose[i];
  p.fx = static_cast<float>(rays->intrinsics[0]);
  p.fy = static_cast<float>(rays->intrinsics[1]);
  p.wcx = static_cast<float>(static_cast<double>(rays->width) * rays->intrinsics[2]);
  p.hcy = static_cast<float>(static_cast<double>(rays->height) * rays->intrinsics[3]);
  p.width = rays->width > 0 ? rays->width : 1;
  p.row_begin = rays->row_begin;
  p.near_ = rays->near_; p.far_ = rays->far_;
  p.dir_z = rays->dir_z; p.bg = rays->background;
  p.geom = nfb::TileGeom::make(rays->n_rays, nc, nf);
  p.perturb = sm->perturb ? 1 : 0;
  p.noise_std = sm->noise_std;
  p.white_bkgd = sm->white_background ? 1 : 0;
  if (sm->t_coarse) p.t_coarse = sm->t_coarse;
  else {
    int rc = ensure_linspace(h->lin_c, &h->lin_c_n, nc, &h->frees, st);
    if (rc) return rc;
    p.t_coarse = h->lin_c.get();
  }
  if (nf > 0) {
    if (sm->u_fine) p.u_fine = sm->u_fine;
    else {
      int rc = ensure_linspace(h->lin_f, &h->lin_f_n, nf, &h->frees, st);
      if (rc) return rc;
      p.u_fine = h->lin_f.get();
    }
  }
  if (noise) { p.t_rand = noise->t_rand; p.noise_c = noise->sigma_noise_c; p.u_rand = noise->u; p.noise_f = noise->sigma_noise_f; }
  const bool exact = sm->precision != NFB_PREC_FAST;  // exact-grad renders with exact mode's streams and kernels
  for (int n = 0; n < 2; ++n) {
    p.wstream[n] = exact ? h->net[n].stream_x3.get() : h->net[n].stream_x1.get();
    // a multi-frame call takes the folded rows of steps 0 and 3 from the frame table; its other bias entries are the static ones
    p.bias[n] = multi ? h->net[n].bias_static.get() : h->net[n].bias_frame.get();
    p.wd0b_t[n] = h->net[n].wd0b_t.get();
    p.fbias[n] = multi ? h->ftab[n].get() : nullptr;
  }
  if (nf == 0) { p.wstream[1] = p.wstream[0]; p.bias[1] = p.bias[0]; p.wd0b_t[1] = p.wd0b_t[0]; p.fbias[1] = p.fbias[0]; }
  if (multi) { p.frame = frame_index; p.n_frames = h->n_frames; }
  p.rgb_c = out->rgb_coarse; p.disp_c = out->disp_coarse; p.acc_c = out->acc_coarse;
  p.rgb_f = out->rgb_fine; p.disp_f = out->disp_fine; p.acc_f = out->acc_fine; p.w_last = out->w_last;
  if (dbg) {
    p.dbg_z_c = dbg->z_coarse; p.dbg_raw_c = dbg->raw_coarse; p.dbg_z_f = dbg->z_fine; p.dbg_raw_f = dbg->raw_fine;
    p.dbg_act = dbg->act_dump; p.dbg_act_step = dbg->act_step; p.prof = dbg->prof;
  }
  if (train) {
    // Saved for nfb_render_backward: per-tile activation records, sample depths, (colour, ReLU input of sigma), |d|.
    NfbHandle::Train& tr = h->tr;
    tr.valid = false;
    tr.per_ray_formed = tr.rows_formed = tr.frame_sums_formed = tr.bwd_formed = false;
    int rc;
    tr.hilo = sm->precision == NFB_PREC_EXACT_GRAD;
    if (tr.hilo && !h->bwd_lo) {  // the first exact-grad training forward: the lo halves of the loaded backward streams
      for (int n = 0; n < 2; ++n) NFB_CUDA(h->net[n].stream_bwd_lo.reserve(nfb::kBwdStreamBytes));
      nfb::NetBuffers* const nbs[2] = {&h->net[0], &h->net[1]};
      NFB_CUDA(nfb::launch_bwd_lo(nbs, h->net[1].loaded ? 2 : 1, st, &h->launches));
      h->bwd_lo = true;
    }
    const size_t rec_bytes = nfb::rec_stride(tr.hilo);
    // a multi-frame backward also keeps per-ray dY0 / dY3 sums: 2 passes x kFrameRows floats = 4 KiB per ray, in the budget too
    const size_t ray_bytes = multi ? 2 * nfb::kFrameRows * sizeof(float) : 0;
    tr.chunked = p.geom.tiles() * rec_bytes + (size_t)p.geom.n_rays * ray_bytes > train_budget(h);
    tr.multi = multi;
    if (multi) {
      // the frame table and conditioning vectors this forward rendered with: a later nfb_set_frames must not change them
      const int nets = nf > 0 ? 2 : 1, F = h->n_frames;
      tr.n_frames = F;
      for (int n = 0; n < nets; ++n) {
        NFB_CUDA(tr.ftab[n].reserve((size_t)(F + 1) * nfb::kFrameRows));
        NFB_CUDA(cudaMemcpyAsync(tr.ftab[n].get(), h->ftab[n].get(), (size_t)(F + 1) * nfb::kFrameRows * sizeof(float),
                                 cudaMemcpyDeviceToDevice, st));
        p.fbias[n] = tr.ftab[n].get();
      }
      if (nf == 0) p.fbias[1] = p.fbias[0];
      NFB_CUDA(tr.fcond.reserve((size_t)F * nfb::kDimCond));
      NFB_CUDA(cudaMemcpyAsync(tr.fcond.get(), h->fcond.get(), (size_t)F * nfb::kDimCond * sizeof(float), cudaMemcpyDeviceToDevice, st));
      NFB_CUDA(tr.fsum.reserve((size_t)F * 2 * nfb::kFrameRows));
    }
    if (tr.chunked) {
      // e.g. a whole frame rendered with gradients enabled: 1.5-2 MiB of records per ray.  Keep the launch parameters, produce
      // the outputs with the evaluation kernel now, and let the backward re-run the training forward in chunks that fit.
      if (!rays->o) { g_last_cuda_error = "training forward over budget needs explicit rays (o, d)"; return NFB_ERR_UNSUPPORTED; }
      size_t units = train_budget(h) / ((size_t)p.geom.tiles_per_unit() * rec_bytes + (size_t)p.geom.rays_per_unit * ray_bytes);
      if (units < 1) units = 1;
      tr.chunk_rays = (int)(units * p.geom.rays_per_unit);
      tr.full = p;
      tr.precision = sm->precision;
      // the re-run forwards must read THIS call's frame and depth tables, whatever is rendered before the backward
      for (int n = 0; n < (nf > 0 ? 2 : 1); ++n) {
        NFB_CUDA(tr.bias[n].reserve(nfb::kBiasFloats));
        NFB_CUDA(cudaMemcpyAsync(tr.bias[n].get(), p.bias[n], nfb::kBiasFloats * sizeof(float), cudaMemcpyDeviceToDevice, st));
        tr.full.bias[n] = tr.bias[n].get();
      }
      if (nf == 0) tr.full.bias[1] = tr.full.bias[0];
      if (p.t_coarse == h->lin_c.get()) {
        NFB_CUDA(tr.lin_c.reserve((size_t)nc));
        NFB_CUDA(cudaMemcpyAsync(tr.lin_c.get(), h->lin_c.get(), nc * sizeof(float), cudaMemcpyDeviceToDevice, st));
        tr.full.t_coarse = tr.lin_c.get();
      }
      if (nf > 0 && p.u_fine == h->lin_f.get()) {
        NFB_CUDA(tr.lin_f.reserve((size_t)nf));
        NFB_CUDA(cudaMemcpyAsync(tr.lin_f.get(), h->lin_f.get(), nf * sizeof(float), cudaMemcpyDeviceToDevice, st));
        tr.full.u_fine = tr.lin_f.get();
      }
    } else if ((rc = ensure_train_buffers(tr, p.geom, h->num_sms))) return rc;
    // a later nfb_set_frame (e.g. a validation render before the backward) must not change what the backward differentiates
    if (!multi) NFB_CUDA(cudaMemcpyAsync(tr.cond.get(), h->cond.get(), nfb::kDimCond * sizeof(float), cudaMemcpyDeviceToDevice, st));
    else NFB_CUDA(cudaMemsetAsync(tr.cond.get(), 0, nfb::kDimCond * sizeof(float), st));
    if (!tr.chunked) set_save_slots(p, tr);
    tr.has_rays = rays->o != nullptr; tr.has_dir_z = rays->dir_z != nullptr;
    tr.geom = p.geom; tr.has_bg = rays->background != nullptr; tr.white_bkgd = p.white_bkgd;
  }
  // exact-grad mode runs its own kernel only where records are saved (p.save_rec); evaluation renders and the over-budget
  // training forward, which saves nothing until the backward re-runs it chunk by chunk, run exact mode's
  NFB_CUDA(nfb::launch_render(p, sm->precision, h->num_sms, st, &h->launches));
  if (train) h->tr.valid = true;
  return NFB_OK;
}

int nfb_render_forward_frames(NfbHandle* h, const NfbRays* rays, const int32_t* frame_index, const NfbSampling* sm, const NfbNoise* noise,
                              const NfbOutputs* out, void* stream) {
  if (!frame_index) return NFB_ERR_INVALID;
  return render_impl(h, rays, sm, noise, out, nullptr, stream, false, frame_index);
}

int nfb_render_forward_frames_train(NfbHandle* h, const NfbRays* rays, const int32_t* frame_index, const NfbSampling* sm,
                                    const NfbNoise* noise, const NfbOutputs* out, void* stream) {
  if (!frame_index) return NFB_ERR_INVALID;
  return render_impl(h, rays, sm, noise, out, nullptr, stream, true, frame_index);
}

int nfb_render_forward(NfbHandle* h, const NfbRays* rays, const NfbSampling* sm, const NfbNoise* noise, const NfbOutputs* out,
                       const NfbDebug* dbg, void* stream) {
  return render_impl(h, rays, sm, noise, out, dbg, stream, false);
}

int nfb_render_forward_train(NfbHandle* h, const NfbRays* rays, const NfbSampling* sm, const NfbNoise* noise,
                             const NfbOutputs* out, void* stream) {
  return render_impl(h, rays, sm, noise, out, nullptr, stream, true);
}

int nfb_render_backward(NfbHandle* h, const NfbOutGrads* og, const float* const params_coarse[26],
                        const float* const params_fine[26], float* const grads_coarse[26], float* const grads_fine[26],
                        float* grad_latent, void* stream) {
  if (!grads_coarse) return NFB_ERR_INVALID;  // input-only mode is nfb_render_backward_ex's
  return nfb_render_backward_ex(h, og, params_coarse, params_fine, grads_coarse, grads_fine, grad_latent, nullptr, stream);
}

// The backward of both kinds of training forward.  frames: a multi-frame backward (grad_latent / in_grads->expression unused;
// the per-frame gradients go to frame_latent / frame_expr, either may be null).
static int backward_impl(NfbHandle* h, const NfbOutGrads* og, const float* const params_coarse[26], const float* const params_fine[26],
                         float* const grads_coarse[26], float* const grads_fine[26], float* grad_latent, const NfbInputGrads* in_grads,
                         bool frames, float* frame_latent, float* frame_expr, void* stream) {
  if (!h || !og || !params_coarse) return NFB_ERR_INVALID;
  NfbHandle::Train& tr = h->tr;
  if (!tr.valid) return NFB_ERR_STATE;
  if (frames != tr.multi) {
    // a single-frame backward of a multi-frame forward has no one latent / expression to differentiate: refuse rather than sum
    if (!frames && (grad_latent || (in_grads && in_grads->expression))) return NFB_ERR_STATE;
    if (frames) return NFB_ERR_STATE;
  }
  if (frames && in_grads && in_grads->expression) return NFB_ERR_INVALID;  // per-frame expression gradients: frame_expr
  const bool frame_grads = tr.multi && (frame_latent || frame_expr || grads_coarse);
  const bool fine = tr.geom.passes() == 2;
  const bool input_only = !grads_coarse && !grads_fine;
  if (input_only && !in_grads && !(frames && (frame_latent || frame_expr))) return NFB_ERR_INVALID;
  if (!input_only && !grads_coarse) return NFB_ERR_INVALID;
  if (fine && (!params_fine || (!input_only && !grads_fine))) return NFB_ERR_INVALID;
  for (int i = 0; i < 26; ++i) {
    if (!params_coarse[i] || (fine && !params_fine[i])) return NFB_ERR_INVALID;
    if (!input_only && i != 22 && i != 23 && (!grads_coarse[i] || (fine && !grads_fine[i]))) return NFB_ERR_INVALID;
  }
  NfbInputGrads ig;
  std::memset(&ig, 0, sizeof(ig));
  if (in_grads) ig = *in_grads;
  if ((ig.dir_z && !tr.has_dir_z) || (ig.background && !tr.has_bg)) return NFB_ERR_INVALID;
  const bool ray_grads = ig.ray_origins || ig.ray_directions || ig.dir_z;
  if (ray_grads && !tr.has_rays) return NFB_ERR_UNSUPPORTED;
  const bool per_ray = ray_grads || ig.background;
  NFB_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* const acc[2] = {tr.acc[0].get(), tr.acc[1].get()};
  NFB_CUDA(cudaMemsetAsync(acc[0], 0, nfb::kAccFloats * sizeof(float), st));
  NFB_CUDA(cudaMemsetAsync(acc[1], 0, nfb::kAccFloats * sizeof(float), st));
  if (frame_grads) NFB_CUDA(cudaMemsetAsync(tr.fsum.get(), 0, (size_t)tr.n_frames * 2 * nfb::kFrameRows * sizeof(float), st));
  tr.per_ray_formed = tr.rows_formed = tr.frame_sums_formed = tr.bwd_formed = false;
  tr.dw_parts[0] = tr.dw_parts[1] = tr.dw_stride = 0;
  tr.dw_pe_only = false;

  // compositing backward -> dX chain -> weight-gradient GEMMs -> fixed-order reduction for the g.n_rays rays from `begin` on,
  // whose training state the buffers hold; the FP32 accumulators tr.acc add up over chunks in chunk order (each chunk has its
  // own power-of-two loss scale, divided out again before the accumulation)
  auto backward_rays = [&](int begin, const nfb::TileGeom& g) -> int {
    const size_t n = (size_t)g.n_rays, tiles = g.tiles();
    float* const scal = tr.scal.get();
    NFB_CUDA(cudaMemsetAsync(tr.draw.get(), 0, tiles * 512 * sizeof(float), st));
    NFB_CUDA(cudaMemsetAsync(scal, 0, 4 * sizeof(float), st));
    nfb::CompBwdParams q;
    std::memset(&q, 0, sizeof(q));
    nfb::ChainParams c;
    nfb::DwParams d = {};
    nfb::InGradRowParams r = {};
    nfb::InGradRayParams a = {};
    q.geom = c.geom = d.geom = r.geom = a.geom = g;
    q.has_bg = tr.has_bg; q.white_bkgd = tr.white_bkgd;
    q.z_c = tr.z_c.get(); q.raw_c = tr.raw_c.get(); q.z_f = tr.z_f.get(); q.raw_f = tr.raw_f.get(); q.dnorm = tr.dnorm.get();
    auto off3 = [&](const float* p) { return p ? p + 3 * (size_t)begin : nullptr; };
    auto off1 = [&](const float* p) { return p ? p + (size_t)begin : nullptr; };
    q.g_rgb[0] = off3(og->rgb_coarse); q.g_disp[0] = off1(og->disp_coarse); q.g_acc[0] = off1(og->acc_coarse);
    q.g_rgb[1] = off3(og->rgb_fine); q.g_disp[1] = off1(og->disp_fine); q.g_acc[1] = off1(og->acc_fine); q.g_wlast = off1(og->w_last);
    q.draw = tr.draw.get(); q.bsum = tr.bsum.get();
    q.absmax = reinterpret_cast<unsigned int*>(scal + 2);
    if (per_ray) {
      NFB_CUDA(tr.ray_dn.reserve(2 * n));
      NFB_CUDA(tr.ray_bg.reserve(6 * n));
      if (ray_grads) NFB_CUDA(tr.rows.reserve(tiles * 512));
      q.ray_dn = tr.ray_dn.get(); q.ray_bg = tr.ray_bg.get();
    }
    NFB_CUDA(nfb::launch_composite_bwd(q, scal, st, &h->launches));

    c.rec = tr.rec.get(); c.draw = tr.draw.get(); c.scal = scal;
    c.wstream[0] = h->net[0].stream_bwd.get();
    c.wstream[1] = h->net[fine ? 1 : 0].stream_bwd.get();
    c.wstream_lo[0] = h->net[0].stream_bwd_lo.get();
    c.wstream_lo[1] = h->net[fine ? 1 : 0].stream_bwd_lo.get();
    NFB_CUDA(nfb::launch_chain(c, h->num_sms, st, &h->launches, tr.hilo));
    // input-only: the PE jobs only serve d latent / d expression (a multi-frame backward forms those from the per-frame sums)
    const bool dw = !input_only || (!tr.multi && (grad_latent || ig.expression));
    if (dw) {
      d.rec = tr.rec.get(); d.ws = tr.dw_ws.get(); d.scal = scal;
      NFB_CUDA(nfb::launch_dw(d, h->num_sms, st, &h->launches, input_only, tr.hilo));  // both networks in one launch
      tr.dw_parts[0] = d.parts[0]; tr.dw_parts[1] = d.parts[1]; tr.dw_stride = d.ws_stride;
      tr.dw_pe_only = input_only;
    }
    if (frame_grads) {
      nfb::FrameSumParams fs = {};
      fs.rec = tr.rec.get(); fs.geom = g; fs.scal = scal; fs.frame = tr.frame.get(); fs.n_frames = tr.n_frames;
      fs.raysum = tr.raysum.get(); fs.fsum = tr.fsum.get();
      NFB_CUDA(nfb::launch_frame_sums(fs, st, &h->launches, tr.hilo));
    }
    NFB_CUDA(nfb::launch_grad_reduce(dw ? &d : nullptr, input_only, tr.bsum.get(), g.n_rays, g.passes(), acc, h->num_sms, st,
                                     &h->launches));
    if (per_ray) {
      r.rec = tr.rec.get();
      r.z_c = tr.z_c.get(); r.z_f = tr.z_f.get(); r.ray = tr.ray.get(); r.scal = scal;
      const float* const* pf = fine ? params_fine : params_coarse;
      r.w0[0] = params_coarse[0]; r.w3[0] = params_coarse[6]; r.wd0[0] = params_coarse[16];
      r.w0[1] = pf[0]; r.w3[1] = pf[6]; r.wd0[1] = pf[16];
      r.out = tr.rows.get();
      a.has_dir_z = tr.has_dir_z;
      a.z_c = tr.z_c.get(); a.z_f = tr.z_f.get(); a.ray = tr.ray.get(); a.dnorm = tr.dnorm.get();
      a.ray_dn = tr.ray_dn.get(); a.ray_bg = tr.ray_bg.get();
      auto at = [&](float* p, int w) { return p ? p + (size_t)w * begin : nullptr; };
      a.g_o = at(ig.ray_origins, 3); a.g_d = at(ig.ray_directions, 3); a.g_dir_z = at(ig.dir_z, 1); a.g_bg = at(ig.background, 3);
      NFB_CUDA(nfb::launch_input_grads(r, a, h->num_sms, st, &h->launches, tr.hilo));
    }
    return NFB_OK;
  };

  if (!tr.chunked) {
    int rc = backward_rays(0, tr.geom);
    if (rc) return rc;
    tr.per_ray_formed = per_ray;
    tr.rows_formed = ray_grads;
    tr.frame_sums_formed = frame_grads;
    tr.bwd_formed = true;
  } else {
    const int n_rays = tr.geom.n_rays;
    for (int begin = 0; begin < n_rays; begin += tr.chunk_rays) {
      const nfb::TileGeom g = tr.geom.chunk(n_rays - begin < tr.chunk_rays ? n_rays - begin : tr.chunk_rays);
      int rc = ensure_train_buffers(tr, g, h->num_sms);
      if (rc) return rc;
      const size_t cn = (size_t)tr.chunk_rays;
      NFB_CUDA(tr.scratch_out.reserve(11 * cn));
      // the training forward of this chunk: the saved launch with every per-ray pointer advanced to `begin`
      nfb::RenderParams p = tr.full;
      const size_t b = (size_t)begin;
      p.o += 3 * b; p.d += 3 * b; p.geom = g;
      if (p.dir_z) p.dir_z += b;
      if (p.bg) p.bg += 3 * b;
      if (p.t_rand) p.t_rand += b * g.nc;
      if (p.noise_c) p.noise_c += b * g.nc;
      if (p.u_rand) p.u_rand += b * g.nf;
      if (p.noise_f) p.noise_f += b * g.samples(1);
      if (p.frame) p.frame += b;
      float* so = tr.scratch_out.get();
      p.rgb_c = so; p.disp_c = so + 3 * cn; p.acc_c = so + 4 * cn; p.rgb_f = so + 5 * cn; p.disp_f = so + 8 * cn; p.acc_f = so + 9 * cn;
      p.w_last = so + 10 * cn;
      set_save_slots(p, tr);
      NFB_CUDA(nfb::launch_render(p, tr.precision, h->num_sms, st, &h->launches));
      rc = backward_rays(begin, g);
      if (rc) return rc;
    }
  }
  if (tr.multi) {  // no single latent / expression: the conditioning columns and the per-frame gradients come from the per-frame sums
    // finalize writes db (x) 0 into the conditioning columns (tr.cond is zeroed by a multi-frame forward); frames_grad_kernel,
    // next on the stream, overwrites them with sum_f db_f (x) c_f
    if (!input_only)
      NFB_CUDA(nfb::launch_finalize_all(params_coarse, grads_coarse, acc[0], fine ? params_fine : nullptr, fine ? grads_fine : nullptr,
                                        acc[1], tr.cond.get(), nullptr, st, &h->launches));
    if (frame_grads)
      NFB_CUDA(nfb::launch_frames_grad(params_coarse, input_only ? nullptr : grads_coarse, fine ? params_fine : nullptr,
                                       (fine && !input_only) ? grads_fine : nullptr, tr.fsum.get(), tr.fcond.get(), tr.n_frames,
                                       frame_latent, frame_expr, st, &h->launches));
    return NFB_OK;
  }
  NFB_CUDA(nfb::launch_finalize_all(params_coarse, input_only ? nullptr : grads_coarse, acc[0], fine ? params_fine : nullptr,
                                    (fine && !input_only) ? grads_fine : nullptr, acc[1], tr.cond.get(), grad_latent, st, &h->launches,
                                    ig.expression));
  return NFB_OK;
}

int nfb_render_backward_ex(NfbHandle* h, const NfbOutGrads* og, const float* const params_coarse[26],
                           const float* const params_fine[26], float* const grads_coarse[26], float* const grads_fine[26],
                           float* grad_latent, const NfbInputGrads* in_grads, void* stream) {
  return backward_impl(h, og, params_coarse, params_fine, grads_coarse, grads_fine, grad_latent, in_grads, false, nullptr, nullptr, stream);
}

int nfb_render_backward_frames(NfbHandle* h, const NfbOutGrads* out_grads, const float* const params_coarse[26],
                               const float* const params_fine[26], float* const grads_coarse[26], float* const grads_fine[26],
                               float* grad_latents, float* grad_expressions, const NfbInputGrads* in_grads, void* stream) {
  return backward_impl(h, out_grads, params_coarse, params_fine, grads_coarse, grads_fine, nullptr, in_grads, true, grad_latents,
                       grad_expressions, stream);
}

int nfb_train_debug(NfbHandle* h, NfbTrainDebug* out) {
  if (!h || !out) return NFB_ERR_INVALID;
  if (!h->tr.valid || h->tr.chunked) return NFB_ERR_STATE;  // chunked: the buffers only ever hold one chunk
  const NfbHandle::Train& tr = h->tr;
  out->records = tr.rec.get(); out->n_tiles = (long long)tr.geom.tiles(); out->record_bytes = (int32_t)nfb::rec_stride(tr.hilo);
  out->d_raw = tr.draw.get(); out->acc_coarse = tr.acc[0].get(); out->acc_fine = tr.acc[1].get(); out->acc_floats = nfb::kAccFloats;
  out->scale = tr.scal.get(); out->z_coarse = tr.z_c.get(); out->raw_coarse = tr.raw_c.get(); out->z_fine = tr.z_f.get();
  out->raw_fine = tr.raw_f.get();
  out->tiles_coarse = tr.geom.tiles_c; out->tiles_fine = tr.geom.tiles_f; out->rays_per_unit = tr.geom.rays_per_unit;
  out->rays = tr.ray.get(); out->dnorm = tr.dnorm.get();
  out->rows = tr.rows_formed ? tr.rows.get() : nullptr;
  out->ray_dn = tr.per_ray_formed ? tr.ray_dn.get() : nullptr;
  out->ray_bg = (tr.per_ray_formed && tr.has_bg) ? tr.ray_bg.get() : nullptr;
  const bool multi = tr.multi;
  out->n_frames = multi ? tr.n_frames : 0;
  out->frame = multi ? tr.frame.get() : nullptr;
  out->frame_table[0] = multi ? tr.ftab[0].get() : nullptr;
  out->frame_table[1] = (multi && tr.geom.passes() == 2) ? tr.ftab[1].get() : nullptr;
  out->frame_cond = multi ? tr.fcond.get() : nullptr;
  out->ray_sums = (multi && tr.frame_sums_formed) ? tr.raysum.get() : nullptr;
  out->frame_sums = (multi && tr.frame_sums_formed) ? tr.fsum.get() : nullptr;
  const bool dw = tr.bwd_formed && tr.dw_parts[0] + tr.dw_parts[1] > 0;
  out->dw_partials = dw ? tr.dw_ws.get() : nullptr;
  out->dw_slot_floats = dw ? tr.dw_stride : 0;
  out->dw_parts[0] = dw ? tr.dw_parts[0] : 0;
  out->dw_parts[1] = dw ? tr.dw_parts[1] : 0;
  out->dw_pe_only = (dw && tr.dw_pe_only) ? 1 : 0;
  out->ray_bias_sums = tr.bwd_formed ? tr.bsum.get() : nullptr;
  return NFB_OK;
}

int nfb_debug_weights(NfbHandle* h, int net, NfbWeightDebug* out) {
  if (!h || !out || (net != NFB_NET_COARSE && net != NFB_NET_FINE)) return NFB_ERR_INVALID;
  const nfb::NetBuffers& nb = h->net[net];
  if (!nb.loaded) return NFB_ERR_STATE;
  out->x1 = nb.stream_x1.get(); out->x3 = nb.stream_x3.get(); out->bwd = nb.stream_bwd.get();
  out->w6 = nb.w6.get(); out->b6 = nb.b6.get(); out->bias_static = nb.bias_static.get(); out->bias_frame = nb.bias_frame.get();
  out->w0c = nb.w0c.get(); out->w3c = nb.w3c.get(); out->wd0b_t = nb.wd0b_t.get();
  out->x1_bytes = nfb::kStreamBytesX1; out->x3_bytes = nfb::kStreamBytesX3; out->bwd_bytes = nfb::kBwdStreamBytes;
  out->bias_floats = nfb::kBiasFloats;
  out->bwd_lo = h->bwd_lo ? nb.stream_bwd_lo.get() : nullptr;
  out->bwd_lo_bytes = h->bwd_lo ? nfb::kBwdStreamBytes : 0;
  return NFB_OK;
}

int nfb_render_frame_host(NfbHandle* h, const float pose[12], const double intrinsics[4], int height, int width, int row_begin,
                          int rows, float near_, float far_, const float* expression_host, const float* latent_host,
                          const float* background_host, const NfbSampling* sm, float* out_host, void* stream) {
  if (!h || !pose || !intrinsics || !expression_host || !latent_host || !sm || !out_host) return NFB_ERR_INVALID;
  if (height <= 0 || width <= 0 || rows <= 0 || row_begin < 0 || row_begin + rows > height) return NFB_ERR_INVALID;
  if (sm->perturb || sm->noise_std > 0.f) return NFB_ERR_UNSUPPORTED;  // host path is the deterministic renderer
  NFB_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t n = (size_t)rows * width;
  NFB_CUDA(h->d_out.reserve(11 * n));
  if (background_host) NFB_CUDA(h->d_bg.reserve(3 * n));
  NFB_CUDA(cudaMemcpyAsync(h->d_expr.get(), expression_host, nfb::kDimExpr * sizeof(float), cudaMemcpyHostToDevice, st));
  NFB_CUDA(cudaMemcpyAsync(h->d_latent.get(), latent_host, nfb::kDimLatent * sizeof(float), cudaMemcpyHostToDevice, st));
  if (background_host) NFB_CUDA(cudaMemcpyAsync(h->d_bg.get(), background_host, 3 * n * sizeof(float), cudaMemcpyHostToDevice, st));
  int rc = nfb_set_frame(h, h->d_expr.get(), h->d_latent.get(), stream);
  if (rc) return rc;
  NfbRays r;
  std::memset(&r, 0, sizeof(r));
  r.n_rays = (int)n;
  for (int i = 0; i < 12; ++i) r.pose[i] = pose[i];
  for (int i = 0; i < 4; ++i) r.intrinsics[i] = intrinsics[i];
  r.height = height; r.width = width; r.row_begin = row_begin;
  r.near_ = near_; r.far_ = far_;
  r.background = background_host ? h->d_bg.get() : nullptr;
  NfbOutputs o;
  float* b = h->d_out.get();
  o.rgb_coarse = b; o.disp_coarse = b + 3 * n; o.acc_coarse = b + 4 * n;
  o.rgb_fine = b + 5 * n; o.disp_fine = b + 8 * n; o.acc_fine = b + 9 * n; o.w_last = b + 10 * n;
  rc = nfb_render_forward(h, &r, sm, nullptr, &o, nullptr, stream);
  if (rc) return rc;
  NFB_CUDA(cudaMemcpyAsync(out_host, h->d_out.get(), 11 * n * sizeof(float), cudaMemcpyDeviceToHost, st));
  NFB_CUDA(cudaStreamSynchronize(st));
  return NFB_OK;
}

int nfb_frame_products(NfbHandle* h, const float* rgb, const float* disparity, const float* w_last, const double intrinsics[4], int height,
                       int width, uint8_t* rgb_u8, uint8_t* normals_u8, uint8_t* disparity_u8, int flags, void* stream) {
  if (!h || !intrinsics || height < 2 || width < 2) return NFB_ERR_INVALID;
  if ((rgb_u8 && !rgb) || ((normals_u8 || disparity_u8) && !disparity)) return NFB_ERR_INVALID;
  if (normals_u8 && height != width) return NFB_ERR_UNSUPPORTED;  // the reference's expression only broadcasts for square frames
  NFB_CUDA(cudaSetDevice(h->device));
  NFB_CUDA(h->minmax.reserve(2));
  NFB_CUDA(nfb::launch_frame_products(rgb, disparity, w_last, intrinsics, height, width, rgb_u8, normals_u8, disparity_u8, h->minmax.get(),
                                      (flags & NFB_PRODUCTS_LIKE_TORCH_CPU) ? 1 : 0, static_cast<cudaStream_t>(stream), &h->launches));
  return NFB_OK;
}

int nfb_sample_rays(NfbHandle* h, const NfbRayMap* map, const double* draws, int size, int max_rounds, long long* indices, int32_t* state,
                    const NfbRayGather* g, void* stream) {
  if (!h || !map || !draws || !indices || !state || size < 1 || size > nfb::kSmpMax || max_rounds < 1) return NFB_ERR_INVALID;
  if (map->height < 1 || map->width < 1 || (long long)map->height * map->width < size) return NFB_ERR_INVALID;
  if (map->bbox[0] < 0 || map->bbox[1] > map->height || map->bbox[2] < 0 || map->bbox[3] > map->width) return NFB_ERR_INVALID;
  if (!(map->q_out > 0.0) || !(map->q_in > 0.0)) return NFB_ERR_INVALID;
  if (1 + 2 * (map->bbox[1] - map->bbox[0]) > nfb::smp::kMaxRuns) return NFB_ERR_UNSUPPORTED;
  NFB_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long N = (long long)map->height * map->width;
  NFB_CUDA(h->smp_runs.reserve(nfb::smp::kMaxRuns));
  NFB_CUDA(h->smp_segs.reserve(nfb::smp::kMaxSegs));
  bool fresh = false;  // a new first_pos starts all INT_MAX (SampleArgs::first_pos)
  NFB_CUDA(h->smp_first.reserve((size_t)N, &fresh));
  if (fresh) NFB_CUDA(nfb::launch_fill_int(h->smp_first.get(), N, 0x7FFFFFFF, st, &h->launches));
  nfb::SampleArgs a;
  std::memset(&a, 0, sizeof(a));
  a.map.H = map->height; a.map.W = map->width;
  a.map.b0 = map->bbox[0]; a.map.b1 = map->bbox[1]; a.map.b2 = map->bbox[2]; a.map.b3 = map->bbox[3];
  a.map.q_out = map->q_out; a.map.q_in = map->q_in;
  a.draws = draws; a.size = size; a.max_rounds = max_rounds; a.found = indices; a.state = state;
  a.runs = h->smp_runs.get(); a.segs = h->smp_segs.get(); a.first_pos = h->smp_first.get();
  if (g) {
    if ((g->target && !g->image) || (g->background_out && !g->background) || (g->ray_origins && !g->ray_directions)) return NFB_ERR_INVALID;
    for (int i = 0; i < 12; ++i) a.pose[i] = g->pose[i];
    a.fx = static_cast<float>(g->intrinsics[0]);
    a.fy = static_cast<float>(g->intrinsics[1]);
    a.wcx = static_cast<float>(static_cast<double>(map->width) * g->intrinsics[2]);
    a.hcy = static_cast<float>(static_cast<double>(map->height) * g->intrinsics[3]);
    a.image = g->image; a.background = g->background; a.ray_o = g->ray_origins; a.ray_d = g->ray_directions;
    a.target = g->target; a.bg_out = g->background_out; a.pixel_rc = g->pixel_rc;
  }
  NFB_CUDA(nfb::launch_sample_rays(a, st, &h->launches));
  return NFB_OK;
}

int nfb_sample_rays_images(NfbHandle* h, const NfbTrainImages* d, const int32_t* image_index, int K, int n, const double* draws,
                           int max_rounds, const float* latent_table, const NfbImageBatch* out, void* stream) {
  if (!h || !d || !image_index || !draws || !latent_table || !out || K < 1 || n < 1 || n > nfb::kSmpMax || max_rounds < 1)
    return NFB_ERR_INVALID;
  if (K > NFB_MAX_STEP_IMAGES) return NFB_ERR_UNSUPPORTED;
  if (!d->maps || !d->poses || !d->expressions || !d->images || d->n_images < 1 || d->height < 1 || d->width < 1 ||
      (long long)d->height * d->width < n)
    return NFB_ERR_INVALID;
  if (out->background && !d->background) return NFB_ERR_INVALID;
  NFB_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t hw = (size_t)d->height * d->width;
  NFB_CUDA(h->smpi_runs.reserve((size_t)K * nfb::smp::kMaxRuns));
  NFB_CUDA(h->smpi_segs.reserve((size_t)K * nfb::smp::kMaxSegs));
  NFB_CUDA(h->smpi_found.reserve((size_t)K * n));
  bool fresh = false;  // a new first-occurrence table starts all INT_MAX (the kernel leaves it so)
  NFB_CUDA(h->smpi_first.reserve((size_t)K * hw, &fresh));
  if (fresh) NFB_CUDA(nfb::launch_fill_int(h->smpi_first.get(), (long long)(K * hw), 0x7FFFFFFF, st, &h->launches));
  nfb::ImageSampleArgs a = {};
  a.maps = reinterpret_cast<const nfb::RayMapRec*>(d->maps);
  a.poses = d->poses; a.expr_table = d->expressions; a.images = d->images; a.background = d->background;
  a.n_images = d->n_images; a.H = d->height; a.W = d->width;
  a.fx = static_cast<float>(d->intrinsics[0]);
  a.fy = static_cast<float>(d->intrinsics[1]);
  a.wcx = static_cast<float>(static_cast<double>(d->width) * d->intrinsics[2]);
  a.hcy = static_cast<float>(static_cast<double>(d->height) * d->intrinsics[3]);
  a.image_index = image_index; a.K = K; a.size = n; a.max_rounds = max_rounds; a.draws = draws; a.latent_table = latent_table;
  a.runs = h->smpi_runs.get(); a.segs = h->smpi_segs.get(); a.first_pos = h->smpi_first.get(); a.found = h->smpi_found.get();
  a.ray_o = out->ray_origins; a.ray_d = out->ray_directions; a.target = out->target; a.bg_out = out->background;
  a.pixel_rc = out->pixel_rc; a.indices = out->indices; a.frame = out->frame_index;
  a.expr_out = out->expressions; a.latent_out = out->latents; a.state = out->state; a.shortfall = out->shortfall;
  NFB_CUDA(nfb::launch_sample_images(a, st, &h->launches));
  return NFB_OK;
}

int nfb_latent_rows_grad(NfbHandle* h, const float* grad_latents, const int32_t* image_index, int K, const float* latent_table, int n_rows,
                         float* table_grads, float reg_weight, void* stream) {
  if (!h || !grad_latents || !image_index || !latent_table || !table_grads || K < 1 || n_rows < 1) return NFB_ERR_INVALID;
  if (K > NFB_MAX_STEP_IMAGES) return NFB_ERR_UNSUPPORTED;
  NFB_CUDA(cudaSetDevice(h->device));
  NFB_CUDA(nfb::launch_latent_rows(grad_latents, image_index, K, latent_table, n_rows, table_grads, reg_weight,
                                   static_cast<cudaStream_t>(stream), &h->launches));
  return NFB_OK;
}

int nfb_fit_rows_grad(NfbHandle* h, const NfbTrainImages* d, const int32_t* image_index, int K, int n, const int32_t* pixel_rc,
                      const float* grad_ray_origins, const float* grad_ray_directions, float* pose_grads, const float* grad_expressions,
                      float* expression_grads, void* stream) {
  if (!h || !d || !image_index || K < 1 || n < 1 || n > nfb::kSmpMax) return NFB_ERR_INVALID;
  if (K > NFB_MAX_STEP_IMAGES) return NFB_ERR_UNSUPPORTED;
  if (d->n_images < 1 || d->height < 1 || d->width < 1) return NFB_ERR_INVALID;
  if (pose_grads && (!pixel_rc || (!grad_ray_origins && !grad_ray_directions))) return NFB_ERR_INVALID;
  if (!expression_grads != !grad_expressions) return NFB_ERR_INVALID;
  if (!pose_grads && !expression_grads) return NFB_OK;  // nothing asked for: nothing written, no launch
  NFB_CUDA(cudaSetDevice(h->device));
  NFB_CUDA(h->fit_slots.reserve((size_t)NFB_MAX_STEP_IMAGES * 12));  // once, at its largest: a graph's address stays valid
  const float fx = static_cast<float>(d->intrinsics[0]), fy = static_cast<float>(d->intrinsics[1]);
  const float wcx = static_cast<float>(static_cast<double>(d->width) * d->intrinsics[2]);  // as nfb_sample_rays_images rounds them
  const float hcy = static_cast<float>(static_cast<double>(d->height) * d->intrinsics[3]);
  NFB_CUDA(nfb::launch_fit_rows(image_index, K, n, d->n_images, pixel_rc, grad_ray_origins, grad_ray_directions, fx, fy, wcx, hcy,
                                h->fit_slots.get(), pose_grads, grad_expressions, expression_grads, static_cast<cudaStream_t>(stream),
                                &h->launches));
  return NFB_OK;
}

int nfb_background_rows_grad(NfbHandle* h, const int32_t* pixel_rc, int n_rays, int height, int width, const float* grad_bg_render,
                             const float* grad_bg_loss, float* table_grads, void* stream) {
  if (!h || !pixel_rc || !grad_bg_render || !table_grads || n_rays < 0 || height < 1 || width < 1) return NFB_ERR_INVALID;
  if ((long long)height * width > 0x7FFFFFFFLL) return NFB_ERR_INVALID;  // the kernel keys pixels by an int index
  if (n_rays == 0) return NFB_OK;  // nothing to add: no launch
  NFB_CUDA(cudaSetDevice(h->device));
  NFB_CUDA(nfb::launch_background_rows(pixel_rc, n_rays, height, width, grad_bg_render, grad_bg_loss, table_grads,
                                       static_cast<cudaStream_t>(stream), &h->launches));
  return NFB_OK;
}

int nfb_loss_background_grad(NfbHandle* h, const float* bg_rays, const float* target, const float* w_last, int n_rays, long long n_total,
                             float weight, float* grad_bg_rays, float* grad_w_last, float* loss, void* stream) {
  if (!h || !bg_rays || !target || !w_last || !grad_bg_rays || !grad_w_last || !loss || n_rays < 0 || n_total < n_rays || n_total <= 0)
    return NFB_ERR_INVALID;
  if (n_rays == 0) return NFB_OK;  // an empty shard adds nothing: no launch
  NFB_CUDA(cudaSetDevice(h->device));
  NFB_CUDA(nfb::launch_loss_background(bg_rays, target, w_last, n_rays, n_total, weight, grad_bg_rays, grad_w_last, loss,
                                       static_cast<cudaStream_t>(stream), &h->launches));
  return NFB_OK;
}

int nfb_host_map_cdf(const NfbRayMap* map, const long long* zeroed_sorted, int n_zero, const long long* ks, int n, double* out) {
  if (!map || !ks || !out || n < 0 || n_zero < 0 || (n_zero && !zeroed_sorted)) return NFB_ERR_INVALID;
  nfb::smp::Map m;
  m.H = map->height; m.W = map->width; m.b0 = map->bbox[0]; m.b1 = map->bbox[1]; m.b2 = map->bbox[2]; m.b3 = map->bbox[3];
  m.q_out = map->q_out; m.q_in = map->q_in;
  if (nfb::smp::num_runs(m) > nfb::smp::kMaxRuns) return NFB_ERR_UNSUPPORTED;
  std::vector<nfb::smp::Run> runs(nfb::smp::kMaxRuns);
  std::vector<nfb::smp::Seg> segs(nfb::smp::kMaxSegs);
  int nr = 0, ns = 0;
  const double total = nfb::smp::build_tables(m, zeroed_sorted, n_zero, runs.data(), nr, segs.data(), ns);
  if (ns > nfb::smp::kMaxSegs) return NFB_ERR_UNSUPPORTED;
  const long long N = (long long)m.H * m.W;
  for (int i = 0; i < n; ++i) {
    if (ks[i] < -1 || ks[i] >= N) return NFB_ERR_INVALID;
    out[i] = ks[i] < 0 ? total : nfb::smp::cdf_at(ks[i], runs.data(), nr, segs.data(), zeroed_sorted, n_zero);
  }
  return NFB_OK;
}

// Host copy of the per-tile unit program a kernel follows through a weight stream (nfb_layout.h: make_prog).
static int debug_prog(int stream, int index, uint32_t* out) {
  const int n = nfb::prog_units(stream);
  if (index < 0) return n;
  if (index >= n) return -1;
  const nfb::ProgEntry e = nfb::make_prog(stream).e[index];
  out[0] = e.x; out[1] = e.y; out[2] = e.z; out[3] = e.w;
  return 4;
}

int nfb_debug_schedule(int which, int index, uint32_t* out, int out_words) {
  if (index >= 0 && (!out || out_words < 10)) return -1;
  switch (which) {
    case 0: return debug_prog(nfb::kFwdStream, index, out);
    case 2: return debug_prog(nfb::kBwdStream, index, out);
    case 3: return nfb::debug_jobs_dw(index, out);
    case 4: return index < 0 ? 1 : nfb::debug_dw_split(out);  // in/out: {num_sms, tiles 0, tiles 1} -> {parts0, parts1, groups}
    default: return -1;
  }
}

int nfb_buffer_epoch(NfbHandle* h, long long* out) {
  if (!h || !out) return NFB_ERR_INVALID;
  *out = h->frees + h->tr.frees;
  return NFB_OK;
}

int nfb_launch_count(NfbHandle* h, long long* out) {
  if (!h || !out) return NFB_ERR_INVALID;
  *out = h->launches;
  return NFB_OK;
}

}  // extern "C"
