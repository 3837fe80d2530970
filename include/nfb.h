/* nfb.h — C ABI of the H100-native NeRFace render path ("nfb" = NeRFace fused render path).
 *
 * This is the drop-in boundary for ONE hot path of gafniguy/4D-Facial-Avatars: the per-ray render
 * loop reached through nerface_code/nerf-pytorch/nerf/train_utils.py (run_one_iter_of_nerf :165-290,
 * predict_and_render_radiance :36-162, run_network :9-33), nerf_helpers.py (get_ray_bundle :68-123,
 * positional_encoding :195-239, sample_pdf_2 :344-387, cumprod_exclusive :44-65),
 * volume_rendering_utils.py (volume_render_radiance_field :7-75) and models.py
 * (ConditionalBlendshapePaperNeRFModel :189-261).  The reference has no FFI (it is pure PyTorch);
 * the Python package 4d-facial-avatars_b200/nerf binds these entry points with ctypes and keeps the
 * reference's call surface.  See INTEGRATION.md.
 *
 * Conventions: plain pointers and sizes, no torch types.  Every entry returns an int status
 * (0 = NFB_OK) and never throws; nfb_strerror() maps it to text.  All device pointers are FP32,
 * row-major, 16-byte aligned, on the device the handle was created for.  Calls are asynchronous on
 * the given cudaStream_t (passed as void*) unless stated otherwise; no entry synchronises the device
 * except nfb_render_frame_host.
 */
#ifndef NFB_H_
#define NFB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NFB_VERSION 131
/* Defined when the backward and the loss repeat bit for bit (no floating-point atomics; see nfb_render_backward).  The
 * version number stayed 130 for this addition, so test this macro rather than the version. */
#define NFB_REPRODUCIBLE_BACKWARD 1
/* Defined when the multi-frame entries exist (nfb_set_frames, nfb_render_forward_frames[_train], nfb_render_backward_frames): one
 * call renders and differentiates rays of up to NFB_MAX_FRAMES frames, each ray conditioned on its own frame.  Test this macro. */
#define NFB_MULTI_FRAME 1
#define NFB_MAX_FRAMES 1024
/* Defined when the training-step entries over several images exist (nfb_sample_rays_images, nfb_latent_rows_grad): one step
 * draws its rays from up to NFB_MAX_STEP_IMAGES training images, reading every per-step input from device memory.  Test this
 * macro. */
#define NFB_TRAIN_IMAGES 1
#define NFB_MAX_STEP_IMAGES 64
/* Defined when precision NFB_PREC_EXACT_GRAD exists (hi + lo gradients, see below), with NfbTrainDebug.record_bytes reporting the
 * record stride and NfbWeightDebug's bwd_lo members.  The version number stayed 131 for this addition: test this macro. */
#define NFB_EXACT_GRAD 1
/* Defined when nfb_fit_rows_grad exists: the pose and expression rows of a fitting step over several images (a frozen avatar's
 * per-frame camera pose, expression and latent fitted to photos).  The version number stayed 131 for this addition: test this
 * macro. */
#define NFB_FIT_STEP 1
/* Defined when nfb_background_rows_grad and nfb_loss_background_grad exist: a training step over several images that learns the
 * background image (the reference's train_background / supervised_train_background).  The version number stayed 131 for this
 * addition: test this macro. */
#define NFB_TRAIN_BACKGROUND 1

typedef struct NfbHandle NfbHandle;

enum {
  NFB_OK = 0,
  NFB_ERR_INVALID = 1,     /* bad argument (null pointer, negative size, ...) */
  NFB_ERR_UNSUPPORTED = 2, /* configuration outside what the kernel implements */
  NFB_ERR_CUDA = 3,        /* a CUDA runtime call failed; see nfb_last_cuda_error() */
  NFB_ERR_STATE = 4,       /* call order violated (weights or frame not set) */
  NFB_ERR_ARCH = 5         /* device is not sm_90 */
};

/* Which of the two networks (models.coarse / models.fine in the reference YAML). */
enum { NFB_NET_COARSE = 0, NFB_NET_FINE = 1 };

/* Arithmetic used by the tensor-core MLP.
 *   NFB_PREC_FAST  : FP16 operands (round-to-nearest), FP32 accumulate, one wgmma pass.
 *   NFB_PREC_EXACT : every operand split x = hi + lo in FP16; hi*hi + hi*lo + lo*hi, FP32
 *                    accumulate (3 wgmma passes, ~2^-21 relative operand error).  The backward carries FP16 operands (one
 *                    value per activation and gradient): exact-mode gradients are FP16-grade.
 *   NFB_PREC_EXACT_GRAD : exact mode's forward, bit for bit (outputs, and the first MiB of every training record), and a backward
 *                    on hi + lo operands end to end: the training records hold a lo half of every activation image, the dX chain
 *                    multiplies hi + lo gradients by the hi + lo transposed weights and the weight-gradient GEMMs hi + lo images,
 *                    each as hi*hi + hi*lo + lo*hi (operand error ~2^-22 relative, below FP32 accumulation; gradients still carry
 *                    one power-of-two loss scale).  Non-finite values as in the other modes: an activation recorded as inf or NaN
 *                    (hi) gives non-finite gradients, as does a scaled gradient beyond the FP16 range (hi inf, lo non-finite).
 *                    Cost: 2 MiB of records per 128-row tile instead of 1 (the memory budget of nfb_render_forward_train counts
 *                    it); measured on an H100 80GB HBM3 (700 W) at 2048 rays, 64c+64f: 2.2x exact mode's dX-chain and
 *                    weight-gradient time, 1.87x its training step (DESIGN.md §6c); one extra launch per weight load / re-pack
 *                    once the handle has run an exact-grad training forward (it writes the lo half of the backward weight stream).
 *                    Evaluation renders run exact mode's kernel.  The backward entries follow the mode of the training forward.
 * Any other value is NFB_ERR_INVALID. */
enum { NFB_PREC_FAST = 0, NFB_PREC_EXACT = 1, NFB_PREC_EXACT_GRAD = 2 };

/* Encoder / conditioning dimensions; mirrors the constructor arguments of
 * ConditionalBlendshapePaperNeRFModel (models.py:193-206).  Only the shipped paper configuration
 * (10, 4, include_input_xyz=1, include_input_dir=0, 76, 32) is implemented. */
typedef struct {
  int32_t num_encoding_fn_xyz;
  int32_t num_encoding_fn_dir;
  int32_t include_input_xyz;
  int32_t include_input_dir;
  int32_t dim_expression;
  int32_t dim_latent;
} NfbModelDims;

/* Rays of one call.  Either explicit rays (o and d non-null; what run_one_iter_of_nerf receives,
 * train_utils.py:171-172) or in-kernel generation from a camera (o == d == NULL; replaces
 * get_ray_bundle, nerf_helpers.py:68-123, for image rows [row_begin, row_begin + n_rays / width)). */
typedef struct {
  const float* o;          /* [n_rays,3] device, or NULL */
  const float* d;          /* [n_rays,3] device, unnormalised, or NULL */
  int32_t n_rays;
  float pose[12];          /* row-major 3x4 camera-to-world (used when o == NULL) */
  double intrinsics[4];    /* fx, fy, cx, cy with cx, cy relative in [0,1]; FP64 like the reference's numpy
                              array (load_flame.py:114-118), rounded to FP32 where torch would */
  int32_t height, width, row_begin;
  float near_, far_;       /* options.dataset.near / far (train_utils.py:210-211) */
  const float* dir_z;      /* optional [n_rays]: overrides d_z as the first input of the direction
                              encoder (ray_directions_ablation path, train_utils.py:81-82); NULL = d_z */
  const float* background; /* optional [n_rays,3] background_prior (train_utils.py:95-96) or NULL */
} NfbRays;

/* options.nerf.<mode>.* (train_utils.py:56-69,108-122). */
typedef struct {
  int32_t num_coarse, num_fine;
  int32_t perturb;          /* stratified coarse samples; also makes the fine resampling stochastic */
  float noise_std;          /* radiance_field_noise_std */
  int32_t white_background;
  int32_t lindisp;          /* must be 0 (all shipped YAMLs) */
  int32_t precision;        /* NFB_PREC_* */
  const float* t_coarse;    /* optional device [num_coarse] = torch.linspace(0,1,num_coarse); NULL: computed */
  const float* u_fine;      /* optional device [num_fine]  = torch.linspace(0,1,num_fine);  NULL: computed */
} NfbSampling;

/* Explicit noise, in the reference's draw order per ray chunk (SURVEY.md §8c).  Required members:
 * t_rand and u when perturb != 0; sigma_noise_* when noise_std > 0.  All device pointers. */
typedef struct {
  const float* t_rand;        /* [n_rays, num_coarse] uniform [0,1) */
  const float* sigma_noise_c; /* [n_rays, num_coarse] standard normal */
  const float* u;             /* [n_rays, num_fine] uniform [0,1) */
  const float* sigma_noise_f; /* [n_rays, num_coarse+num_fine] standard normal */
} NfbNoise;

/* The 7-tuple of predict_and_render_radiance (train_utils.py:162).  Fine members may be NULL when
 * num_fine == 0; then w_last receives the coarse pass's last weight. */
typedef struct {
  float* rgb_coarse;  /* [n_rays,3] */
  float* disp_coarse; /* [n_rays] */
  float* acc_coarse;  /* [n_rays] */
  float* rgb_fine;    /* [n_rays,3] */
  float* disp_fine;   /* [n_rays] */
  float* acc_fine;    /* [n_rays] */
  float* w_last;      /* [n_rays] weights[:, -1] of the last pass */
} NfbOutputs;

/* Optional per-sample dumps (tests, and the tensors a backward pass needs).  Any member may be NULL. */
typedef struct {
  float* z_coarse;   /* [n_rays, num_coarse] */
  float* raw_coarse; /* [n_rays, num_coarse, 4] MLP output (rgb raw, sigma raw), before the bg overwrite */
  float* z_fine;     /* [n_rays, num_coarse+num_fine] sorted */
  float* raw_fine;   /* [n_rays, num_coarse+num_fine, 4] */
  /* Layer probe: post-activation FP32 values the epilogue of tensor-core step `act_step` (0..8, see
   * nfb_layout.h; -1 = the 64-lane positional encoding) produced for the first 128 coarse rows
   * (rays 0.., samples in order).  [128, 256] floats; columns beyond the step's width are untouched. */
  float* act_dump;
  int32_t act_step;
  /* Phase timers: 64 uint64 cycle counters (zeroed by the caller), accumulated over all CTAs by one observer
   * thread per warp role.  Slots: 0 ray setup, 1 per-ray direction term, 2 sampling+encoding (prologue),
   * 10+s wait for tensor-core step s, 20+s epilogue of step s, 3 end-of-pass barrier, 4 compositing,
   * 5 cdf, 6 inverse-cdf sampling, 7 sort; 41 producer waiting for a free ring slot; 45 MMA issuer waiting for
   * the A operand, 46 waiting for weights, 44 issuing. */
  unsigned long long* prof;
} NfbDebug;

int nfb_version(void);
const char* nfb_strerror(int status);
/* Text of the last CUDA error seen by this thread's calls (empty string if none). */
const char* nfb_last_cuda_error(void);

/* Create / destroy a renderer bound to one CUDA device.  Allocates the packed-weight streams,
 * per-frame constant buffers and per-CTA scratch (a few MB). */
int nfb_create(const NfbModelDims* dims, int device, NfbHandle** out);
int nfb_destroy(NfbHandle* h);

/* Load one network.  `params` holds 26 DEVICE pointers in the reference's state_dict order
 * (models.py:218-233): layers_xyz.{0..5}.{weight,bias}, fc_feat.{weight,bias}, fc_alpha.{weight,bias},
 * layers_dir.{0..3}.{weight,bias}, fc_rgb.{weight,bias} — weights row-major (out,in).  Folds fc_feat
 * into fc_alpha / layers_dir.0 (exact algebra, FP64), splits to FP16 hi/lo and writes the
 * shared-memory-image weight streams the kernel's bulk copies read.  layers_dir.3 is ignored, as in
 * the reference's forward (models.py:257). */
int nfb_load_weights(NfbHandle* h, int which, const float* const params[26], void* stream);

/* Per-frame conditioning: expression[76] (divided by 3 inside, models.py:241) and latent[32], both
 * DEVICE pointers.  Folds W0[:,63:171]·c and W3[:,63:171]·c into the layer-0 / layer-3 biases of both
 * loaded networks. */
int nfb_set_frame(NfbHandle* h, const float* expression, const float* latent, void* stream);

/* The hot path: coarse sampling -> encode -> coarse MLP -> composite -> inverse-CDF resample -> sort
 * -> encode -> fine MLP -> composite, one persistent sm_90a kernel launch.
 * Non-finite values: a NaN or inf in an input (ray, background, noise draw, parameter, expression) gives non-finite outputs
 * wherever FP32 torch would, never finite ones: the ReLUs keep NaN, and NaN fine samples sort last.  A hidden activation
 * beyond the FP16 range (65504 in fast mode; about 131008, hi + lo, in exact mode) becomes inf, never a clamped value.
 * Only the rays an input belongs to are affected. */
int nfb_render_forward(NfbHandle* h, const NfbRays* rays, const NfbSampling* sampling,
                       const NfbNoise* noise /* nullable */, const NfbOutputs* out,
                       const NfbDebug* dbg /* nullable */, void* stream);

/* ---- Training (replaces torch.autograd over the unfused graph, train_transformed_rays.py:389) ----
 * nfb_render_forward_train is nfb_render_forward that additionally keeps, in buffers owned by the handle, what the
 * backward needs: per-sample depths, colours and ReLU inputs of both passes, and per 128-row tile the FP16 activations
 * of every layer (about 1 MiB per tile; 2048 rays at 64+64 samples = 3 GiB).  nfb_render_backward on the same handle
 * consumes that state.  Between the two, nfb_set_frame and nfb_render_forward calls (e.g. a validation render of another
 * frame, with other sample counts) are allowed and do not change what is differentiated; re-loading weights
 * (nfb_load_weights, nfb_repack) is not.
 * Memory: when the records of the whole call would exceed the budget (environment NFB_TRAIN_MEM_MB, default 60 % of the free
 * device memory) — e.g. a full frame rendered with gradients enabled — the forward only renders (evaluation kernel) and the
 * backward re-runs the training forward chunk by chunk inside the budget: same gradients, one extra forward; the caller must
 * then keep the forward's input buffers alive until the backward, and explicit rays are required. */
int nfb_render_forward_train(NfbHandle* h, const NfbRays* rays, const NfbSampling* sampling,
                             const NfbNoise* noise /* nullable */, const NfbOutputs* out, void* stream);

/* dL/d(outputs) of the 7-tuple; any member may be NULL (= zero).  All device pointers, shapes as NfbOutputs. */
typedef struct {
  const float* rgb_coarse;
  const float* disp_coarse;
  const float* acc_coarse;
  const float* rgb_fine;
  const float* disp_fine;
  const float* acc_fine;
  const float* w_last;
} NfbOutGrads;

/* Backward of the last nfb_render_forward_train: compositing backward -> wgmma dX chain -> wgmma weight-gradient GEMMs
 * -> gradients in the reference's parameter layout.  `params_*` are the 26 FP32 parameter pointers given to
 * nfb_load_weights; `grads_*` receive dL/dparam with the same shapes (entries 22, 23 = layers_dir.3.*, unused by the
 * forward, models.py:257: may be NULL and are never written).  `grad_latent` [32] receives dL/d latent_code (NULL: skipped);
 * the sample depths carry no gradient (z_samples.detach(), train_utils.py:124).  Gradients are OVERWRITTEN, not accumulated.
 * The call may be repeated on one saved forward with other output gradients (each call starts from zeroed accumulators).
 * A non-finite output gradient gives non-finite parameter gradients, as autograd does; so does a loss-scaled FP16 gradient
 * that overflows inside the dX chain (it is not clamped), and so does a hidden activation beyond what the forward's FP16
 * records can hold (it is recorded as inf, not 65504).  Tile rows that hold no sample never contribute: their records are zero.
 * params_fine / grads_fine may be NULL when the forward had num_fine == 0.
 * Reproducibility: the path has no floating-point atomics; every sum over rays, tiles and CTAs runs in a fixed order.  Given the
 * same library build, device model (SM count), inputs (noise tensors included), sequence of calls and chunk plan, the forward
 * outputs, all parameter, latent, expression and input gradients and nfb_loss_mse_grad's loss repeat bit for bit.  The chunk
 * plan follows from the memory budget, which is NFB_TRAIN_MEM_MB when set and otherwise 60 % of the device memory free at the
 * handle's first training call, so runs meant to repeat should set NFB_TRAIN_MEM_MB.  Results across chunk plans, SM counts
 * or builds agree to rounding only.  In a multi-rank run each rank's backward repeats, but the summation order of the
 * gradient all-reduce (NCCL, gloo) is the collective's.
 * Launches: compositing backward, scale, dX chain, weight-gradient GEMMs and their fixed-order reduction per chunk, then the
 * finalize step. */
int nfb_render_backward(NfbHandle* h, const NfbOutGrads* out_grads, const float* const params_coarse[26],
                        const float* const params_fine[26], float* const grads_coarse[26], float* const grads_fine[26],
                        float* grad_latent, void* stream);

/* Gradients with respect to the render's inputs (device pointers; any member may be NULL = not computed).  Shapes as in
 * NfbRays: ray_origins, ray_directions [n,3], dir_z [n], background [n,3]; expression [76] is dL/d the expression given to
 * nfb_set_frame before the forward (before its division by 3).  Outputs are OVERWRITTEN, never accumulated.  Both passes add
 * into the same per-ray gradients.  The near/far bounds (NfbRays.near_/far_) and the sample depths carry no gradient: the
 * coarse depths depend only on near/far/t_rand, the fine ones are detached as in the reference (train_utils.py:124). */
typedef struct {
  float* ray_origins;
  float* ray_directions;
  float* dir_z;
  float* background;
  float* expression;
} NfbInputGrads;

/* nfb_render_backward plus input gradients (in_grads NULL: exactly nfb_render_backward).
 * Input-only mode: grads_coarse and grads_fine both NULL.  No parameter gradient is formed; of the weight-gradient GEMMs only
 * the four that yield the layer-0 / layer-3 bias sums run (d latent and d expression need them), and the finalize step runs
 * only its latent / expression block.  This is what fitting a frozen avatar (expression, pose, latent) to images uses.
 * params_* are still required (the input gradients multiply by the PE, conditioning and direction columns).
 * Errors: NFB_ERR_INVALID when a dir_z or background gradient is requested and the forward had no dir_z / background;
 * NFB_ERR_UNSUPPORTED when a ray gradient (origins, directions, dir_z) is requested after a forward that generated its rays
 * in the kernel (NfbRays.o == NULL).  Works through the chunked backward.  The training forward saves o, d and the direction
 * input per ray (28 B) with its other state, so no caller buffer beyond those nfb_render_backward already needs must stay
 * alive.  In input-only mode with neither grad_latent nor in_grads->expression, the weight-gradient launch is skipped.
 * Launches: nfb_render_backward's, plus one (background / expression only) or two (ray gradients) per chunk.  The same
 * reproducibility holds as for nfb_render_backward, in input-only mode too. */
int nfb_render_backward_ex(NfbHandle* h, const NfbOutGrads* out_grads, const float* const params_coarse[26],
                           const float* const params_fine[26], float* const grads_coarse[26], float* const grads_fine[26],
                           float* grad_latent, const NfbInputGrads* in_grads, void* stream);

/* ---- Several frames in one call (NFB_MULTI_FRAME) ----
 * A loss over rays of several frames (one latent code fitted to several frames, a clip's per-frame expressions in one step,
 * training batches drawn from several images) as ONE forward with ONE saved training state and ONE backward: every ray names its
 * frame, and the kernel adds that frame's folded layer-0 / layer-3 biases to the ray's rows.  Each frame's folded rows are the
 * bits nfb_set_frame would fold for it alone, so a ray renders exactly as a single-frame call of its frame renders it.
 *
 * State.  The frames of nfb_set_frames and the frame of nfb_set_frame are independent: each leaves the other as it was, and the
 * single-frame entries keep using the frame of nfb_set_frame.  Loading weights (nfb_load_weights, nfb_repack) makes both stale.
 * A multi-frame training forward replaces the handle's saved training state like nfb_render_forward_train does, and copies the
 * frame table and conditioning vectors: a later nfb_set_frame(s) or evaluation render does not change what is differentiated.
 *
 * nfb_set_frames: expressions [n_frames,76] and latents [n_frames,32], DEVICE, row-major.  Folds each (expression / 3, latent) pair
 * into the layer-0 / layer-3 biases of both loaded networks, about 4 KB per frame.  1 <= n_frames <= NFB_MAX_FRAMES, else
 * NFB_ERR_INVALID / NFB_ERR_UNSUPPORTED.  1 launch. */
int nfb_set_frames(NfbHandle* h, const float* expressions, const float* latents, int n_frames, void* stream);

/* nfb_render_forward / nfb_render_forward_train with a per-ray frame: frame_index is a DEVICE int32 [n_rays] in [0, n_frames) of
 * the last nfb_set_frames.  Explicit rays only (rays->o, d): in-kernel generation is one pose per call, so o == NULL gives
 * NFB_ERR_UNSUPPORTED.  A ray whose index is out of range (negative or >= n_frames) reads nothing out of bounds: it renders as if
 * its conditioning were NaN, so its outputs are NaN and gradients that reach it are non-finite; no other ray is affected.
 * Without nfb_set_frames first: NFB_ERR_STATE.  The chunked training forward (over the memory budget, see
 * nfb_render_forward_train) also re-reads frame_index in the backward: keep it alive with the rays.  1 launch each (the training
 * forward copies the frame table first). */
int nfb_render_forward_frames(NfbHandle* h, const NfbRays* rays, const int32_t* frame_index, const NfbSampling* sampling,
                              const NfbNoise* noise /* nullable */, const NfbOutputs* out, void* stream);
int nfb_render_forward_frames_train(NfbHandle* h, const NfbRays* rays, const int32_t* frame_index, const NfbSampling* sampling,
                                    const NfbNoise* noise /* nullable */, const NfbOutputs* out, void* stream);

/* Backward of the last nfb_render_forward_frames_train: nfb_render_backward_ex's parameter and input gradients (in_grads may be
 * NULL; its `expression` member must be NULL: NFB_ERR_INVALID), plus per-frame conditioning gradients grad_latents [n_frames,32]
 * and grad_expressions [n_frames,76] (device; either may be NULL), dL/d the rows given to nfb_set_frames (the expression before its
 * division by 3).  A frame without rays gets exactly zero.  The conditioning columns of layers_xyz.0 / .3 become
 * sum_f db_f (x) c_f, with db_f the layer's bias gradient summed over frame f's rays; the bias gradients themselves are the totals
 * as always.  Input-only mode (grads_coarse and grads_fine NULL) forms no parameter gradient, as in nfb_render_backward_ex; with
 * neither conditioning nor input gradients requested it is NFB_ERR_INVALID.  The per-frame sums are taken per ray, then per frame
 * over the rays in ascending order, and across chunks in chunk order: the reproducibility of nfb_render_backward holds.
 * nfb_render_backward_frames after a single-frame training forward is NFB_ERR_STATE; nfb_render_backward(_ex) after a multi-frame
 * forward is NFB_ERR_STATE when it is asked for grad_latent or in_grads->expression (there is no one latent to return; the other
 * gradients are formed as here).
 * Launches: nfb_render_backward_ex's (without the weight-gradient launch in input-only mode), plus two per chunk for the per-frame
 * sums, and one for the per-frame gradients. */
int nfb_render_backward_frames(NfbHandle* h, const NfbOutGrads* out_grads, const float* const params_coarse[26],
                               const float* const params_fine[26], float* const grads_coarse[26], float* const grads_fine[26],
                               float* grad_latents, float* grad_expressions, const NfbInputGrads* in_grads, void* stream);

/* ---- Training-step tail: loss, optimizer, re-pack (replaces train_transformed_rays.py:355-400 for callers that adopt it;
 * the drop-in Python surface keeps working with torch.nn.functional.mse_loss + torch.optim.Adam) ----
 *
 * nfb_loss_mse_grad: d/d rgb of mse(rgb_coarse, target) + mse(rgb_fine, target) (train_transformed_rays.py:355-362, 382), the
 * means taken over n_total * 3 elements — n_total is the GLOBAL batch size when the n_rays of this call are one shard of it, so
 * that a SUM all-reduce of the parameter gradients gives the single-process gradient.  Writes grad_rgb_* [n_rays,3] (feed them
 * to nfb_render_backward) and ADDS this shard's share of the two loss values to loss[0], loss[1] (zero them first).  1 launch
 * of one thread block, so the loss sums meet in a fixed order.  Cost: that block streams all 3 * n_rays elements on one SM,
 * so its time grows with n_rays: measured on an H100 80GB HBM3 (700 W), 11-17 us at 2048 rays as before, but 142 us at
 * 262,144 rays (a 512x512 frame) where the earlier multi-block launch took 10-17 us. */
int nfb_loss_mse_grad(NfbHandle* h, const float* rgb_coarse, const float* rgb_fine /* nullable */, const float* target,
                      int n_rays, long long n_total, float* grad_rgb_coarse, float* grad_rgb_fine, float* loss, void* stream);

/* torch.optim.Adam (betas, eps as given; no weight decay / amsgrad; YAML optimizer block) over ONE flat FP32 bucket of n
 * floats — the caller lays out both networks' parameters and the latent-code table in it and hands views of it to
 * nfb_render_backward as gradient targets, so neither a gradient copy nor a torch.cat precedes an all-reduce.  In place:
 * params, exp_avg, exp_avg_sq are updated, grads are multiplied by grad_scale before use and ZEROED afterwards
 * (optimizer.zero_grad()).  The latent-code regulariser 10 * 0.0005 * ||latent||_2 (train_transformed_rays.py:369-372, 386) is
 * applied here: reg_weight * l / ||l|| is added to the gradient of the 32 floats at reg_offset (reg_offset < 0: none).
 * `step` counts from 1; `lr` is this step's learning rate (the caller evaluates the schedule of :393-399).  1 launch. */
typedef struct {
  float lr, beta1, beta2, eps;
  int32_t step;
  float grad_scale;
  long long reg_offset;
  float reg_weight;
} NfbAdam;
int nfb_adam_step(NfbHandle* h, float* params, float* grads, float* exp_avg, float* exp_avg_sq, long long n, const NfbAdam* hp,
                  void* stream);

/* nfb_adam_step with its per-step scalars in DEVICE memory, so that a whole training iteration can be captured once in a CUDA graph
 * and replayed: `dev_state` points to an NfbAdamDev on the device.  Each call first advances `step` and evaluates the reference's
 * learning-rate schedule lr0 * decay_factor ^ ((i - 1) / decay_steps) for loop index i = step - 1 >= 1 (lr0 at i = 0;
 * train_transformed_rays.py:393-399) in float64 on the caller's double constants, and the bias corrections 1 - beta^step from the
 * FP32 betas the moment update uses (1 thread), then runs the Adam kernel; lr_over_bc1 and sqrt_bc2 are rounded to FP32 once.  The
 * regularised row is table_offset + 32 * row[0]; there is none when table_offset < 0, row is NULL or row[0] < 0 (row = device pointer
 * to the current latent index, so eager steps and graph replays of one trainer can share one state and one step counter).
 * 2 launches.  Version 131 made lr0, decay_factor and decay_steps double (they were float). */
typedef struct {
  int32_t step, pad;               /* in/out: steps taken so far (start at 0) */
  double lr0, decay_factor, decay_steps;
  float beta1, beta2, eps, grad_scale, reg_weight;
  long long table_offset;
  const long long* row;
  float lr_over_bc1, sqrt_bc2;     /* out: this step's scalars (written by the prepare kernel) */
  long long reg_offset;            /* out */
} NfbAdamDev;
int nfb_adam_step_dev(NfbHandle* h, float* params, float* grads, float* exp_avg, float* exp_avg_sq, long long n, NfbAdamDev* dev_state,
                      void* stream);

/* nfb_load_weights for both networks at once (params_fine may be NULL), two launches (FP64 fold, pack): the re-pack after an
 * optimizer step.  With params_fine NULL only network 0 is re-packed: network 1's buffers keep their bytes (and a network 1
 * loaded before stays loaded), so a fine network loaded earlier renders with its earlier weights. */
int nfb_repack(NfbHandle* h, const float* const params_coarse[26], const float* const params_fine[26], void* stream);

/* ---- The steps either side of the path (SURVEY.md 8f ranks 3, 4) ----
 *
 * nfb_frame_products: the 8-bit images eval_transformed_rays.py writes per rendered frame, from the path's outputs still on the
 * device: rgb_u8 = cast_to_image(rgb) (:184-192), normals_u8 [(H-1),(W-1),3] = torch_normal_map(disparity, intrinsics, w_last,
 * clean=True) (:84-119, called at :469 with disp_fine and weights_fine[:, -1]), disparity_u8 = cast_to_disparity_image (:195-198).
 * Any output (and w_last) may be NULL.  The bytes equal the reference functions' (same FP32 operation order).  torch's two back
 * ends round torch_normal_map differently in two places: CUDA turns ".../ fx" (division by a host scalar) into a multiplication by
 * the reciprocal (1 / fx in double, rounded to FP32) and sums the normal's squared components as (x2 + z2) + y2; the CPU divides
 * and sums (x2 + y2) + z2.  The default follows the CUDA back end — what the eval script computes on a GPU; NFB_PRODUCTS_LIKE_TORCH_CPU follows the CPU back
 * end (the two differ by one level in ~2e-4 of the bytes).  Square frames only for the normal map (the reference's expression
 * does not broadcast otherwise).  1 launch (+1 for disparity_u8). */
enum { NFB_PRODUCTS_LIKE_TORCH_CPU = 1 };
int nfb_frame_products(NfbHandle* h, const float* rgb /* [H,W,3] */, const float* disparity /* [H,W] */,
                       const float* w_last /* [H,W] or NULL */, const double intrinsics[4], int height, int width, uint8_t* rgb_u8,
                       uint8_t* normals_u8, uint8_t* disparity_u8, int flags, void* stream);

/* Importance map of one training image (train_transformed_rays.py:230-239): probs[bbox[0]:bbox[1], bbox[2]:bbox[3]] = p, 1 - p
 * elsewhere, normalised; q_out / q_in are the two float64 values of the normalised map exactly as numpy produced them. */
typedef struct {
  int32_t height, width;
  int32_t bbox[4];
  double q_out, q_in;
} NfbRayMap;
/* Optional gathers of nfb_sample_rays (train_transformed_rays.py:323-331); every member may be NULL / unused.  Pixel of flat
 * index k: (row, col) = (k % height, k / height) — the reference's transposed-meshgrid indexing. */
typedef struct {
  float pose[12];            /* camera-to-world 3x4 of the frame: rays as get_ray_bundle would give them */
  double intrinsics[4];
  const float* image;        /* [H,W,3] device */
  const float* background;   /* [H,W,3] device */
  float* ray_origins;        /* [size,3] out */
  float* ray_directions;     /* [size,3] out */
  float* target;             /* [size,3] out */
  float* background_out;     /* [size,3] out */
  int32_t* pixel_rc;         /* [size,2] out */
} NfbRayGather;
/* np.random.choice(H * W, size, replace=False, p=map.reshape(-1)) (:319-321) on the device, bit-identical indices for the same
 * uniform draws: `draws` (device, float64 in [0,1)) is consumed exactly like RandomState.rand inside choice — round r reads
 * (size - n_found) values.  state (device int32[3] = n_found, rounds run, draws consumed; zero it to start) lets a caller that must
 * stay in lock-step with a host RNG run one round per call.  indices [size] receives the selection in numpy's order; size <= 2048.
 * 1 launch (one thread block; the float64 cumulative sum is evaluated exactly without being materialised, csrc/nfb_sampler.h). */
int nfb_sample_rays(NfbHandle* h, const NfbRayMap* map, const double* draws, int size, int max_rounds, long long* indices,
                    int32_t* state, const NfbRayGather* gather /* nullable */, void* stream);
/* ---- Training rays from several images per step (NFB_TRAIN_IMAGES) ----
 * The training set as the sampler reads it, built once: every table holds one row per training image.  `images` and
 * `background` may be DEVICE memory or pinned HOST memory (read in place through unified addressing: only the selected pixels
 * are read, so a large FP32 dataset may stay on the host).  The maps must be importance_map's (nerf/ray_sampler.py): height x
 * width of the batch, the box inside the frame. */
typedef struct {
  const NfbRayMap* maps;     /* DEVICE [n_images] */
  const float* poses;        /* DEVICE [n_images][12] camera-to-world 3x4, row-major */
  const float* expressions;  /* DEVICE [n_images][76] */
  const float* images;       /* [n_images][height][width][3] FP32 */
  const float* background;   /* [height][width][3] FP32 or NULL (one background for the whole set, as the reference loads it) */
  int32_t n_images, height, width, pad;
  double intrinsics[4];
} NfbTrainImages;
/* What nfb_sample_rays_images writes; every member may be NULL (not written).  Ray k * n + j is ray j of image_index[k]. */
typedef struct {
  float* ray_origins;        /* [K * n][3] */
  float* ray_directions;     /* [K * n][3] */
  float* target;             /* [K * n][3] */
  float* background;         /* [K * n][3]; needs data->background */
  int32_t* pixel_rc;         /* [K * n][2] */
  long long* indices;        /* [K * n] flat map indices, numpy's order per image */
  int32_t* frame_index;      /* [K * n] = k: the frame_index of nfb_render_forward_frames[_train] */
  float* expressions;        /* [K][76] = expressions[image_index[k]]: the expressions of nfb_set_frames */
  float* latents;            /* [K][32] = latent_table[image_index[k]]: the latents of nfb_set_frames */
  int32_t* state;            /* [K][3] per image: n_found, rounds run, draws consumed */
  long long* shortfall;      /* [K] running count: slot k += n - n_found (pixels the selection repeated) */
} NfbImageBatch;
/* np.random.choice(H * W, n, replace=False, p=map[image_index[k]]) and the gathers of nfb_sample_rays for K images in ONE launch
 * (one 1024-thread block per image).  image_index (DEVICE int32 [K], repeats allowed) and draws (DEVICE float64
 * [K][max_rounds * n]; image k consumes its own slice exactly as nfb_sample_rays consumes `draws`) are read at run time, as is
 * latent_table ([n_images][32], DEVICE), so a captured launch samples whatever the tables hold at replay.  Per image the indices,
 * pixel_rc, rays, target and background equal nfb_sample_rays' on that image fed the same draw slice, bit for bit.  The launch
 * resets its own per-image state (no memset between calls).
 * Incomplete selection: when max_rounds rounds do not find n distinct pixels of an image (e.g. a tiny box holding most of the
 * mass), the missing slots j >= n_found repeat the first pixels, slot j taking selected pixel j % n_found, so the batch stays
 * finite; state[k][0] < n says so, and shortfall[k] adds n - n_found.  A caller that must not train on repeats checks state.
 * An image index outside [0, n_images), or a map the sampler cannot follow (another shape, a box outside the frame), reads
 * nothing: that image's rays, target, background and conditioning rows are NaN, its indices and pixel_rc -1 and its frame_index
 * K, which is out of range for nfb_set_frames of K frames, so those rays render NaN.
 * Scratch: handle-owned, sized on first use, K * (H * W * 4 B + 708 KiB) (64 MiB of first-occurrence table for 64 images at
 * 512 x 512).  Errors: NFB_ERR_INVALID for a null handle / data / table / index / draws / out, K, n or max_rounds < 1, n > 2048,
 * height * width < n, a requested background without one; NFB_ERR_UNSUPPORTED for K > NFB_MAX_STEP_IMAGES.  1 launch (+1 the
 * first time the scratch grows). */
int nfb_sample_rays_images(NfbHandle* h, const NfbTrainImages* data, const int32_t* image_index, int K, int n, const double* draws,
                           int max_rounds, const float* latent_table, const NfbImageBatch* out, void* stream);
/* The latent-table rows of a flat gradient bucket for a step over K images (what autograd leaves for
 * mse + mse + reg_weight * sum_k ||latent_table[image_index[k]]||_2 with per-frame conditioning): table_grads ([n_rows][32],
 * DEVICE) receives, in ascending k, grad_latents[k] (DEVICE [K][32], nfb_render_backward_frames' grad_latents) on row
 * image_index[k]; then, in ascending k, reg_weight * l / ||l|| with l = latent_table[image_index[k]] (nothing at l == 0, as
 * torch.norm's subgradient).  Each addition is one FP32 add of one FP32 term: term = (reg_weight * (1 / sqrt(s))) * l, each
 * operation rounded, s = the sum of the 32 squares in xor-butterfly order (offsets 16, 8, 4, 2, 1).  No atomics: the sums
 * repeat bit for bit.  Rows not named get nothing; an index outside [0, n_rows) adds nothing.  reg_weight == 0: no
 * regulariser term.  K in [1, NFB_MAX_STEP_IMAGES].  1 launch. */
int nfb_latent_rows_grad(NfbHandle* h, const float* grad_latents, const int32_t* image_index, int K, const float* latent_table, int n_rows,
                         float* table_grads, float reg_weight, void* stream);
/* ---- Fitting steps over several images (NFB_FIT_STEP) ----
 * The pose and expression rows of a fitting step's gradient: what autograd leaves in data->poses and data->expressions (as
 * [n_images][12] and [n_images][76] leaves) for a loss over the K * n rays nfb_sample_rays_images drew from `data` with the same
 * image_index, given the per-ray ray gradients and per-frame expression gradients of nfb_render_backward_frames.
 *
 * Pose rows.  Ray j of slot k sits at pixel (row, col) = pixel_rc[k * n + j] (nfb_sample_rays_images' pixel_rc); the sampler
 * built it as d = R c, o = t from the 3x4 row-major pose [R | t] and the camera direction c = (cx, cy, -1), cx = (col - W * cx0)
 * / fx, cy = -(row - H * cy0) / fy in FP32 (the same device helper forms both, so these are the rays' own bits).  So
 *     dR[q][0] = sum_j dd_j[q] * cx_j,  dR[q][1] = sum_j dd_j[q] * cy_j,  dR[q][2] = sum_j (-dd_j[q]),  dt[q] = sum_j do_j[q].
 * Order (no atomics: the rows repeat bit for bit).  First, per slot k, 256 partial sums: partial t adds the terms of rays
 * j = t, t + 256, t + 512, ... in ascending j, each term one rounded FP32 product (dd * cx, dd * cy), a negation (-dd) or the
 * value (do), each addition one rounded FP32 add starting from +0; then the partials meet in a halving tree, partial[t] +=
 * partial[t + s] for s = 128, 64, 32, 16, 8, 4, 2, 1, and partial[0] is slot k's sum.  Then, in ascending k, slot k's 12 sums
 * are added (one FP32 add each) onto pose_grads[image_index[k]]: rows are ADDED to, and an image named twice accumulates both
 * slots in that order.  A NULL grad_ray_directions (origins) counts as zero for the R (t) columns.
 * Expression rows.  In ascending k, grad_expressions[k] ([K][76], nfb_render_backward_frames' grad_expressions) is added onto
 * expression_grads[image_index[k]], one FP32 add per element, in the same launch as the pose rows.
 * Edges.  An image_index outside [0, n_images) adds nothing (its slot's sums are formed and dropped).  A NaN ray gradient
 * reaches only its own slot's row.  An incomplete selection (state[k][0] < n: repeated pixels) counts every repeat, each
 * repeated pixel being a ray of the batch.  Rows not named get nothing.
 * Errors, before any CUDA call: NFB_ERR_INVALID for a null handle / data / image_index, K or n < 1, n > 2048, a data set with
 * n_images, height or width < 1, pose_grads without pixel_rc or without any ray gradient, expression_grads without
 * grad_expressions or the other way round; NFB_ERR_UNSUPPORTED for K > NFB_MAX_STEP_IMAGES.  With pose_grads and
 * expression_grads both NULL nothing is written and nothing launched.
 * Launches: 2 with pose rows (slot sums: K blocks of 256 threads; rows: one block), 1 with expression rows only.  Scratch: the
 * handle's [NFB_MAX_STEP_IMAGES][12] slot sums, allocated once at the first call (it never moves: nfb_buffer_epoch does not
 * change). */
int nfb_fit_rows_grad(NfbHandle* h, const NfbTrainImages* data, const int32_t* image_index, int K, int n,
                      const int32_t* pixel_rc,           /* [K*n][2], nfb_sample_rays_images' */
                      const float* grad_ray_origins,     /* [K*n][3] or NULL */
                      const float* grad_ray_directions,  /* [K*n][3] or NULL */
                      float* pose_grads,                 /* [n_images][12] or NULL: rows ADDED to */
                      const float* grad_expressions,     /* [K][76] or NULL */
                      float* expression_grads,           /* [n_images][76] or NULL: rows ADDED to */
                      void* stream);

/* ---- A learned background (NFB_TRAIN_BACKGROUND) ----
 * The rows of a learned [height][width][3] background table's gradient: what autograd leaves in the table for a loss over rays
 * whose background colours were gathered from it at pixel_rc (nfb_sample_rays_images' pixel_rc, or any slice [r0, r1) of it, as a
 * data-parallel rank passes its own rays), given the per-ray render term grad_bg_render (NfbInputGrads.background of the
 * backward) and the per-ray loss term grad_bg_loss (nfb_loss_background_grad's grad_bg_rays; NULL: none), each [n_rays][3].
 * Ray r sits at table row row * width + col, the index the sampler's gathers read (one shared device helper forms both).
 * Order: table_grads[row r][c] += g_r[c] for r = 0 .. n_rays - 1 in ascending r, where g_r = grad_bg_render[r] +
 * grad_bg_loss[r] is rounded once (g_r = grad_bg_render[r] without a loss term) and each add into a row is one rounded FP32 add.
 * Rows are ADDED to; rows no ray names get nothing.  No atomics: the rows repeat bit for bit.  (The pixels are split between the
 * 1024 warps of the launch by table index; each warp walks all rays in ascending order, 32 at a time, and one lane adds each of
 * its pixels' rays of those 32 in ascending order.  So the order holds for any batch, with no sort.)
 * Edges: a pixel_rc entry outside the table (-1, as the sampler writes for an out-of-range image slot) adds nothing.  A NaN in
 * g_r reaches only its own pixel's row.  A pixel named several times (an incomplete selection's repeats, two slots drawing the
 * same pixel) accumulates every ray in ascending r.
 * Errors, before any CUDA call: NFB_ERR_INVALID for a null handle / pixel_rc / grad_bg_render / table_grads, n_rays < 0,
 * height or width < 1, height * width > 2^31 - 1.  n_rays == 0 adds nothing and launches nothing.  Launches: 1. */
int nfb_background_rows_grad(NfbHandle* h, const int32_t* pixel_rc /* [n_rays][2] */, int n_rays, int height, int width,
                             const float* grad_bg_render /* [n_rays][3] */, const float* grad_bg_loss /* [n_rays][3] or NULL */,
                             float* table_grads /* [height][width][3]: rows ADDED to */, void* stream);
/* The supervised background term of train_transformed_rays.py:375-387, weight * mean_r(w_last[r] * ||bg[r] - target[r]||^2) with
 * the mean over n_total rays (the GLOBAL batch when these n_rays are one shard of it, as in nfb_loss_mse_grad); the reference's
 * weight is 0.001 and its w_last the last pass's (NfbOutputs.w_last).
 * Order, every operation one FP32 rounding: s = weight * (1 / n_total) (as autograd's mean backward forms it on CUDA); per ray
 * d[c] = bg[c] - target[c], e = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2];  grad_bg_rays[r][c] = (2 * d[c]) * (s * w_last[r]),
 * grad_w_last[r] = s * e (OVERWRITTEN);  loss[0] += S * s, S the sum of the terms w_last[r] * e over the rays in loss_mse_grad's
 * fixed order: thread t of one 1024-thread block adds rays t, t + 1024, ... in ascending order from +0, the lanes of each warp
 * meet by xor butterfly (offsets 16, 8, 4, 2, 1: lane value += the partner's), and warp 0 .. 31's lane-0 sums are added in
 * ascending order from +0.  So the loss repeats bit for bit, and the shards' shares sum to the batch's loss to rounding.
 * Errors, before any CUDA call: NFB_ERR_INVALID for any null pointer, n_rays < 0, n_total < n_rays or n_total <= 0.  n_rays == 0
 * writes and launches nothing.  Launches: 1 (one thread block). */
int nfb_loss_background_grad(NfbHandle* h, const float* bg_rays /* [n_rays][3] */, const float* target /* [n_rays][3] */,
                             const float* w_last /* [n_rays] */, int n_rays, long long n_total, float weight,
                             float* grad_bg_rays /* [n_rays][3] */, float* grad_w_last /* [n_rays] */, float* loss /* ADDED to */,
                             void* stream);

/* Host-only test hook of the same arithmetic: out[i] = np.cumsum(p)[ks[i]] (ks[i] == -1: the last entry) for the map with the
 * ascending flat indices zeroed_sorted set to zero.  No CUDA call. */
int nfb_host_map_cdf(const NfbRayMap* map, const long long* zeroed_sorted, int n_zero, const long long* ks, int n, double* out);

/* Test hook: device pointers of the training state (valid until the next forward_train on the handle).  NFB_ERR_STATE after a
 * chunked (over-budget) forward: its buffers only ever hold one chunk. */
typedef struct {
  const uint8_t* records;      /* n_tiles records of record_bytes (layout: nfb_layout.h kRec*); 1 MiB, 2 MiB after an exact-grad
                                  forward: the lo images at +1 MiB, at the offsets of their hi images */
  long long n_tiles;
  int32_t record_bytes;
  const float* d_raw;          /* [n_tiles][128][4] dL/d(rgb_raw, sigma_raw), unscaled */
  const float* acc_coarse;     /* acc_floats accumulators in the kernel's folded parametrisation (kAcc*) */
  const float* acc_fine;
  int32_t acc_floats;
  const float* scale;          /* [0] loss scale, [1] its inverse */
  const float *z_coarse, *raw_coarse, *z_fine, *raw_fine;
  int32_t tiles_coarse, tiles_fine, rays_per_unit;
  /* What the input gradients of nfb_render_backward_ex are formed from.  rays and dnorm are the training forward's: rays
   * [n][7] = (o, d, v0) with v0 the direction encoder's first input (dir_z, else d_z), dnorm [n] = |d| in FP32.  The other three
   * are NULL until a backward of this forward has formed per-ray terms, and stay NULL when that backward did not need them:
   * rows [n_tiles][128][4] = (dp, d v0) per sample row, unscaled (written when a ray gradient was requested), ray_dn
   * [passes][n] = dL/d|d| of each pass, ray_bg [passes][n][3] = dL/d background of each pass (only with a background). */
  const float* rays;
  const float* dnorm;
  const float* rows;
  const float* ray_dn;
  const float* ray_bg;
  /* What a multi-frame forward (nfb_render_forward_frames_train) saved; n_frames is 0 and the pointers NULL after a single-frame
   * one.  frame [n] = the slot each ray rendered with (n_frames where its index was out of range); frame_table[net]
   * [n_frames + 1][512] = the folded rows of steps 0 and 3 per frame, the last row NaN ([1] NULL without a fine pass);
   * frame_cond [n_frames][108] = [expression / 3 ; latent] per frame.  ray_sums [passes][n][512] (dY0 | dY3 summed over each
   * ray's samples, unscaled) and frame_sums [n_frames][2][512] (those summed over each frame's rays) are NULL until a backward of
   * this forward has formed them. */
  int32_t n_frames;
  const int32_t* frame;
  const float* frame_table[2];
  const float* frame_cond;
  const float* ray_sums;
  const float* frame_sums;
  /* What the parameter-gradient backward summed, NULL / 0 until a backward of this forward has run.  dw_partials = the
   * weight-gradient partials of the last backward: slot (network 0 parts first, then network 1's) of dw_slot_floats floats
   * each, filled by the parts that got tiles (part p of a network owns its tiles [p per, (p + 1) per), per = ceil(tiles /
   * parts)); dw_slot_floats is the accumulator range below the raw-output biases (kAccBRaw, nfb_layout.h) after a full launch,
   * the compact [dW0 | dW3a | db0 | db3] slot after a PE-only one (dw_pe_only = 1: an input-only backward that formed d latent
   * or d expression); dw_parts = parts per network of that launch (0, 0 and dw_partials NULL when the backward ran no
   * weight-gradient launch).  ray_bias_sums [passes][n][4] = each ray's sums of d raw over its samples, unscaled. */
  const float* dw_partials;
  int32_t dw_slot_floats;
  int32_t dw_parts[2];
  int32_t dw_pe_only;
  const float* ray_bias_sums;
} NfbTrainDebug;
int nfb_train_debug(NfbHandle* h, NfbTrainDebug* out);

/* Test hook: device pointers of the packed weights of network `net` (NFB_NET_COARSE / NFB_NET_FINE), the buffers every kernel
 * reads its weights from, as nfb_load_weights / nfb_repack wrote them (layout: DESIGN.md §3, nfb_layout.h).  x1 [x1_bytes]: the
 * FP16 forward stream of fast mode; x3 [x3_bytes]: exact mode's stream, per unit the hi unit then the lo unit; bwd [bwd_bytes]:
 * the transposed FP16 stream of the backward chain; w6 [144][256] and b6 [144]: the folded layers_dir.0[:, :256] . fc_feat
 * (rows 0..127) and fc_alpha . fc_feat (row 128), rows 129..143 zero; bias_static [bias_floats]: the bias block; bias_frame
 * [bias_floats]: the bias block with the frame of the last nfb_set_frame folded into the rows of steps 0 and 3 (unwritten before
 * the first); w0c / w3c [256][108]: the conditioning columns of layers_xyz.0 / .3; wd0b_t [24][128]: the direction columns of
 * layers_dir.0, transposed.  Valid until the handle is destroyed.  No CUDA call.  NFB_ERR_STATE if that network is not
 * loaded. */
typedef struct {
  const uint8_t *x1, *x3, *bwd;
  const float *w6, *b6, *bias_static, *bias_frame, *w0c, *w3c, *wd0b_t;
  int64_t x1_bytes, x3_bytes, bwd_bytes;
  int32_t bias_floats;
  /* The lo half of the backward stream (exact-grad mode; bwd's layout): the transposition of the lo units of x3 as bwd is of its hi
   * units.  NULL and 0 until the handle's first exact-grad training forward. */
  const uint8_t* bwd_lo;
  int64_t bwd_lo_bytes;
} NfbWeightDebug;
int nfb_debug_weights(NfbHandle* h, int net, NfbWeightDebug* out);

/* End-to-end convenience for callers with HOST buffers (bench.py's e2e leg, C/C++ users): copies
 * expression/latent/background to the device, renders image rows [row_begin,row_begin+rows) of a
 * height x width frame with in-kernel ray generation, and copies the outputs back.  Host pointers
 * should be pinned for full copy speed.  Output layout: out_host = rgb_c[n,3] | disp_c[n] | acc_c[n] |
 * rgb_f[n,3] | disp_f[n] | acc_f[n] | w_last[n], n = rows*width, 11*n floats.  Synchronises `stream`. */
int nfb_render_frame_host(NfbHandle* h, const float pose[12], const double intrinsics[4],
                          int height, int width, int row_begin, int rows, float near_, float far_,
                          const float* expression_host, const float* latent_host,
                          const float* background_host /* [rows*width,3] or NULL */,
                          const NfbSampling* sampling, float* out_host, void* stream);

/* Test hook, host only (no CUDA call): the compile-time schedules the kernels execute.  which: 0 = render program,
 * 2 = backward chain program (each: MMA N, K atom of the A operand, flags, (stream offset / 16) | rows << 20), 3 = weight-gradient jobs (a_off, a_rows, a_half, b_off, b_rows, bias_layer, out_off,
 * out_ld, out_row0, group), 4 = the CTA split of the weight-gradient launch (in/out: out[0..2] = SMs, tiles of network 0, tiles of
 * network 1 -> parts of network 0, parts of network 1, job groups per part).  index < 0: returns the number of entries; otherwise fills out[0..] (out_words >= 10) and returns
 * the number of words written, or -1. */
int nfb_debug_schedule(int which, int index, uint32_t* out, int out_words);

/* Number of kernel launches issued by this handle so far (all kernels of this library). */
int nfb_launch_count(NfbHandle* h, long long* out);

/* The handle's buffer epoch: how many times it has freed (to grow) or refilled a device buffer whose address a training step's
 * launches take — the training state nfb_render_forward_train saves, the frame table of nfb_set_frames, the scratch of
 * nfb_sample_rays_images and the linspace tables.  A CUDA graph captured over the handle's calls is valid while the epoch is the
 * one read after capture; once it has changed, the graph points at freed or rewritten memory and must be captured again.  The
 * staging buffers of nfb_render_frame_host and the scratch of nfb_frame_products / nfb_sample_rays are not counted (no training
 * step reads them).  Host read, no CUDA call and no synchronisation. */
int nfb_buffer_epoch(NfbHandle* h, long long* out);

/* Host helper: out[i] = torch.linspace(0, 1, n)[i] bit-for-bit (ATen's CPU kernel: step = 1/(n-1) in
 * FP32; first half start + i*step, second half end - (n-1-i)*step).  Used for t_coarse / u_fine when the
 * caller passes NULL.  No CUDA involved. */
int nfb_host_linspace(float* out, int n);

#ifdef __cplusplus
}
#endif
#endif /* NFB_H_ */
