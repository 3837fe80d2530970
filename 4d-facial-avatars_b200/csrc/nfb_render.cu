// nfb_render.cu — the per-ray hot path as ONE persistent sm_90a kernel: both precision modes, the training forward (SAVE:
// also writes the activation records the backward reads; exact-grad mode's also their lo halves) and the debug probes.
//
// Reference path replaced (nerface_code/nerf-pytorch/nerf/):
//   train_utils.py:36-162  predict_and_render_radiance   (sampling, coarse->fine control flow)
//   train_utils.py:9-33    run_network                    (encode + MLP over all samples)
//   nerf_helpers.py:195-239 positional_encoding, :344-387 sample_pdf_2, :44-65 cumprod_exclusive,
//   nerf_helpers.py:68-123 get_ray_bundle (optional in-kernel ray generation)
//   volume_rendering_utils.py:7-75 volume_render_radiance_field
//   models.py:236-261      ConditionalBlendshapePaperNeRFModel.forward
//
// Work decomposition.  A "unit of work" is R (1 or 2) rays.  One CTA per SM loops over them; per unit it runs the coarse
// pass (R*Nc sample rows) and the fine pass (R*(Nc+Nf) rows) as 128-row tiles.  Per tile the MLP is 10 GEMM steps
// (nfb_layout.h), each on wgmma: warpgroup w computes rows [64w, 64w+64) of the tile with its FP32 accumulators in
// registers.  Its epilogue (bias, ReLU, FP16 conversion) produces the A operand of the next step: in fast mode as packed
// register fragments (an m64nN accumulator fragment is, packed to f16x2, the A fragment of the next register-A wgmma), in
// exact mode as hi and lo halves written back in place into the shared-memory activation buffer the step has just finished
// reading.  Either way hidden activations never leave the SM.  In fast mode the steps are unrolled at compile time, so each
// weight unit's wgmmas are issued as one batch, and one unit stays in flight while the next is issued.
// Weights stream L2 -> shared memory through the bulk-copy (TMA) engine into a ring of pre-swizzled 32 KB units
// ([N rows x 64 K], the layout a wgmma shared-memory descriptor reads): 5 slots in fast mode, 1 in exact mode, whose hi+lo
// activation buffers take the space.
//
// Warp roles (nfb_pipeline.cuh): warp 0 = weight producer, warpgroups 1 and 2 = "row" warps.  For the per-row work
// (sampling, positional encoding, compositing, inverse-CDF resampling, the per-ray sort) thread <-> sample row; for the MLP
// each warpgroup issues the wgmma of its 64 rows and runs their epilogues.  Inside a pass each warpgroup runs the tiles on
// its own rows (prologue, MLP, post-processing) under its own named barrier; in fast mode a ping-pong of two more named
// barriers staggers their MMA issue by one step, so one's epilogue runs under the other's MMAs.  CTA-wide barriers remain at
// unit and pass boundaries only.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include "nfb_internal.h"
#include "nfb_layout.h"
#include "nfb_pipeline.cuh"
#include "nfb_ptx.cuh"
#include "nfb_save.cuh"
#include "nfb_render_common.cuh"

namespace nfb {

constexpr int kRowsMax = 512;  // sample rows of one pass of one unit of work

// shared memory map (bytes from the 1024-aligned base).  The exact-grad training forward uses exact mode's map.  Activation buffers (exact mode only; fast mode keeps the hidden
// activations in registers): 4 K atoms x [128 rows x 128 B], swizzled.
template <bool EXACT>
struct SmemMap {
  static constexpr int kSlots = EXACT ? 1 : 5;
  using WeightRing = Ring<kSlots, kMaxUnitBytes>;
  static constexpr int kActBytes = EXACT ? 4 * kTileM * 128 : 0;
  static constexpr int kRing = 0;
  static constexpr int kActHi = kRing + kSlots * kMaxUnitBytes;
  static constexpr int kActLo = kActHi + kActBytes;
  static constexpr int kPeHi = kActLo + kActBytes;
  static constexpr int kPeLo = kPeHi + kTileM * 128;
  // Per-unit buffers, one copy each unless noted (the table in DESIGN §4 gives each one's writer, reader and lifetime):
  static constexpr int kRaw = kPeLo + (EXACT ? kTileM * 128 : 0);  // coarse carry: (colour, sigma) per sample row
  static constexpr int kRawF = kRaw + kRowsMax * 16;                  // fine carry (nf == 0: the second coarse copy)
  static constexpr int kZ = kRawF + kRowsMax * 16;                    // coarse depths
  static constexpr int kZF = kZ + kRowsMax * 4;                       // fine depths (nf == 0: the second coarse copy)
  static constexpr int kW = kZF + kRowsMax * 4;                       // ray warps' scratch: [ray][kRowsMax / 2] each
  static constexpr int kCdf = kW + kRowsMax * 4;
  static constexpr int kBins = kCdf + kRowsMax * 4;
  static constexpr int kSort = kBins + kRowsMax * 4;
  static constexpr int kDirBias = kSort + kRowsMax * 4;  // [coarse of an even unit, coarse of an odd unit, fine][ray][128]
  static constexpr int kRay = kDirBias + 3 * 2 * 128 * 4;            // RayP [unit % 3][ray]
  static constexpr int kTileRaw = kRay + 3 * 2 * kRayFloats * 4;  // [128] (rgb raw, sigma raw) of the current tile
  static constexpr int kBars = kTileRaw + kTileM * 16;
  static constexpr int kHand = kBars + 2 * kSlots * 8;  // the hand-off mbarriers (Hand)
  // Fast mode: both networks' bias blocks, copied once per CTA, so the epilogues read them from shared memory.  Exact mode has
  // no room for them and reads them from global memory.
  static constexpr int kBias = (kHand + 9 * 8 + 15) / 16 * 16;
  static constexpr int kBytes = kBias + (EXACT ? 0 : 2 * kBiasFloats * 4);
  static_assert(kBytes <= 232448, "exceeds the 227 KB per-CTA shared memory limit");
  static_assert(kRaw % 16 == 0 && kBars % 8 == 0 && kHand % 8 == 0 && kBias % 16 == 0, "alignment");
};

constexpr int kTileUnits = prog_units(kFwdStream);
__constant__ ProgTable c_prog = make_prog(kFwdStream);

constexpr int max_step_units() {
  int m = 0;
  for (int s = 0; s < kNumSteps; ++s) m = step_info(s).k_atoms > m ? step_info(s).k_atoms : m;
  return m;
}
// The two row warpgroups walk the same ring and may drift apart: the one ahead holds a step's units until the other has
// consumed them too.  Each warpgroup waits for and releases every unit of a step before its epilogue, so both can always
// finish a step when the ring holds all of its units at once.
static_assert(max_step_units() <= SmemMap<false>::kSlots, "a fast-mode MLP step must fit in the weight ring");

// A compile-time MLP step: converts to its index, and keeps it usable as a constant expression (Step::value).
template <int V>
struct StepC {
  static constexpr int value = V;
  __device__ constexpr operator int() const { return V; }
};
// Calls f(StepC<I>{}) for I = B, ..., E - 1: the MLP steps as compile-time constants, so that each step's MMA issue and
// epilogue are straight-line code.
template <int B, int E, class F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (B < E) {
    f(StepC<B>{});
    static_for<B + 1, E>(f);
  }
}

// m64nNk16 wgmma into a 128- or 16-column accumulator, A from a shared-memory descriptor or from four register fragments.
__device__ __forceinline__ void mma_ss(float (&d)[64], uint64_t a, uint64_t b, uint32_t accf) { wgmma_n128(d, a, b, accf); }
__device__ __forceinline__ void mma_ss(float (&d)[8], uint64_t a, uint64_t b, uint32_t accf) { wgmma_n16(d, a, b, accf); }
__device__ __forceinline__ void mma_rs(float (&d)[64], const uint32_t* a, uint64_t b, uint32_t accf) {
  wgmma_rs_n128(d, a[0], a[1], a[2], a[3], b, accf);
}
__device__ __forceinline__ void mma_rs(float (&d)[8], const uint32_t* a, uint64_t b, uint32_t accf) {
  wgmma_rs_n16(d, a[0], a[1], a[2], a[3], b, accf);
}

// The MMAs of step `step` for this warpgroup's 64 rows: acc0 = output columns [0, 128) (or [0, 16) in acc_s when the step has
// nh0 == 16), acc1 = [128, 256), acc_s = the 16-column second half of step 6.  Consumes the step's units from the ring
// (exact mode: two slots per unit, hi then lo weights), each slot's wgmmas issued as one batch.  The ring's kLag batches
// stay in flight: a slot is released once the batch after it has been issued and its own batch waited on.  On return every
// MMA of the step is complete.
// A operand: the PE buffer for the step's PE atom; otherwise the activation buffer (exact mode) or the packed fragments the
// previous step's epilogue left in registers (fast mode: act[16 a + 4 ks + i] = fragment register i of K atom a, K slice ks).
// `step` is a StepC in fast mode (the steps unrolled, each unit's wgmmas one straight-line batch) and a
// runtime int in exact mode, whose steps stay a loop: exact mode gains nothing from the unrolling but code size.
// `issued()` runs once the step's last batch is committed, before the wait for it.
template <bool EXACT, class Step, class WeightRing, class Issued>
__device__ __forceinline__ void mlp_step_mma(Step step, WeightRing& ring, uint32_t act_hi, uint32_t act_lo, uint32_t pe_hi, uint32_t pe_lo,
                                             uint32_t row_off, uint32_t (&act)[64], float (&acc0)[64], float (&acc1)[64],
                                             float (&acc_s)[8], PhaseTimer& tm, Issued&& issued) {
  constexpr int NPART = EXACT ? 2 : 1;
  constexpr int kLag = WeightRing::kLag;
  const StepInfo si = step_info(step);
  asm volatile("" : "+r"(row_off));  // as in epi_half: the operand descriptors are formed per step, not hoisted and held
#pragma unroll
  for (int u = 0; u < si.k_atoms; ++u) {
    const bool from_pe = si.pe_first && u == 0;
    const bool rs = !EXACT && !from_pe;
    const int atom = u - si.pe_first;
    const uint32_t a_hi = (from_pe ? pe_hi : act_hi + atom * (kTileM * 128)) + row_off;
    const uint32_t a_lo = (from_pe ? pe_lo : act_lo + atom * (kTileM * 128)) + row_off;
    const uint64_t dh = wgmma_desc_sw128(a_hi), dl = wgmma_desc_sw128(a_lo);
#pragma unroll
    for (int part = 0; part < NPART; ++part) {
      const uint32_t b = ring.wait_full();
      tm.lap(10);
      const uint64_t b0 = wgmma_desc_sw128(b), b1 = wgmma_desc_sw128(b + si.nh0 * 128);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint32_t accf = (u | part | ks) ? 1u : 0u;
        const uint64_t ah = dh + (uint64_t)(ks * 2), al = dl + (uint64_t)(ks * 2);
        const uint32_t* af = act + (rs ? 16 * atom + 4 * ks : 0);
        auto mma = [&](auto& d, uint64_t bd) {
          if (rs) {
            mma_rs(d, af, bd, accf);
          } else {
            mma_ss(d, ah, bd, accf);
            if (EXACT && part == 0) mma_ss(d, al, bd, 1u);
          }
        };
        const uint64_t bh0 = b0 + (uint64_t)(ks * 2), bh1 = b1 + (uint64_t)(ks * 2);
        if (si.nh0 == 16) {
          mma(acc_s, bh0);
        } else {
          mma(acc0, bh0);
          if (si.nh1 == 128) mma(acc1, bh1);
          else if (si.nh1 == 16) mma(acc_s, bh1);
        }
      }
      wgmma_commit();
      if (u == si.k_atoms - 1 && part == NPART - 1) issued();
      if (u * NPART + part >= kLag) {
        wgmma_wait<kLag>();
        reg_fence(acc0);
        reg_fence(acc1);
        reg_fence(acc_s);
        ring.release();
      }
      tm.lap(11);
    }
  }
  if constexpr (kLag > 0) {
    wgmma_wait<0>();
    reg_fence(acc0);
    reg_fence(acc1);
    reg_fence(acc_s);
    ring.release();
    tm.lap(11);
  }
  // The fragments were read asynchronously: the epilogue overwrites them only from here.
  if constexpr (!EXACT) reg_fence<16 * (step_info(Step::value).k_atoms - step_info(Step::value).pe_first)>(act);
}

// Epilogue of one 128-column accumulator half (columns [c_base, c_base + 128)) of a ReLU layer: + bias (+ the per-ray
// direction term of step 6), ReLU, FP16 hi (and lo) written in place into the activation buffer (exact mode) or packed
// into the A fragments of the next step (fast mode: act[c_base / 4 + 2 j + hh] holds columns c_base + 8 j + 2 c, +1 of
// row r0 + 8 hh); the training record image and ReLU mask of the layer (SAVE), and the layer probe dump (PROBE, when `dump`
// is set; the production instantiations carry no probe code, which ptxas would otherwise issue as predicated stores).
// SAVE: bit hh of `live` is set when row r0 + 8 hh holds a sample of a valid ray.  The other rows (the tile's rows beyond
// R*S, the rows of an invalid ray) still go through the MLP, at points no reference evaluates; their records and masks are
// stored as zero, so that an out-of-range activation there cannot reach a weight gradient as 0 * inf.
// ROWB (multi-frame kernels): row r0 + 8 adds bias1 instead of bias, as rows of two rays add their own direction terms.
// HILO (exact-grad training forward, EXACT and SAVE): also the lo half of the record image, FP16(x - hi) of the value the record
// holds, at rec + kRecBytes (nfb_layout.h rec_stride).
template <bool EXACT, bool SAVE, bool PROBE, bool ROWB = false, bool HILO = false>
__device__ __forceinline__ void epi_half(const float (&acc)[64], int s, int c_base, const float* __restrict__ bias,
                                         const float* dirb0, const float* dirb1, uint8_t* act_hi, uint8_t* act_lo,
                                         uint32_t (&act)[64], int r0, uint8_t* rec, uint32_t live, float* dump,
                                         const float* __restrict__ bias1 = nullptr) {
  int c = threadIdx.x & 3;
  // Fast mode unrolls the steps: without this the compiler hoists the per-thread addresses of all ten epilogues out of the
  // tile loop and keeps them in registers (spilling) across the MMAs.
  asm volatile("" : "+r"(r0), "+r"(c));
  uint32_t mask[2][4] = {{0u, 0u, 0u, 0u}, {0u, 0u, 0u, 0u}};
  // SAVE: byte offset of element (feature col, sample R) of the layer's transposed record image is
  // img_offset(W, col, R) = (c_base + 8 j) * 128 + img_base[hh][e] for col = c_base + 8 j + 2 c + e, R = r0 + 8 hh, since
  // col & 7 == 2 c + e for every j: one base per (hh, e) and compile-time offsets, instead of the full swizzle per element.
  int img_base[2][2] = {{0, 0}, {0, 0}};
  if constexpr (SAVE) {
    const int W = rec_width(s);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int e = 0; e < 2; ++e) img_base[hh][e] = img_offset(W, 2 * c + e, r0 + 8 * hh);
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = c_base + 8 * j + 2 * c;
    // fast mode: `bias` is the shared-memory copy, except for ROWB's per-frame rows (global)
    float2 b;
    if constexpr (EXACT || ROWB) b = __ldg(reinterpret_cast<const float2*>(bias + col));
    else b = *reinterpret_cast<const float2*>(bias + col);
    float2 b1 = b;
    if constexpr (ROWB) b1 = __ldg(reinterpret_cast<const float2*>(bias1 + col));
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int R = r0 + 8 * hh;
      const float2 bb = hh ? b1 : b;
      float x0 = __fadd_rn(acc[4 * j + 2 * hh], bb.x), x1 = __fadd_rn(acc[4 * j + 2 * hh + 1], bb.y);
      const float* db = hh ? dirb1 : dirb0;
      if (db) { x0 = __fadd_rn(x0, db[col]); x1 = __fadd_rn(x1, db[col + 1]); }
      if (PROBE && dump) { dump[R * 256 + col] = relu_nan(x0); dump[R * 256 + col + 1] = relu_nan(x1); }
      uint32_t hi, lo = 0u, saved;
      uint32_t saved_lo = 0u;
      if constexpr (EXACT) {
        // NaN stays NaN; hi saturates at 65504 and lo carries the rest, so hi + lo reaches ~131008 and beyond that lo is
        // inf: out of range gives a non-finite render, never a clamped one.
        const float a = relu_nan(x0), bb = relu_nan(x1);
        hi = pack_f16x2(a, bb);
        const float2 h = unpack_f16x2(hi);
        lo = pack_f16x2_inf(a - h.x, bb - h.y);
        // the record is one FP16 value: converted without saturation, so an activation beyond its range is inf there (a
        // non-finite weight gradient), not 65504 (a finite, wrong one); equal to hi for every activation up to 65504
        saved = SAVE ? pack_f16x2_inf(a, bb) : hi;
        if constexpr (HILO) {  // an inf record keeps a non-finite remainder: the weight gradient stays non-finite
          const float2 s2 = unpack_f16x2(saved);
          saved_lo = pack_f16x2_inf(a - s2.x, bb - s2.y);
        }
      } else {
        hi = pack_relu_f16x2(x0, x1);
        saved = hi;
      }
      if constexpr (EXACT) {
        const int off = (col >> 6) * (kTileM * 128) + sw128_offset(R, col & 63);
        *reinterpret_cast<uint32_t*>(act_hi + off) = hi;
        *reinterpret_cast<uint32_t*>(act_lo + off) = lo;
      } else {
        act[c_base / 4 + 2 * j + hh] = hi;
      }
      if constexpr (SAVE) {
        if (rec) {
          uint8_t* img = rec + rec_x_off(s);
          uint8_t* img_j = img + (c_base + 8 * j) * 128;
          const uint32_t v = ((live >> hh) & 1u) ? saved : 0u;
          *reinterpret_cast<uint16_t*>(img_j + img_base[hh][0]) = (uint16_t)(v & 0xFFFFu);
          *reinterpret_cast<uint16_t*>(img_j + img_base[hh][1]) = (uint16_t)(v >> 16);
          if constexpr (HILO) {
            const uint32_t vl = ((live >> hh) & 1u) ? saved_lo : 0u;
            *reinterpret_cast<uint16_t*>(img_j + kRecBytes + img_base[hh][0]) = (uint16_t)(vl & 0xFFFFu);
            *reinterpret_cast<uint16_t*>(img_j + kRecBytes + img_base[hh][1]) = (uint16_t)(vl >> 16);
          }
          const uint32_t bits = ((v & 0xFFFFu) ? 1u : 0u) | ((v >> 16) ? 2u : 0u);
          mask[hh][j >> 2] |= bits << ((col & 31));
        }
      }
    }
  }
  if constexpr (SAVE) {
    if (rec) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          uint32_t m = mask[hh][w];
          m |= __shfl_xor_sync(0xffffffffu, m, 1);
          m |= __shfl_xor_sync(0xffffffffu, m, 2);
          mask[hh][w] = m;
        }
      if (c == 0) {
        uint32_t* mw = reinterpret_cast<uint32_t*>(rec + kRecMask);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          *reinterpret_cast<uint4*>(mw + (s * 128 + r0 + 8 * hh) * 8 + (c_base >> 5)) =
              make_uint4(mask[hh][0], mask[hh][1], mask[hh][2], mask[hh][3]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Hand-offs between the row warps (tiles) and the ray warps (per-ray stages), one mbarrier each, phases counted per unit:
//   cdone[b]  row warps -> ray warps: the coarse tiles of the unit in coarse buffer b are done (arrivals: every row thread)
//   cfree[b]  ray warps -> row warps: coarse buffer b has been read (arrivals: every ray-warp thread)
//   fdone     row warps -> ray warps: the unit's fine tiles are done
//   fready    ray warps -> row warps: the unit's fine depths and fine direction term are written, and the fine carry of the
//             unit before it has been read
//   sready[s] ray warps -> row warps: RayP slot s and the coarse direction term of its unit are written
// A unit's coarse buffer is it % nb, nb = 1 with a fine pass (its slack is the fine tiles of the unit before) and 2
// without one; its RayP slot is it % 3.
struct Hand {
  uint32_t base;
  __device__ __forceinline__ uint32_t cdone(int b) const { return base + 8 * b; }
  __device__ __forceinline__ uint32_t cfree(int b) const { return base + 16 + 8 * b; }
  __device__ __forceinline__ uint32_t fdone() const { return base + 32; }
  __device__ __forceinline__ uint32_t fready() const { return base + 40; }
  __device__ __forceinline__ uint32_t sready(int s) const { return base + 48 + 8 * s; }
  __device__ __forceinline__ void init() const {
    for (int b = 0; b < 2; ++b) { mbar_init(cdone(b), kRowThreads); mbar_init(cfree(b), kRayThreads); }
    mbar_init(fdone(), kRowThreads);
    mbar_init(fready(), kRayThreads);
    for (int s = 0; s < 3; ++s) mbar_init(sready(s), kRayThreads);
    mbar_fence_init();
  }
};

// PROBE: the instantiation that honours the activation probe (RenderParams::dbg_act); launch_render picks it only when the
// probe is requested.
//
// Roles.  Warp 0 streams the weights; warps 1..3 (the "ray warps") run the per-ray stages, warp 1 + rr those of ray rr of
// each unit (warp 3 only keeps the arrival counts); warpgroups 1 and 2 (the "row warps") run the tiles.  The producer and
// the row warps walk the CTA's tile stream (stream_tile, nfb_layout.h): C(0), C(1), F(0), C(2), F(1), ...  The ray warps
// run, for unit it: wait cdone(it); composite the coarse pass, CDF, inverse-CDF samples; arrive cfree; wait fdone(it-1),
// composite the fine pass of it-1; merge-sort the fine depths of it, its fine direction term; arrive fready; set up unit
// it+2 (RayP, direction encoding, coarse direction term); arrive sready.  The row warps wait sready(it) and cfree(it-nb)
// before the first tile of C(it), fready(it) before that of F(it), and arrive cdone / fdone after the last tile of a pass.
//
// Deadlock freedom.  Every arrival above is made by every thread of its side on every path: for invalid rays, for the warp
// without a ray, for n_iter = 1 and for the CTA's last unit (the loops run the same n_iter on both sides, n_iter >= 1); no
// arrival sits under a data-dependent condition.  What the ray warps arrive for unit it depends only on cdone(v <= it) and
// fdone(v <= it-1) (they run their units in order), so cfree(it - nb) and sready(it) depend on the tiles of C(v <= it-1)
// and F(v <= it-2), fready(it) on those of C(v <= it) and F(v <= it-1), and stream_order (nfb_layout.h) asserts that all
// of these come before the tile that waits.  Induction over the stream position: no wait depends on itself.  No barrier
// runs more than one phase ahead of a waiter, which the parity waits need: cdone(b)'s next phase needs C(it + nb), after
// cfree(it); fdone's needs fready(it + 1), after the ray warps' wait for fdone(it); cfree and fready need cdone / fdone of
// the next unit, after the row warps' waits; sready(s)'s needs cdone(it + 1).  The producer depends on the row warps
// only through the weight ring, which both walk in stream order.
//
// MULTI: the multi-frame kernel (render_frames_kernel).  Each ray carries a frame index (RenderParams::frame); the epilogues of
// steps 0 and 3 add the folded bias row of the ray's own frame (RenderParams::fbias) instead of the call's one frame bias, per
// accumulator row as the direction term of step 6 is.  Everything else is the same code.
//
// HILO: the exact-grad training forward (render_hilo_kernel; EXACT and SAVE): exact mode's training forward, whose records are
// 2 MiB apart and also hold the lo half of every activation image (nfb_layout.h rec_stride).  The first MiB of each is exact
// mode's record, byte for byte.
template <bool EXACT, bool SAVE, bool PROBE, bool MULTI, bool HILO = false>
__device__ __forceinline__ void render_body(const RenderParams& p) {
  static_assert(!HILO || (EXACT && SAVE), "the lo record belongs to the exact training forward");
  using M = SmemMap<EXACT>;
  constexpr size_t kRecStride = rec_stride(HILO);
  // Use the dynamic shared array directly (no integer round trip) so the compiler keeps the shared address
  // space and emits LDS/STS instead of generic loads; the swizzled operands need 1024-byte alignment.
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t smem_base = smem_base_aligned(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int NPART = EXACT ? 2 : 1;

  typename M::WeightRing ring(smem_base + M::kRing, smem_base + M::kBars);
  const Hand hand{smem_base + M::kHand};
  if (threadIdx.x == 0) {
    ring.init();
    hand.init();
  }
  float* sbias = reinterpret_cast<float*>(smem + M::kBias);
  if constexpr (!EXACT) {
    for (int i = threadIdx.x; i < 2 * kBiasFloats; i += kThreads)
      sbias[i] = p.bias[i / kBiasFloats][i % kBiasFloats];
  }
  __syncthreads();

  const TileGeom& geom = p.geom;
  const int n_iter = (geom.n_units - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int n_stream = stream_tiles(geom, n_iter);
  const int nb = geom.nf > 0 ? 1 : 2;  // coarse buffers
  const int R = geom.rays_per_unit;
  float4* raw_c = reinterpret_cast<float4*>(smem + M::kRaw);
  float4* raw_f = reinterpret_cast<float4*>(smem + M::kRawF);
  float* z_c = reinterpret_cast<float*>(smem + M::kZ);
  float* z_f = reinterpret_cast<float*>(smem + M::kZF);
  float* dirbias = reinterpret_cast<float*>(smem + M::kDirBias);
  RayP* rayp_all = reinterpret_cast<RayP*>(smem + M::kRay);

  if (warp < 4) {
    reg_dec<kRegsRenderLight>();
    if (warp == 0) {
      // ============================== weight producer ==============================
      // The whole warp runs the (warp-uniform) loop; one elected lane issues the copies.
      for (int k = 0; k < n_stream; ++k) {
        const uint8_t* base = p.wstream[stream_tile(geom, n_iter, k).pass];
        for (int i = 0; i < kTileUnits; ++i) {
          const uint32_t w = c_prog.e[i].w;
          const uint32_t off = (w & 0xFFFFFu) << 4, bytes = (w >> 20) * 128u;
#pragma unroll
          for (int part = 0; part < NPART; ++part)  // exact mode: the hi unit, then the lo unit
            ring.produce(EXACT ? base + 2 * (size_t)off + part * bytes : base + off, bytes);
        }
      }
    } else {
      // ============================== ray warps ==============================
      const int rr = warp - 1;  // this warp's ray within each unit
      const bool mine = rr < R;
      const int rs = rr * (kRowsMax / 2);  // this ray's part of the scratch buffers (R == 1: ray 0, all of them)
      float* scr_w = reinterpret_cast<float*>(smem + M::kW) + rs;
      float* scr_cdf = reinterpret_cast<float*>(smem + M::kCdf) + rs;
      float* scr_bins = reinterpret_cast<float*>(smem + M::kBins) + rs;
      float* scr_sort = reinterpret_cast<float*>(smem + M::kSort) + rs;
      const bool has_bg = p.bg != nullptr;
      const int nc = geom.nc, nf = geom.nf, SF = geom.samples(1);
      // observer: lane 0 of warp 1, laps at kProfRay + slot
      PhaseTimer tm(p.prof ? p.prof + kProfRay : nullptr, p.prof != nullptr && threadIdx.x == 32);
      // The CDF of an invalid ray reads weights no compositing wrote: give them a value.
      if (mine)
        for (int k = lane; k < kRowsMax / R; k += 32) scr_w[k] = 0.f;

      // per-ray term of layers_dir.0 of network `pass`: W[:, 256:280] . PE_dir (one output feature per lane and step), read by
      // every step-6 epilogue of the unit's tiles of that network
      auto dir_term = [&](const RayP& rq, int pass, float* dst) {
        const float* wt = p.wd0b_t[pass];
        for (int col = lane; col < 128; col += 32) {
          float acc0 = 0.f;
#pragma unroll 8
          for (int j = 0; j < kDimDir; ++j) acc0 = fmaf(wt[j * 128 + col], rq.ped[j], acc0);
          dst[rr * 128 + col] = acc0;
        }
      };
      // ---- per-ray constants of unit `it`, its direction encoding and its coarse direction term
      auto setup = [&](int it) {
        if (mine) {
          const int unit = blockIdx.x + it * gridDim.x;
          RayP& rp = rayp_all[(it % 3) * 2 + rr];
          if (lane == 0) {
            const int g = geom.ray_index(unit, rr);
            rp.valid = g < geom.n_rays;
            rp.gidx = g;
            if (rp.valid) {
              float o0, o1, o2, d0, d1, d2;
              if (p.o) {
                o0 = p.o[3 * g]; o1 = p.o[3 * g + 1]; o2 = p.o[3 * g + 2];
                d0 = p.d[3 * g]; d1 = p.d[3 * g + 1]; d2 = p.d[3 * g + 2];
              } else {  // get_ray_bundle (nerf_helpers.py:111-122), same operation order in FP32
                const int pj = p.row_begin + g / p.width, pi = g % p.width;
                const float cx = __fdiv_rn(__fsub_rn((float)pi, p.wcx), p.fx);
                const float cy = -__fdiv_rn(__fsub_rn((float)pj, p.hcy), p.fy);
                d0 = __fadd_rn(__fadd_rn(__fmul_rn(cx, p.pose[0]), __fmul_rn(cy, p.pose[1])), __fmul_rn(-1.f, p.pose[2]));
                d1 = __fadd_rn(__fadd_rn(__fmul_rn(cx, p.pose[4]), __fmul_rn(cy, p.pose[5])), __fmul_rn(-1.f, p.pose[6]));
                d2 = __fadd_rn(__fadd_rn(__fmul_rn(cx, p.pose[8]), __fmul_rn(cy, p.pose[9])), __fmul_rn(-1.f, p.pose[10]));
                o0 = p.pose[3]; o1 = p.pose[7]; o2 = p.pose[11];
              }
              rp.o[0] = o0; rp.o[1] = o1; rp.o[2] = o2;
              rp.d[0] = d0; rp.d[1] = d1; rp.d[2] = d2;
              rp.dnorm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2)));
              if (has_bg) { rp.bg[0] = p.bg[3 * g]; rp.bg[1] = p.bg[3 * g + 1]; rp.bg[2] = p.bg[3 * g + 2]; }
              rp.dz = p.dir_z ? p.dir_z[g] : d2;
              if constexpr (MULTI) {  // an index out of range selects the NaN row after the last frame: no out-of-bounds read
                const int f = p.frame[g];
                rp.frame = (f >= 0 && f < p.n_frames) ? f : p.n_frames;
                if (SAVE && p.save_frame) p.save_frame[g] = rp.frame;
              }
              if constexpr (SAVE) {
                p.save_dnorm[g] = rp.dnorm;
                if (p.save_ray) {  // the ray as the input gradients need it: o, d, direction-encoder input
                  float* sr = p.save_ray + 7 * (size_t)g;
                  sr[0] = o0; sr[1] = o1; sr[2] = o2; sr[3] = d0; sr[4] = d1; sr[5] = d2; sr[6] = rp.dz;
                }
              }
            } else {
              for (int k = 0; k < 3; ++k) { rp.o[k] = 0.f; rp.d[k] = 0.f; rp.bg[k] = 0.f; }
              rp.dnorm = 0.f;
              rp.dz = 0.f;
              if constexpr (MULTI) rp.frame = 0;
            }
          }
          __syncwarp();
          // direction encoder input is (d_z, near, far): run_network reads ray_batch[..., -3:] (train_utils.py:14);
          // one accurate sincos per lane
          if (lane < 12) {
            const int f = lane / 3, c = lane - f * 3;
            const float v = (c == 0) ? rp.dz : (c == 1 ? p.near_ : p.far_);
            float sn, cs;
            sincosf(v * (float)(1 << f), &sn, &cs);
            rp.ped[6 * f + c] = rp.valid ? sn : 0.f;
            rp.ped[6 * f + 3 + c] = rp.valid ? cs : 0.f;
          }
          __syncwarp();
          dir_term(rp, 0, dirbias + (it & 1) * 256);
        }
        __syncwarp();
        mbar_arrive(hand.sready(it % 3));
      };
      // ---- compositing of this warp's ray in pass `pass` of unit `it`
      auto composite = [&](int it, int pass, const float4* carry_raw, const float* carry_z) {
        const RayP& rp = rayp_all[(it % 3) * 2 + rr];
        const int S = geom.samples(pass);
        float* dz = pass ? p.dbg_z_f : p.dbg_z_c;  // debug dump of the sample depths
        if (dz && rp.valid)
          for (int i = lane; i < S; i += 32) dz[(size_t)rp.gidx * S + i] = carry_z[rr * S + i];
        if (rp.valid) {
          const int g = rp.gidx;
          float* o_rgb = pass ? p.rgb_f : p.rgb_c;
          float* o_disp = pass ? p.disp_f : p.disp_c;
          float* o_acc = pass ? p.acc_f : p.acc_c;
          const float wl = composite_ray(carry_raw + rr * S, carry_z + rr * S, scr_w, S, rp.dnorm, p.white_bkgd != 0,
                                         o_rgb ? o_rgb + 3 * (size_t)g : nullptr, o_disp ? o_disp + g : nullptr,
                                         o_acc ? o_acc + g : nullptr, lane);
          const bool last_pass = (pass == 1) || (nf == 0);
          if (last_pass && lane == 0 && p.w_last) p.w_last[g] = wl;
        }
        __syncwarp();
      };

      setup(0);
      if (n_iter > 1) setup(1);
      tm.lap(7);
      for (int it = 0; it < n_iter; ++it) {
        const int cb = it % nb;
        const float4* craw = cb ? raw_f : raw_c;
        const float* cz = cb ? z_f : z_c;
        mbar_wait(hand.cdone(cb), (uint32_t)(it / nb) & 1u);
        tm.lap(0);
        if (mine) {
          composite(it, 0, craw, cz);
          tm.lap(1);
          if (nf > 0) {
            // ---- inverse-CDF resampling (nerf_helpers.py:344-387) on weights[1:-1] over the mid-point bins
            const RayP& rp = rayp_all[(it % 3) * 2 + rr];
            const int nb_ = nc - 1;  // bins / cdf entries
            const int nw = nc - 2;   // interior weights
            {
              const float* w = scr_w;
              const float* zc = cz + rr * nc;
              float* cdf = scr_cdf;
              float* bins = scr_bins;
              for (int k = lane; k < nb_; k += 32) bins[k] = __fmul_rn(0.5f, __fadd_rn(zc[k + 1], zc[k]));
              const int per = (nw + 31) >> 5;
              const int k0 = lane * per;
              float part = 0.f;
              for (int j = 0; j < per; ++j)
                if (k0 + j < nw) part += __fadd_rn(w[k0 + j + 1], 1e-5f);
              const float total = warp_sum(part);
              float psum = 0.f;
              for (int j = 0; j < per; ++j)
                if (k0 + j < nw) psum += __fdiv_rn(__fadd_rn(w[k0 + j + 1], 1e-5f), total);
              float incl = psum;
#pragma unroll
              for (int o = 1; o < 32; o <<= 1) {
                const float tt = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += tt;
              }
              float run = incl - psum;  // exclusive prefix of this lane's block
              if (lane == 0) cdf[0] = 0.f;
              for (int j = 0; j < per; ++j)
                if (k0 + j < nw) {
                  run += __fdiv_rn(__fadd_rn(w[k0 + j + 1], 1e-5f), total);
                  cdf[k0 + j + 1] = run;
                }
            }
            __syncwarp();
            tm.lap(2);
            // cat(z_coarse, z_samples) of the ray into scr_sort
            for (int i = lane; i < SF; i += 32) {
              float val;
              if (i < nc) {
                val = cz[rr * nc + i];
              } else {
                const int j = i - nc;
                const float* cdf = scr_cdf;
                const float* bins = scr_bins;
                const float u = p.perturb ? (rp.valid ? p.u_rand[(size_t)rp.gidx * nf + j] : 0.f) : p.u_fine[j];
                int lo = 0, hi = nb_;  // searchsorted(..., right=True): number of cdf entries <= u
                while (lo < hi) {
                  const int mid = (lo + hi) >> 1;
                  if (cdf[mid] <= u) lo = mid + 1; else hi = mid;
                }
                const int below = max(0, lo - 1), above = min(nb_ - 1, lo);
                const float cb_ = cdf[below], ca = cdf[above];
                float den = __fsub_rn(ca, cb_);
                if (den < 1e-5f) den = 1.f;
                const float tt = __fdiv_rn(__fsub_rn(u, cb_), den);
                val = __fadd_rn(bins[below], __fmul_rn(tt, __fsub_rn(bins[above], bins[below])));
              }
              scr_sort[i] = val;
            }
            tm.lap(3);
          }
        }
        __syncwarp();
        mbar_arrive(hand.cfree(cb));  // the coarse carry of unit it is read
        if (nf > 0) {
          if (it > 0) {
            mbar_wait(hand.fdone(), (uint32_t)(it - 1) & 1u);
            tm.lap(4);
            if (mine) composite(it - 1, 1, raw_f, z_f);
            tm.lap(5);
          }
          if (mine) {
            // ---- torch.sort(cat(z, z_samples)) (train_utils.py:126) as a rank merge: the coarse depths are sorted, the
            //      samples need not be (stochastic u), so an element's rank = (# coarse before it, by binary search)
            //      + (# samples before it, counted).  Ties: coarse first, then samples by index — equal values make any
            //      tie order give the same sorted array.  A NaN sample (from non-finite weights) goes after every number,
            //      by index, as torch.sort places it; no comparison with a NaN counts, so the other ranks stay as they are.
            //      When the samples are already sorted and hold no NaN (deterministic u), the same ranks follow from binary
            //      searches alone: # samples < v for a coarse depth, and j itself for sample j.
            __syncwarp();
            bool sorted = true;
            for (int j = lane; j < nf; j += 32) {
              const float y = scr_sort[nc + j];
              sorted = sorted && y == y && (j + 1 == nf || y <= scr_sort[nc + j + 1]);
            }
            sorted = __all_sync(0xffffffffu, sorted);
            for (int i = lane; i < SF; i += 32) {
              const float* zc = scr_sort;
              const float* zs = zc + nc;
              const float v = zc[i];
              int rank;
              if (sorted) {
                const float* a = i < nc ? zs : zc;
                int lo = 0, hi = i < nc ? nf : nc;  // coarse: # samples < v; sample: # coarse depths <= v
                while (lo < hi) {
                  const int mid = (lo + hi) >> 1;
                  if (i < nc ? a[mid] < v : a[mid] <= v) lo = mid + 1; else hi = mid;
                }
                rank = lo + (i < nc ? i : i - nc);
              } else if (i < nc) {
                rank = i;
                for (int j = 0; j < nf; ++j) rank += (zs[j] < v) ? 1 : 0;
              } else if (v != v) {
                const int jm = i - nc;
                rank = nc;
                for (int j = 0; j < nf; ++j) rank += (zs[j] == zs[j] || j < jm) ? 1 : 0;
              } else {
                const int jm = i - nc;
                int lo = 0, hi = nc;  // # coarse depths <= v
                while (lo < hi) {
                  const int mid = (lo + hi) >> 1;
                  if (zc[mid] <= v) lo = mid + 1; else hi = mid;
                }
                rank = lo;
                for (int j = 0; j < nf; ++j) {
                  const float y = zs[j];
                  rank += (y < v || (y == v && j < jm)) ? 1 : 0;
                }
              }
              z_f[rr * SF + rank] = v;
            }
            tm.lap(6);
            dir_term(rayp_all[(it % 3) * 2 + rr], 1, dirbias + 512);
          }
          __syncwarp();
          mbar_arrive(hand.fready());
        }
        if (it + 2 < n_iter) setup(it + 2);
        tm.lap(7);
      }
      if (nf > 0) {
        mbar_wait(hand.fdone(), (uint32_t)(n_iter - 1) & 1u);
        tm.lap(4);
        if (mine) composite(n_iter - 1, 1, raw_f, z_f);
        tm.lap(5);
      }
    }
  } else {
    // ============================== row warps ==============================
    reg_inc<kRegsRenderRow>();
    const int q = warp & 3;
    const int wg = (warp - 4) >> 2;        // row warpgroup: tile rows [64 wg, 64 wg + 64)
    const int etid = wg * 128 + q * 32 + lane;  // 0..255
    // per-tile row stages (prologue, post-processing): the warpgroup's own rows, two threads per row, one PE half each
    const int half = q >> 1;
    const int row = 64 * wg + (q & 1) * 32 + lane;
    const int g = 16 * q + (lane >> 2);  // MLP: first of this thread's two accumulator rows within the warpgroup's 64
    const int r0 = 64 * wg + g;          // ... as a tile row (the other one is r0 + 8)
    uint8_t* pe_hi = smem + M::kPeHi;
    uint8_t* pe_lo = smem + M::kPeLo;
    uint8_t* act_hi = smem + M::kActHi;
    uint8_t* act_lo = smem + M::kActLo;
    float4* tile_raw = reinterpret_cast<float4*>(smem + M::kTileRaw);
    const bool has_bg = p.bg != nullptr;
    // observers: the first thread of each row warpgroup, warpgroup w's laps at slot + kProfWgStride * w
    PhaseTimer tm(p.prof ? p.prof + kProfWgStride * wg : nullptr, p.prof != nullptr && (etid & 127) == 0);

    for (int k = 0; k < n_stream; ++k) {
      const StreamTile stile = stream_tile(geom, n_iter, k);
      const int it = stile.it, pass = stile.pass, t = stile.t;
      const int unit = blockIdx.x + it * gridDim.x;
      const int S = geom.samples(pass);
      const int n_tiles = geom.tile_count(pass);
      const float* bias_n = EXACT ? p.bias[pass] : sbias + pass * kBiasFloats;
      const int cb = it % nb;
      float4* carry_raw = (pass || cb) ? raw_f : raw_c;
      float* carry_z = (pass || cb) ? z_f : z_c;
      const RayP* rayp = rayp_all + (it % 3) * 2;
      const float* dirb = dirbias + (pass ? 512 : (it & 1) * 256);  // [ray][128]
      if (t == 0) {  // the pass's inputs from the ray warps, and its carry buffer free
        if (pass == 0) {
          mbar_wait(hand.sready(it % 3), (uint32_t)(it / 3) & 1u);
          if (it >= nb) mbar_wait(hand.cfree(cb), (uint32_t)((it - nb) / nb) & 1u);
        } else {
          mbar_wait(hand.fready(), (uint32_t)it & 1u);
        }
        tm.lap(16);
      }

      // ---- prologue of tile t: sample depth + positional encoding -> PE buffer.
      auto prologue = [&](int t) {
        const TileGeom::Row rw = geom.row(pass, t, row);
        const int prow = rw.pass_row, i = rw.sample;
        const bool live = rw.used;
        const RayP& rp = rayp[rw.ray];
        float z = 0.f;
        if (live) {
          if (pass == 0) {
            const float tc = p.t_coarse[i];
            z = __fadd_rn(__fmul_rn(p.near_, __fsub_rn(1.f, tc)), __fmul_rn(p.far_, tc));
            if (p.perturb) {  // stratified jitter (train_utils.py:69-76)
              float lower = z, upper = z;
              if (i > 0) {
                const float tp = p.t_coarse[i - 1];
                const float zp = __fadd_rn(__fmul_rn(p.near_, __fsub_rn(1.f, tp)), __fmul_rn(p.far_, tp));
                lower = __fmul_rn(0.5f, __fadd_rn(z, zp));
              }
              if (i < S - 1) {
                const float tn = p.t_coarse[i + 1];
                const float zn = __fadd_rn(__fmul_rn(p.near_, __fsub_rn(1.f, tn)), __fmul_rn(p.far_, tn));
                upper = __fmul_rn(0.5f, __fadd_rn(zn, z));
              }
              const float tr = rp.valid ? p.t_rand[(size_t)rp.gidx * geom.nc + i] : 0.f;
              z = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), tr));
            }
            if (half == 0) carry_z[prow] = z;
          } else {
            z = carry_z[prow];
          }
        }
        // positional encoding of o + d*z: 63 lanes + 1 zero pad, FP16 (hi[,lo]) into the swizzled PE buffer.
        // The two threads of a row write lanes [0,32) and [32,64) respectively.
        const float px = __fadd_rn(rp.o[0], __fmul_rn(rp.d[0], z));
        const float py = __fadd_rn(rp.o[1], __fmul_rn(rp.d[1], z));
        const float pz = __fadd_rn(rp.o[2], __fmul_rn(rp.d[2], z));
        float f[32];
        if (half == 0) {  // lanes 0..31: xyz, frequencies 0..3, sin of frequency 4, cos(x), cos(y) of frequency 4
          f[0] = px; f[1] = py; f[2] = pz;
#pragma unroll
          for (int fr = 0; fr < 4; ++fr) {
            const float sc = (float)(1 << fr);
            pe_sincos<EXACT>(px * sc, f[3 + 6 * fr + 0], f[3 + 6 * fr + 3]);
            pe_sincos<EXACT>(py * sc, f[3 + 6 * fr + 1], f[3 + 6 * fr + 4]);
            pe_sincos<EXACT>(pz * sc, f[3 + 6 * fr + 2], f[3 + 6 * fr + 5]);
          }
          float cz;
          pe_sincos<EXACT>(px * 16.f, f[27], f[30]);
          pe_sincos<EXACT>(py * 16.f, f[28], f[31]);
          pe_sincos<EXACT>(pz * 16.f, f[29], cz);
        } else {          // lanes 32..63: cos(z) of frequency 4, frequencies 5..9, zero pad
          float sz;
          pe_sincos<EXACT>(pz * 16.f, sz, f[0]);
#pragma unroll
          for (int fr = 5; fr < 10; ++fr) {
            const float sc = (float)(1 << fr);
            const int b = 6 * fr - 29;  // lane 3 + 6*fr, minus 32
            pe_sincos<EXACT>(px * sc, f[b + 0], f[b + 3]);
            pe_sincos<EXACT>(py * sc, f[b + 1], f[b + 4]);
            pe_sincos<EXACT>(pz * sc, f[b + 2], f[b + 5]);
          }
          f[31] = 0.f;
        }
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float a = f[qq * 8 + 2 * e], b = f[qq * 8 + 2 * e + 1];
            hi[e] = pack_f16x2(a, b);
            if constexpr (EXACT) {
              const float2 hf = unpack_f16x2(hi[e]);
              lo[e] = pack_f16x2(a - hf.x, b - hf.y);
            }
          }
          const int off = row * 128 + (((half * 4 + qq) ^ (row & 7)) << 4);
          *reinterpret_cast<uint4*>(pe_hi + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          if constexpr (EXACT) *reinterpret_cast<uint4*>(pe_lo + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        if (PROBE && p.dbg_act && p.dbg_act_step == -1 && unit == 0 && pass == 0 && t == 0) {
#pragma unroll
          for (int k = 0; k < 32; ++k) p.dbg_act[row * 256 + half * 32 + k] = f[k];
        }
        if constexpr (SAVE) {  // FP16 encoding of this tile as a transposed image (input of layers_xyz.0 / .3 in dW)
          if (unit < geom.n_units) {
            uint8_t* rec = p.save_rec + geom.global_tile(unit, pass, t) * kRecStride;
            uint32_t hh[16];
#pragma unroll
            for (int e = 0; e < 16; ++e) hh[e] = pack_f16x2(f[2 * e], f[2 * e + 1]);
            store_t32(rec + kRecPE + img_row_base(64, row), row, 32 * half, hh);
            if constexpr (HILO) {  // the lo half the PE buffer's lo atom holds
#pragma unroll
              for (int e = 0; e < 16; ++e) {
                const float2 hf = unpack_f16x2(hh[e]);
                hh[e] = pack_f16x2(f[2 * e] - hf.x, f[2 * e + 1] - hf.y);
              }
              store_t32(rec + kRecBytes + kRecPE + img_row_base(64, row), row, 32 * half, hh);
            }
          }
        }
        fence_proxy_async_smem();  // make the generic-proxy PE stores visible to the tensor core
      };


      {
        prologue(t);
        uint8_t* rec = nullptr;  // this tile's training record (SAVE mode)
        if constexpr (SAVE) {
          if (unit < geom.n_units) {
            const TileGeom::Row rw = geom.row(pass, t, row);
            const bool live = rw.used;
            const RayP& rp = rayp[rw.ray];
            rec = p.save_rec + geom.global_tile(unit, pass, t) * kRecStride;
            uint32_t hh[8];  // direction encoding of this row's ray: features [16*half, 16*half+16)
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int k = 16 * half + 2 * e;
              const float a = (live && rp.valid && k < kDimDir) ? rp.ped[k] : 0.f;
              const float b = (live && rp.valid && k + 1 < kDimDir) ? rp.ped[k + 1] : 0.f;
              hh[e] = pack_f16x2(a, b);
            }
            uint8_t* img = rec + kRecPEd + img_row_base(32, row);
            const uint32_t cr = (uint32_t)((row & 63) >> 3);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int ka = 16 * half + 2 * e, kb = ka + 1;
              *reinterpret_cast<uint16_t*>(img + ka * 128 + ((cr ^ (uint32_t)(ka & 7)) << 4)) = (uint16_t)(hh[e] & 0xFFFFu);
              *reinterpret_cast<uint16_t*>(img + kb * 128 + ((cr ^ (uint32_t)(kb & 7)) << 4)) = (uint16_t)(hh[e] >> 16);
            }
            if constexpr (HILO) {
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                const int ka = 16 * half + 2 * e, kb = ka + 1;
                const float a = (live && rp.valid && ka < kDimDir) ? rp.ped[ka] : 0.f;
                const float b = (live && rp.valid && kb < kDimDir) ? rp.ped[kb] : 0.f;
                const float2 hf = unpack_f16x2(hh[e]);
                const uint32_t l = pack_f16x2(a - hf.x, b - hf.y);
                *reinterpret_cast<uint16_t*>(img + kRecBytes + ka * 128 + ((cr ^ (uint32_t)(ka & 7)) << 4)) = (uint16_t)(l & 0xFFFFu);
                *reinterpret_cast<uint16_t*>(img + kRecBytes + kb * 128 + ((cr ^ (uint32_t)(kb & 7)) << 4)) = (uint16_t)(l >> 16);
              }
            }
          }
        }
        // this warpgroup's PE rows complete.  Nothing else inside the tile is shared between the warpgroups: each reads
        // and writes only its own 64 rows of the PE buffer, the activation buffers, tile_raw and the carry buffers.
        named_bar_sync(2 + wg, 128);
        tm.lap(2);

        // ---- the MLP: this warpgroup's 64 rows
        {
          const bool probe = PROBE && p.dbg_act && unit == 0 && pass == 0 && t == 0;
          float acc0[64], acc1[64], acc_s[8];
          uint32_t act[64];  // fast mode: this thread's part of the hidden activations, as the next step's A fragments
          const TileGeom::Row rw0 = geom.row(pass, t, r0), rw1 = geom.row(pass, t, r0 + 8);
          const int ray0 = rw0.ray, ray1 = rw1.ray;
          uint32_t live = 0u;  // SAVE: which of this thread's two rows hold a sample (see epi_half)
          if constexpr (SAVE) live = ((rw0.used && rayp[ray0].valid) ? 1u : 0u) | ((rw1.used && rayp[ray1].valid) ? 2u : 0u);
          auto mlp_step = [&](auto step) {
            const int s = step;
            const StepInfo si = step_info(s);
            // Fast mode staggers the warpgroups (ping-pong): warpgroup 1 issues step s after warpgroup 0 has issued it, and
            // warpgroup 0 issues step s + 1 after warpgroup 1 has issued step s, so one's epilogue runs under the other's
            // MMAs.  Barrier 4 + w is the one warpgroup w waits on.  The pairs close over the CTA's tile stream: warpgroup 0
            // does not wait before its first step, warpgroup 1 does not arrive after its last.  Exact mode's one-slot ring
            // already keeps the warpgroups within one unit of each other, and a forced order there would deadlock it.
            const bool pp_wait = !EXACT && (wg == 1 || s > 0 || k > 0);
            const bool pp_arrive = !EXACT && (wg == 0 || s < kNumSteps - 1 || k < n_stream - 1);
            if (pp_wait) named_bar_sync(4 + wg, 256);
            tm.lap(15);
            auto issued = [&] { if (pp_arrive) named_bar_arrive(5 - wg, 256); };
            mlp_step_mma<EXACT>(step, ring, smem_base + M::kActHi, smem_base + M::kActLo, smem_base + M::kPeHi,
                                smem_base + M::kPeLo, (uint32_t)(64 * wg * 128), act, acc0, acc1, acc_s, tm, issued);
            float* dump = (probe && p.dbg_act_step == s) ? p.dbg_act : nullptr;
            const float* bias = bias_n + si.bias_off;
            if (s <= 8) {
              const float* db0 = (s == 6) ? dirb + ray0 * 128 : nullptr;
              const float* db1 = (s == 6) ? dirb + ray1 * 128 : nullptr;
              if constexpr (MULTI) {
                // steps 0 and 3, whose bias carries the conditioning fold: the rows of the frames of this thread's two
                // accumulator rows (step 0 at +0, step 3 at +256), looked up here rather than held in registers across the tile.
                // In fast mode (steps unrolled) the other steps run the single-frame epilogue.  Exact mode's steps are a runtime
                // loop: there one row-bias epilogue serves every step (b0 == b1 outside steps 0 and 3), since a second copy of the
                // epilogue in the loop costs registers (ptxas: 40 bytes of spill in the training forward).
                if (EXACT || s == 0 || s == 3) {
                  const bool cond = s == 0 || s == 3;
                  const float* fb = p.fbias[pass] + (s == 3 ? 256 : 0);
                  const float* b0 = cond ? fb + (size_t)rayp[ray0].frame * kFrameRows : bias;
                  const float* b1 = cond ? fb + (size_t)rayp[ray1].frame * kFrameRows : bias;
                  epi_half<EXACT, SAVE, PROBE, true, HILO>(acc0, s, 0, b0, db0, db1, act_hi, act_lo, act, r0, rec, live, dump, b1);
                  if (si.nh1 == 128)
                    epi_half<EXACT, SAVE, PROBE, true, HILO>(acc1, s, 128, b0, nullptr, nullptr, act_hi, act_lo, act, r0, rec, live, dump, b1);
                } else {
                  epi_half<EXACT, SAVE, PROBE, false, HILO>(acc0, s, 0, bias, db0, db1, act_hi, act_lo, act, r0, rec, live, dump);
                  if (si.nh1 == 128)
                    epi_half<EXACT, SAVE, PROBE, false, HILO>(acc1, s, 128, bias, nullptr, nullptr, act_hi, act_lo, act, r0, rec, live, dump);
                }
              } else {
                epi_half<EXACT, SAVE, PROBE, false, HILO>(acc0, s, 0, bias, db0, db1, act_hi, act_lo, act, r0, rec, live, dump);
                if (si.nh1 == 128)
                  epi_half<EXACT, SAVE, PROBE, false, HILO>(acc1, s, 128, bias, nullptr, nullptr, act_hi, act_lo, act, r0, rec, live, dump);
              }
              if (s == 6 && (lane & 3) == 0) {  // sigma = first column of the 16-column half
                const float b = bias[128];
                tile_raw[r0].w = acc_s[0] + b;
                tile_raw[r0 + 8].w = acc_s[2] + b;
              }
              if constexpr (EXACT) {
                fence_proxy_async_smem();  // generic-proxy activation stores -> the next step's wgmma
                named_bar_sync(2 + wg, 128);
              }
            } else {  // fc_rgb: raw colour of columns 0..2
              const int c = lane & 3;
              if (c == 0) {
                tile_raw[r0].x = acc_s[0] + bias[0]; tile_raw[r0].y = acc_s[1] + bias[1];
                tile_raw[r0 + 8].x = acc_s[2] + bias[0]; tile_raw[r0 + 8].y = acc_s[3] + bias[1];
              } else if (c == 1) {
                tile_raw[r0].z = acc_s[0] + bias[2];
                tile_raw[r0 + 8].z = acc_s[2] + bias[2];
              }
            }
            tm.lap(12);
          };
          if constexpr (EXACT) {
#pragma unroll 1
            for (int s = 0; s < kNumSteps; ++s) mlp_step(s);
          } else {
            static_for<0, kNumSteps>(mlp_step);
          }
        }
        named_bar_sync(2 + wg, 128);  // this warpgroup's rows of tile_raw complete
        tm.lap(14);
        // fc_rgb output.  Prepare what compositing needs per sample: colour and sigma (volume_rendering_utils.py:29-33,
        // 41-53); the exp(-sigma*delta) needs the neighbour depth and stays in composite_ray.  One thread per row of the
        // warpgroup's 64.
        if (half == 0) {
          const TileGeom::Row rw = geom.row(pass, t, row);
          const int prow = rw.pass_row, i = rw.sample;
          const RayP& rp = rayp[rw.ray];
          if (rw.used) {
            const float4 v = tile_raw[row];
            const float r0_ = v.x, r1 = v.y, r2 = v.z, sigma_raw = v.w;
            if (rp.valid) {
              float* dr = pass ? p.dbg_raw_f : p.dbg_raw_c;
              if (dr) reinterpret_cast<float4*>(dr)[(size_t)rp.gidx * S + i] = make_float4(r0_, r1, r2, sigma_raw);
            }
            float sig = sigma_raw;
            if (p.noise_std > 0.f && rp.valid)
              sig = __fadd_rn(sig, __fmul_rn((pass ? p.noise_f : p.noise_c)[(size_t)rp.gidx * S + i], p.noise_std));
            const float sig_in = sig;  // what the ReLU sees (volume_rendering_utils.py:52)
            sig = relu_nan(sig);
            float4 pre;
            if (i == S - 1) {
              sig = __fadd_rn(sig, 1e-6f);
              if (has_bg) { pre.x = rp.bg[0]; pre.y = rp.bg[1]; pre.z = rp.bg[2]; }
            }
            if (!(has_bg && i == S - 1)) {
              pre.x = 1.f / (1.f + expf(-r0_));
              pre.y = 1.f / (1.f + expf(-r1));
              pre.z = 1.f / (1.f + expf(-r2));
            }
            pre.w = sig;
            carry_raw[prow] = pre;
            if constexpr (SAVE) {  // what the compositing backward needs: colour (or bg) and the ReLU input
              if (rp.valid) reinterpret_cast<float4*>(pass ? p.save_raw_f : p.save_raw_c)[(size_t)rp.gidx * S + i] = make_float4(pre.x, pre.y, pre.z, sig_in);
            }
          }
        }
        tm.lap(13);
        if (t == n_tiles - 1) mbar_arrive(pass ? hand.fdone() : hand.cdone(cb));  // the pass's carry complete
      }
    }  // tile stream
  }
}

template <bool EXACT, bool SAVE, bool PROBE>
__global__ void __launch_bounds__(kThreads, 1) render_kernel(const __grid_constant__ RenderParams p) {
  render_body<EXACT, SAVE, PROBE, false>(p);
}
// The multi-frame instantiations: a kernel of their own (not a fourth template parameter of render_kernel), so that each
// single-frame instantiation keeps its name and its code.  No probe instantiation.
template <bool EXACT, bool SAVE>
__global__ void __launch_bounds__(kThreads, 1) render_frames_kernel(const __grid_constant__ RenderParams p) {
  render_body<EXACT, SAVE, false, true>(p);
}

// The exact-grad training forwards (NFB_PREC_EXACT_GRAD): kernels of their own, so the other instantiations keep their names
// and code.  MULTI: the multi-frame one.
template <bool MULTI>
__global__ void __launch_bounds__(kThreads, 1) render_hilo_kernel(const __grid_constant__ RenderParams p) {
  render_body<true, true, false, MULTI, true>(p);
}
template <class Kernel>
static cudaError_t smem_opt_in(Kernel* kernel, int bytes) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}
// The training forward takes no debug dumps (nfb_render_forward_train), and a multi-frame call none at all, so only the
// single-frame evaluation kernels have a probe instantiation.
template <bool EXACT, bool SAVE>
static void render_launch(const RenderParams& p, bool probe, bool multi, int grid, cudaStream_t st) {
  constexpr int kBytes = SmemMap<EXACT>::kBytes;
  if (multi) render_frames_kernel<EXACT, SAVE><<<grid, kThreads, kBytes, st>>>(p);
  else if (!SAVE && probe) render_kernel<EXACT, false, true><<<grid, kThreads, kBytes, st>>>(p);
  else render_kernel<EXACT, SAVE, false><<<grid, kThreads, kBytes, st>>>(p);
}

cudaError_t render_kernel_setup() {
  constexpr int B = SmemMap<true>::kBytes, F = SmemMap<false>::kBytes;
  const cudaError_t e[12] = {smem_opt_in(render_kernel<false, false, false>, F), smem_opt_in(render_kernel<true, false, false>, B),
                             smem_opt_in(render_kernel<false, true, false>, F),  smem_opt_in(render_kernel<true, true, false>, B),
                             smem_opt_in(render_kernel<false, false, true>, F),  smem_opt_in(render_kernel<true, false, true>, B),
                             smem_opt_in(render_frames_kernel<false, false>, F), smem_opt_in(render_frames_kernel<true, false>, B),
                             smem_opt_in(render_frames_kernel<false, true>, F),  smem_opt_in(render_frames_kernel<true, true>, B),
                             smem_opt_in(render_hilo_kernel<false>, B),          smem_opt_in(render_hilo_kernel<true>, B)};
  for (const cudaError_t x : e)
    if (x != cudaSuccess) return x;
  return cudaSuccess;
}

cudaError_t launch_render(const RenderParams& p, int precision, int num_sms, cudaStream_t st, long long* launches) {
  const int grid = p.geom.n_units < num_sms ? p.geom.n_units : num_sms;
  if (grid <= 0) return cudaSuccess;
  const bool save = p.save_rec != nullptr;  // training forward: also writes the per-tile activation records
  const bool probe = p.dbg_act != nullptr;  // the activation probe (evaluation only): its own instantiation
  const bool multi = p.frame != nullptr;    // multi-frame call: render_frames_kernel / render_hilo_kernel<true>
  if (precision == 2 && save) {
    if (multi) render_hilo_kernel<true><<<grid, kThreads, SmemMap<true>::kBytes, st>>>(p);
    else render_hilo_kernel<false><<<grid, kThreads, SmemMap<true>::kBytes, st>>>(p);
  } else if (precision != 0) {  // exact, and the evaluation renders of exact-grad mode
    if (save) render_launch<true, true>(p, probe, multi, grid, st);
    else render_launch<true, false>(p, probe, multi, grid, st);
  } else {
    if (save) render_launch<false, true>(p, probe, multi, grid, st);
    else render_launch<false, false>(p, probe, multi, grid, st);
  }
  ++*launches;
  return cudaGetLastError();
}

}  // namespace nfb
