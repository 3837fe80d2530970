// nfb_pipeline.cuh — the warp-specialised pipeline of the three wgmma kernels (render_kernel, chain::chain_kernel,
// dw::dw_kernel): the thread roles, the register split between them, and the ring of shared-memory slots that the producer
// warp fills with bulk copies and the consumer warpgroups drain, under full / empty mbarriers.
//
// Roles (384 threads): warpgroup 0 is the producer side (warp 0 issues the copies; warps 1..3 idle, except in render_kernel,
// where they run the per-ray stages), warpgroups 1 and 2 are
// the consumers ("row" warps), each issuing the wgmma of 64 tile rows.  The register file is re-partitioned per warpgroup.
#pragma once
#include <stdint.h>

#include "nfb_ptx.cuh"

namespace nfb {

constexpr int kThreads = 384;        // producer warpgroup + 2 consumer warpgroups
constexpr int kRowThreads = 256;     // the two consumer warpgroups
constexpr int kRayThreads = 96;      // render_kernel: warps 1..3 of the producer warpgroup, its per-ray stages
constexpr uint32_t kRowBarrier = 1;  // named barrier id of the eight consumer warps; 2 + w: warpgroup w alone (render_kernel: 4 + w, its MMA ping-pong)
constexpr int kRegsLight = 40, kRegsRow = 232;
static_assert((4 * kRegsLight + 8 * kRegsRow) * 32 <= 65536, "register file");
// render_kernel's producer warpgroup also runs the per-ray stages (warps 1..3), which spill at 40 registers.  setmaxnreg.inc
// takes registers only from those the CTA's other warps released, so a split must fit the kernel's own allocation (384
// threads x 168 registers under __launch_bounds__(384, 1)), not just the register file: the row warps give up 8.
constexpr int kRegsRenderLight = 56, kRegsRenderRow = 224;
static_assert(4 * kRegsLight + 8 * kRegsRow <= 12 * 168 && 4 * kRegsRenderLight + 8 * kRegsRenderRow <= 12 * 168,
              "a register split must fit the 168 registers per thread a 384-thread kernel is compiled for");
template <int N> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// Shared address of the dynamic shared memory.  Swizzled wgmma operands need a 1024-byte-aligned base: trap otherwise.
__device__ __forceinline__ uint32_t smem_base_aligned(const uint8_t* smem) {
  const uint32_t base = smem_u32(smem);
  if ((base & 1023u) != 0u) __trap();
  return base;
}

// A ring of SLOTS shared-memory slots, STRIDE bytes apart from `base`, with a full and an empty mbarrier per slot at `bars`
// (2 * SLOTS * 8 bytes).  Every thread keeps its own copy of the position (slot, phase); the producer warp and every consumer
// warp walk the slots in the same order.  A consumer has two cursors: `slot` (the next slot to wait on) and `rel` (the oldest
// slot it has read but not yet released), so it may hold up to kLag + 1 slots: it issues the MMAs of unit u + 1 before it
// waits for those of unit u and releases u's slot.  With one slot there is nothing to read ahead into, so kLag = 0.
template <int SLOTS, int STRIDE>
struct Ring {
  static constexpr int kLag = SLOTS >= 2 ? 1 : 0;
  uint32_t base, bars;
  uint32_t slot = 0, phase = 0;
  uint32_t rel = 0;

  __device__ __forceinline__ Ring(uint32_t base_, uint32_t bars_) : base(base_), bars(bars_) {}

  // One thread, before the block-wide barrier that precedes any use.  full: one arrival (the producer's expect_tx);
  // empty: one arrival per consumer warp.
  __device__ __forceinline__ void init() const {
    for (int i = 0; i < SLOTS; ++i) {
      mbar_init(full_bar(i), 1);
      mbar_init(empty_bar(i), kRowThreads / 32);
    }
    mbar_fence_init();
  }

  // Producer, the whole warp (warp-uniform control flow): wait for the current slot to be free, then one elected lane arms
  // its full barrier for the bytes of the copies and issues them.  One copy of `bytes` to the slot start ...
  __device__ __forceinline__ void produce(const void* src, uint32_t bytes) {
    fill(bytes, [&](uint32_t dst, uint32_t bar) { bulk_g2s(dst, src, bytes, bar); });
  }
  // ... or two: `bytes0` to the slot start and `bytes1` to offset `off1`, completing one slot.
  __device__ __forceinline__ void produce(const void* src0, uint32_t bytes0, uint32_t off1, const void* src1, uint32_t bytes1) {
    fill(bytes0 + bytes1, [&](uint32_t dst, uint32_t bar) {
      bulk_g2s(dst, src0, bytes0, bar);
      bulk_g2s(dst + off1, src1, bytes1, bar);
    });
  }

  // Consumer, the whole warp: wait until the next slot is full; returns its shared address.
  __device__ __forceinline__ uint32_t wait_full() {
    mbar_wait(full_bar(slot), phase);
    const uint32_t addr = base + slot * STRIDE;
    advance();
    return addr;
  }
  // Consumer, the whole warp, once this warp's reads of the oldest unreleased slot are complete (its wgmma waited on): one
  // lane releases that slot to the producer.
  __device__ __forceinline__ void release() {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(empty_bar(rel));
    if (++rel == SLOTS) rel = 0;
  }

 private:
  __device__ __forceinline__ uint32_t full_bar(uint32_t i) const { return bars + i * 8; }
  __device__ __forceinline__ uint32_t empty_bar(uint32_t i) const { return bars + (SLOTS + i) * 8; }
  __device__ __forceinline__ void advance() {
    if (++slot == SLOTS) { slot = 0; phase ^= 1; }
  }
  template <class Copies>
  __device__ __forceinline__ void fill(uint32_t bytes, Copies copies) {
    mbar_wait(empty_bar(slot), phase ^ 1);
    if (elect_one()) {
      mbar_arrive_expect_tx(full_bar(slot), bytes);
      copies(base + slot * STRIDE, full_bar(slot));
    }
    __syncwarp();
    advance();
  }
};

}  // namespace nfb
