// nfb_layout.h — the MLP as the kernel executes it: 10 tensor-core "steps", each a GEMM
//   D[128 rows, N] = A[128 rows, K] * W[N, K]^T   (FP16 operands, FP32 accumulate in registers)
// and the byte layout of the packed weight streams (forward and backward chain) the kernels bulk-copy into shared memory,
// with the per-tile unit program they follow through them.  Shared by host (packing, tests) and device code.
//
// Reference model: ConditionalBlendshapePaperNeRFModel.forward (nerf/models.py:236-261).  Exact
// algebra applied at load / per frame (SURVEY.md §8 a''):
//   * the 108 expression/latent columns of layers_xyz.0 and layers_xyz.3 multiply a per-frame constant
//     vector -> folded into those layers' biases (nfb_set_frame);
//   * fc_feat has no activation -> pre-multiplied into fc_alpha and layers_dir.0[:, :256] (FP64 fold);
//   * the 24 direction-encoding columns of layers_dir.0 depend on the ray only -> a per-ray bias.
//
//   step  reference layer            N (half 0 + half 1)  K (atoms of 64)            A operand
//   0     layers_xyz.0               128 + 128            64  = PE(63)+pad           SMEM (PE buffer)
//   1,2   layers_xyz.1,2             128 + 128            256                        SMEM (activations)
//   3     layers_xyz.3               128 + 128            320 = PE(63)+pad | h(256)  SMEM atom + activations
//   4,5   layers_xyz.4,5             128 + 128            256                        SMEM (activations)
//   6     layers_dir.0∘fc_feat | σ   128 + 16 (σ)         256                        SMEM (activations)
//   7,8   layers_dir.1,2             128                  128                        SMEM (activations)
//   9     fc_rgb                     16 (3 used)          128                        SMEM (activations)
//
// A weight "unit" = all N rows of the step x one 64-wide K atom (<= 32 KB), consumed by 4 wgmma (M=64 per warpgroup, N, K=16).
// The accumulator is kept in two column halves ("half 0" = output columns [0,128) = K atoms 0,1 of the next step,
// "half 1" = [128,256) = atoms 2,3), one m64n128 (or n16) wgmma accumulator each.
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define NFB_HD __host__ __device__
#else
#define NFB_HD
#endif

namespace nfb {

constexpr int kTileM = 128;      // rows (samples) per tensor-core tile (two warpgroups of 64)
constexpr int kAtomK = 64;       // fp16 elements per 128-byte swizzle row
constexpr int kNumSteps = 10;
constexpr int kMaxUnitBytes = 256 * 128;  // one weight unit: <=256 output rows x 64 K x 2 B
constexpr int kDimXyz = 63, kDimDir = 24, kDimExpr = 76, kDimLatent = 32, kDimCond = 108;

struct StepInfo {
  int16_t nh0, nh1;   // output columns (= MMA N) of half 0 / half 1; nh1 == 0: single half
  int16_t k_atoms;    // K / 64 including the PE atom
  int16_t pe_first;   // 1: the first K atom is the positional encoding (A from shared memory)
  int16_t bias_off;   // float offset of this step's bias vector in the per-network bias block
  int16_t n_bias;     // bias floats
};

NFB_HD constexpr StepInfo step_info(int s) {
  return s == 0   ? StepInfo{128, 128, 1, 1, 0, 256}
         : s == 1 ? StepInfo{128, 128, 4, 0, 256, 256}
         : s == 2 ? StepInfo{128, 128, 4, 0, 512, 256}
         : s == 3 ? StepInfo{128, 128, 5, 1, 768, 256}
         : s == 4 ? StepInfo{128, 128, 4, 0, 1024, 256}
         : s == 5 ? StepInfo{128, 128, 4, 0, 1280, 256}
         : s == 6 ? StepInfo{128, 16, 4, 0, 1536, 144}
         : s == 7 ? StepInfo{128, 0, 2, 0, 1680, 128}
         : s == 8 ? StepInfo{128, 0, 2, 0, 1808, 128}
                  : StepInfo{16, 0, 2, 0, 1936, 16};
}
constexpr int kBiasFloats = 1952;  // 6*256 + 144 + 128 + 128 + 16
// Multi-frame conditioning: per (network, frame) the folded bias rows of step 0 (256) then of step 3 (256); nfb.h NFB_MAX_FRAMES frames.
constexpr int kFrameRows = 512;
constexpr int kMaxFrames = 1024;

// Byte offset of element (row n, k in [0,64)) inside one swizzled unit: 128-byte rows, 16-byte chunks
// XORed with (row & 7) — the SWIZZLE_128B pattern the wgmma shared-memory descriptor expects.
NFB_HD constexpr int sw128_offset(int n, int k) { return n * 128 + ((((k >> 3) ^ (n & 7)) & 7) << 4) + ((k & 7) << 1); }

// ------------------------------------------------------------------------------------------------
// How a call's rays are cut into work.  A unit is R = rays_per_unit consecutive rays (two when both fit the 512 sample rows a
// unit's pass may hold, else one).  A unit's pass p (0 coarse, 1 fine; network p evaluates it) is the R * samples(p) rows
// "ray rr, sample i" -> rr * samples(p) + i, cut into 128-row tiles; a unit's tiles are its coarse ones, then its fine ones,
// and units follow each other.  Every per-tile array (the activation records, d raw, the input-gradient rows) is indexed by
// that global tile.  The only definition: the kernels that write such an array and the ones that read it all ask here.
struct TileGeom {
  int n_rays, nc, nf;      // rays of the launch; coarse samples per ray; additional fine samples per ray (0: no fine pass)
  int rays_per_unit;       // R
  int tiles_c, tiles_f;    // 128-row tiles per coarse / fine pass of one unit
  int n_units;

  static NFB_HD constexpr TileGeom make(int n_rays, int nc, int nf) {
    const int R = 2 * (nc + nf) <= 512 ? 2 : 1;
    return TileGeom{n_rays, nc, nf, R, (R * nc + kTileM - 1) / kTileM, nf > 0 ? (R * (nc + nf) + kTileM - 1) / kTileM : 0,
                    (n_rays + R - 1) / R};
  }
  // The same cut for a chunk of n of the rays (a chunk that starts at a multiple of R holds whole units of the full call).
  NFB_HD constexpr TileGeom chunk(int n) const { return make(n, nc, nf); }

  NFB_HD constexpr int passes() const { return nf > 0 ? 2 : 1; }
  NFB_HD constexpr int samples(int pass) const { return pass ? nc + nf : nc; }
  NFB_HD constexpr int tile_count(int net) const { return net ? tiles_f : tiles_c; }
  NFB_HD constexpr int tile_base(int net) const { return net ? tiles_c : 0; }  // first tile of the network within a unit
  NFB_HD constexpr int tiles_per_unit() const { return tiles_c + tiles_f; }
  NFB_HD constexpr size_t tiles() const { return (size_t)n_units * tiles_per_unit(); }
  NFB_HD constexpr int net_of(int unit_tile) const { return unit_tile < tiles_c ? 0 : 1; }  // unit_tile in [0, tiles_per_unit)
  NFB_HD constexpr size_t global_tile(int unit, int unit_tile) const { return (size_t)unit * tiles_per_unit() + unit_tile; }
  NFB_HD constexpr size_t global_tile(int unit, int net, int local_tile) const { return global_tile(unit, tile_base(net) + local_tile); }
  // Index of sample i of ray g in pass `pass` within a [tiles][128] array: row (prow & 127) of the pass's tile (prow >> 7),
  // prow = rr * samples(pass) + i for ray rr of the unit.  A kernel that sweeps a ray's samples asks for ray_rows once.
  struct RayRows {
    int tile0, rr, S;  // global tile of the unit's pass, ray within the unit, samples per ray
    NFB_HD constexpr size_t slot(int i) const { return (size_t)(tile0 + ((rr * S + i) >> 7)) * 128 + ((rr * S + i) & 127); }
  };
  NFB_HD constexpr RayRows ray_rows(int pass, int g) const {
    const int unit = g / rays_per_unit;
    return RayRows{(int)global_tile(unit, pass, 0), g - unit * rays_per_unit, samples(pass)};
  }
  NFB_HD constexpr size_t slot(int pass, int g, int i) const { return ray_rows(pass, g).slot(i); }
  // The inverse for one row of a tile.  used: the row holds a sample of one of the unit's R rays (else ray = sample = 0);
  // whether that ray exists is ray_index(unit, ray) < n_rays.
  struct Row { int pass_row, ray, sample; bool used; };  // row within the unit's pass, ray within the unit, sample of the ray
  NFB_HD constexpr Row row(int pass, int local_tile, int tile_row) const {
    const int S = samples(pass), prow = local_tile * kTileM + tile_row;
    const bool used = prow < rays_per_unit * S;
    const int ray = used ? prow / S : 0;
    return Row{prow, ray, used ? prow - ray * S : 0, used};
  }
  NFB_HD constexpr int ray_index(int unit, int ray) const { return unit * rays_per_unit + ray; }
};

namespace geom_check {
constexpr bool cut(int nc, int nf, int R, int tc, int tf) {
  const TileGeom g = TileGeom::make(5, nc, nf);
  return g.rays_per_unit == R && g.tiles_c == tc && g.tiles_f == tf && g.n_units == (5 + R - 1) / R &&
         g.chunk(3).n_units == (3 + R - 1) / R && g.chunk(3).tiles_f == tf;
}
// row() takes every sample's slot() back to that sample, in a tile of the sample's own network, inside the array.
constexpr bool round_trip(int n_rays, int nc, int nf) {
  const TileGeom g = TileGeom::make(n_rays, nc, nf);
  for (int pass = 0; pass < g.passes(); ++pass)
    for (int r = 0; r < n_rays; ++r)
      for (int i = 0; i < g.samples(pass); ++i) {
        const size_t s = g.slot(pass, r, i);
        const int unit = (int)((s >> 7) / g.tiles_per_unit()), lt = (int)((s >> 7) % g.tiles_per_unit()) - g.tile_base(pass);
        if (lt < 0 || lt >= g.tile_count(pass) || g.net_of(g.tile_base(pass) + lt) != pass) return false;
        const TileGeom::Row w = g.row(pass, lt, (int)(s & 127));
        if (!w.used || w.sample != i || g.ray_index(unit, w.ray) != r || s >= g.tiles() * 128) return false;
      }
  return true;
}
static_assert(cut(64, 128, 2, 1, 3) && cut(128, 256, 1, 1, 3) && cut(64, 0, 2, 1, 0) && cut(256, 256, 1, 2, 4), "tile cut");
static_assert(round_trip(5, 64, 128) && round_trip(3, 128, 256) && round_trip(5, 64, 0) && round_trip(2, 256, 256) &&
              round_trip(5, 3, 7), "slot / row round trip");
}  // namespace geom_check

// The order in which one CTA of the render kernel runs the tiles of its n_iter units (its "tile stream"; the weight producer
// and the row warps both walk it).  With C(u) = the coarse tiles of the CTA's u-th unit and F(u) = its fine tiles:
//   C(0), [C(u+1), F(u)] for u = 0 .. n_iter-2, F(n_iter-1)        (nf == 0: C(0), C(1), ...)
// so the per-ray stages of unit u (compositing, resampling, sorting) run on other warps while the tensor cores run C(u+1)
// and the fine tiles of u-1.  Only the order changes: global_tile(unit, pass, t) still names each tile's record.
struct StreamTile { int it, pass, t; };  // the CTA's unit iteration, pass (= network), tile within the pass
NFB_HD constexpr int stream_tiles(const TileGeom& g, int n_iter) { return n_iter * g.tiles_per_unit(); }
NFB_HD constexpr StreamTile stream_tile(const TileGeom& g, int n_iter, int k) {
  const int tc = g.tiles_c, tpu = g.tiles_per_unit();
  if (g.nf == 0) return StreamTile{k / tc, 0, k - (k / tc) * tc};
  if (k < tc) return StreamTile{0, 0, k};
  const int b = (k - tc) / tpu, r = (k - tc) - b * tpu;
  if (b == n_iter - 1) return StreamTile{b, 1, r};
  return r < tc ? StreamTile{b + 1, 0, r} : StreamTile{b, 1, r - tc};
}

namespace geom_check {
// Every tile of every unit appears once, in its own network; C(u) precedes F(u); and the first tile of C(u) comes after
// every tile of C(v <= u-1) and F(v <= u-2), the first tile of F(u) after every tile of C(v <= u) and F(v <= u-1): what
// the render kernel's hand-offs wait for before those tiles (nfb_render.cu) is produced from strictly earlier tiles.
constexpr bool stream_order(int nc, int nf, int n_iter) {
  const TileGeom g = TileGeom::make(2 * n_iter, nc, nf);
  constexpr int kMaxIt = 4, kMaxT = 8;
  int pos[kMaxIt][2][kMaxT] = {};
  int seen[kMaxIt][2][kMaxT] = {};
  const int n = stream_tiles(g, n_iter);
  for (int k = 0; k < n; ++k) {
    const StreamTile s = stream_tile(g, n_iter, k);
    if (s.it < 0 || s.it >= n_iter || s.pass < 0 || s.pass >= g.passes() || s.t < 0 || s.t >= g.tile_count(s.pass)) return false;
    if (g.net_of(g.tile_base(s.pass) + s.t) != s.pass) return false;
    ++seen[s.it][s.pass][s.t];
    pos[s.it][s.pass][s.t] = k;
  }
  for (int u = 0; u < n_iter; ++u)
    for (int pass = 0; pass < g.passes(); ++pass)
      for (int t = 0; t < g.tile_count(pass); ++t) {
        if (seen[u][pass][t] != 1) return false;
        const int first = pos[u][pass][0];
        for (int v = 0; v < n_iter; ++v)
          for (int q = 0; q < g.passes(); ++q)
            for (int x = 0; x < g.tile_count(q); ++x) {
              const bool before = pass == 0 ? (q == 0 ? v <= u - 1 : v <= u - 2) : (q == 0 ? v <= u : v <= u - 1);
              if (before && pos[v][q][x] >= first) return false;
            }
      }
  return true;
}
static_assert(stream_order(64, 128, 1) && stream_order(64, 128, 2) && stream_order(64, 128, 3) && stream_order(128, 256, 3) &&
              stream_order(256, 256, 1) && stream_order(256, 256, 2) && stream_order(256, 256, 3) && stream_order(64, 0, 1) &&
              stream_order(64, 0, 3) && stream_order(3, 7, 1) && stream_order(3, 7, 2) && stream_order(3, 7, 3),
              "render tile stream order");
}  // namespace geom_check

// ------------------------------------------------------------------------------------------------
// Training: per-tile activation record (written by the forward kernel in SAVE mode and by the backward chain kernel,
// read by the weight-gradient kernel).  Every entry is a TRANSPOSED image of a [128 sample rows x C features] FP16
// matrix: element (feature k, sample r) lives in r-atom (r >> 6) — a [C rows x 64 r] block in the same 128-byte-swizzled
// K-major layout as a weight unit — so the weight-gradient GEMM  dW[n,k] = sum_r dY[r,n] X[r,k]  reads both operands
// with plain bulk copies and the K-major descriptors of the forward pass (reduction dimension = sample rows).
constexpr int kRecPE = 0;                         // positional encoding, 64 features (lane 63 = 0)
constexpr int kRecH0 = 16384;                     // h0..h5 (outputs of tensor-core steps 0..5), 256 features each
constexpr int kRecG0 = kRecH0 + 6 * 65536;        // g0..g2 (steps 6..8), 128 features each
constexpr int kRecPEd = kRecG0 + 3 * 32768;       // per-ray direction encoding replicated per sample, 32 rows (24 used)
constexpr int kRecMask = kRecPEd + 8192;          // ReLU masks: [9 layers][128 rows][8 x u32]
constexpr int kRecDY0 = kRecMask + 9 * 128 * 32;  // dY0..dY5 (gradient w.r.t. the pre-activation of steps 0..5), 256 features
constexpr int kRecDY6 = kRecDY0 + 6 * 65536;      // dY6..dY8, 128 features
constexpr int kRecDRaw = kRecDY6 + 3 * 32768;     // scaled (d rgb_raw[3], d sigma_raw) image, 16 rows (4 used)
constexpr int kRecBytes = kRecDRaw + 4096;
static_assert(kRecBytes == (1 << 20), "tile record is 1 MiB");
// Exact-grad mode (NFB_PREC_EXACT_GRAD) keeps a second MiB behind every record: at kRecBytes + the offset of each image above,
// its lo half, lo = FP16(x - hi), so that hi + lo carries the value to ~2^-22 relative.  The training forward writes the lo images
// of PE, h0..h5, g0..g2 and PEd; the dX chain those of dY0..dY8 and d raw.  The mask block has no lo half (its bytes are unused).
NFB_HD constexpr size_t rec_stride(bool hilo) { return hilo ? 2 * (size_t)kRecBytes : (size_t)kRecBytes; }
NFB_HD constexpr int rec_x_off(int layer) { return layer < 6 ? kRecH0 + layer * 65536 : kRecG0 + (layer - 6) * 32768; }
NFB_HD constexpr int rec_dy_off(int layer) { return layer < 6 ? kRecDY0 + layer * 65536 : kRecDY6 + (layer - 6) * 32768; }
NFB_HD constexpr int rec_width(int layer) { return layer < 6 ? 256 : 128; }
// Byte offset of element (feature k, sample row r) inside an image with `rows` features.
NFB_HD constexpr int img_offset(int rows, int k, int r) { return (r >> 6) * rows * 128 + sw128_offset(k, r & 63); }

// Backward chain (dX): 9 tensor-core steps per 128-row tile, same machinery as the forward pass with transposed weights.
//   step  computes                         N (half0+half1)  K atoms                A operand
//   0     d g2 = d rgb . Wrgb              128              1 (smem, k<3 used)     SMEM (d raw operand)
//   1     d g1 = dY8 . Wd2                 128              2                      SMEM (activations)
//   2     d g0 = dY7 . Wd1                 128              2                      SMEM (activations)
//   3     d h5 = dY6 . M1 + d sigma . m2   128 + 128        1 (smem, k=3) + 2      SMEM atom + activations
//   4..8  d h4..h0 = dY . W5, W4, W3[:,171:], W2, W1   128 + 128   4               SMEM (activations)
// The epilogue of step s multiplies by the ReLU mask of forward layer (8 - s) and yields dY(8 - s).
constexpr int kBwdSteps = 9;
NFB_HD constexpr StepInfo bwd_step_info(int s) {
  return s == 0   ? StepInfo{128, 0, 1, 1, 0, 0}
         : s <= 2 ? StepInfo{128, 0, 2, 0, 0, 0}
         : s == 3 ? StepInfo{128, 128, 3, 1, 0, 0}
                  : StepInfo{128, 128, 4, 0, 0, 0};
}

// ------------------------------------------------------------------------------------------------
// The two weight streams: the forward MLP (step_info) and the backward chain (bwd_step_info, transposed weights).  Both are
// laid out by one rule: a unit = all N rows of a step x one 64-wide K atom, units in consumption order (step by step, K atom
// by K atom), so unit u of step s starts at (offset of step s) + u * rows * 128.  The x1 stream holds FP16 weights; the x3
// stream of exact mode holds the hi unit then the lo unit at twice the x1 offset.  Written by repack_kernel (nfb_pack.cu),
// read by the kernels through the unit program below.  The backward stream has a lo half of its own for exact-grad mode, a
// separate buffer with the backward stream's layout (bwd_lo_kernel, nfb_pack.cu).
enum : int { kFwdStream = 0, kBwdStream = 1 };
NFB_HD constexpr int stream_steps(int stream) { return stream == kFwdStream ? kNumSteps : kBwdSteps; }
NFB_HD constexpr StepInfo stream_step(int stream, int s) { return stream == kFwdStream ? step_info(s) : bwd_step_info(s); }
NFB_HD constexpr int unit_rows(int stream, int s) { return stream_step(stream, s).nh0 + stream_step(stream, s).nh1; }
NFB_HD constexpr int unit_offset(int stream, int s, int u) {
  int off = 0;
  for (int i = 0; i < s; ++i) off += stream_step(stream, i).k_atoms * unit_rows(stream, i) * 128;
  return off + u * unit_rows(stream, s) * 128;
}
constexpr int kStreamBytesX1 = unit_offset(kFwdStream, kNumSteps, 0);  // 864256
constexpr int kStreamBytesX3 = 2 * kStreamBytesX1;
constexpr int kBwdStreamBytes = unit_offset(kBwdStream, kBwdSteps, 0);  // 835584

// Per-tile unit program of a stream, built at compile time: one entry per unit in consumption order.  x = MMA N (rows of the
// unit), y = K atom of the activation buffer the A operand comes from, z = flags, w = (byte offset in the stream, x1 layout)
// / 16 | rows << 20.  kUnitFromOperand: the A operand is the step's own shared-memory operand (the PE buffer forward, the d raw
// operand backward), not the activation buffer.
enum : uint32_t { kUnitFromOperand = 1u, kUnitFirst = 8u, kUnitLast = 16u };
struct ProgEntry { uint32_t x, y, z, w; };
constexpr int kMaxProgUnits = 32;
struct ProgTable { ProgEntry e[kMaxProgUnits]; };
NFB_HD constexpr int prog_units(int stream) {
  int n = 0;
  for (int s = 0; s < stream_steps(stream); ++s) n += stream_step(stream, s).k_atoms;
  return n;
}
static_assert(prog_units(kFwdStream) <= kMaxProgUnits && prog_units(kBwdStream) <= kMaxProgUnits, "program table too small");
constexpr ProgTable make_prog(int stream) {
  ProgTable t{};
  int i = 0;
  for (int s = 0; s < stream_steps(stream); ++s) {
    const StepInfo si = stream_step(stream, s);
    const uint32_t rows = (uint32_t)unit_rows(stream, s);  // <= 256
    for (int u = 0; u < si.k_atoms; ++u, ++i) {
      const bool from_op = si.pe_first && u == 0;
      t.e[i].x = rows;
      t.e[i].y = from_op ? 0u : (uint32_t)(u - si.pe_first);
      t.e[i].z = (from_op ? kUnitFromOperand : 0u) | (u == 0 ? kUnitFirst : 0u) | (u == si.k_atoms - 1 ? kUnitLast : 0u);
      t.e[i].w = ((uint32_t)unit_offset(stream, s, u) >> 4) | (rows << 20);
    }
  }
  return t;
}

// Weight-gradient accumulators of one network (FP32, float offsets), in the kernel's folded parametrisation.
constexpr int kAcc0 = 0;                       // [256][64]   d W0[:, PE lanes]
constexpr int kAcc1 = kAcc0 + 256 * 64;        // [256][256]
constexpr int kAcc2 = kAcc1 + 65536;
constexpr int kAcc3a = kAcc2 + 65536;          // [256][64]   d W3[:, PE lanes]
constexpr int kAcc3b = kAcc3a + 256 * 64;      // [256][256]  d W3[:, 171:427]
constexpr int kAcc4 = kAcc3b + 65536;
constexpr int kAcc5 = kAcc4 + 65536;
constexpr int kAcc6 = kAcc5 + 65536;           // [128][256]  d M1 (layers_dir.0[:, :256] . fc_feat)
constexpr int kAcc6d = kAcc6 + 128 * 256;      // [128][32]   d layers_dir.0[:, 256:280]
constexpr int kAccSig = kAcc6d + 128 * 32;     // [256][16]   column 3 = d m2 (fc_alpha . fc_feat)
constexpr int kAcc7 = kAccSig + 256 * 16;      // [128][128]
constexpr int kAcc8 = kAcc7 + 128 * 128;
constexpr int kAcc9 = kAcc8 + 128 * 128;       // [128][16]   transposed: [k][n], n < 3 = d fc_rgb.weight[n][k]
constexpr int kAccB = kAcc9 + 128 * 16;        // biases: b0..b5 [256] each, b6..b8 [128] each, then [4] = (d b_rgb[3], d b_sigma)
constexpr int kAccBRaw = kAccB + 6 * 256 + 3 * 128;
constexpr int kAccFloats = kAccBRaw + 4;
NFB_HD constexpr int acc_bias_off(int layer) { return kAccB + (layer < 6 ? layer * 256 : 1536 + (layer - 6) * 128); }

// Algorithmic cost used for the roofline (SURVEY.md §8d): 550,016 MAC per MLP evaluation.
constexpr long long kAlgoFlopPerEval = 1100032LL;
// MACs the kernel actually issues per evaluation after the folds above.
constexpr long long kExecMacPerEval = 64LL * 256 + 4LL * 256 * 256 + 320LL * 256 + 256LL * 144 + 2LL * 128 * 128 + 128LL * 16;

}  // namespace nfb
