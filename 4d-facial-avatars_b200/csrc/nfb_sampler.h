// nfb_sampler.h — exact arithmetic behind the training-ray sampler (host + device).
//
// Reference (train_transformed_rays.py:230-239, 319-331): per training image a probability map over the H x W pixels — (1 - p)
// everywhere, p inside the image's bounding box, normalised — and per iteration
//     select_inds = np.random.choice(H * W, size=2048, replace=False, p=map)
// numpy's algorithm (RandomState.choice): repeat { x = rand(size - n_found); zero p at the indices found so far;
// cdf = cumsum(p); cdf /= cdf[-1]; new = searchsorted(cdf, x, side='right'); keep first occurrences in draw order } until `size`
// distinct indices are found.  np.cumsum is a SEQUENTIAL float64 accumulation, so cdf[k] carries 262,144 ordered roundings.
//
// To reproduce the indices bit for bit without a 262,144-step serial loop per round, use the map's structure: in row-major order
// it is a few hundred RUNS of one constant (q_out or q_in) each.  Adding a constant c repeatedly to s in round-to-nearest: while
// s stays inside one binade, every add moves s by the SAME exact multiple d of ulp(s) (the discarded part of c is the same
// each time) — also when that part is exactly half an ulp, once s sits on an even multiple of ulp (round-half-even keeps it there).  So the partial sums of a run are a short list of exact arithmetic progressions (SEGMENTS), one per
// binade crossed, and cdf[k] is one multiply-add in exact arithmetic.  Entries zeroed in later rounds only shift the add count.
// An ABSORBED add (s + c == s: c below half an ulp of s, or exactly half with s on an even multiple) is the case d = 0: s never
// moves again, so every later add of the run is absorbed too and one segment covers the rest of the run.  (Maps far from the
// reference's p = 0.9 reach it: p = 1e-12 or 1 - 1e-12 absorbs one of the two constants once the sum nears 1.)
// Segments per map: a run starts with at most a tie step (odd s -> even) and one progression, and each binade it enters adds at
// most three (the crossing add, a tie step, a progression), so R runs whose running sum crosses B binades need at most
// 2 R + 3 B + 1 segments (+1: the first add from s = 0).  A normalised map's sum stays below 2 and no add is below 2^-1074, so
// B <= 1075 and kMaxRuns runs fit kMaxSegs: 2 * 4096 + 3 * 1075 + 1 = 11,418 <= 16,384.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define NFB_SHD __host__ __device__ inline
#else
#define NFB_SHD inline
#endif

namespace nfb {
namespace smp {

struct Map {       // one training image's importance map (flat index k = row * W + col of the PROBABILITY map)
  int H, W;
  int b0, b1, b2, b3;  // probs[b0:b1, b2:b3] = p
  double q_out, q_in;  // the two values of the normalised map, as numpy computed them
};
struct Run { long long k0, len; double c; double s_before; int seg0, nseg; long long adds; };
struct Seg { long long t0, n; double v0, d; };  // value after add t (1-based inside the run), t0 <= t < t0 + n: v0 + (t - t0) * d

constexpr int kMaxRuns = 4096, kMaxSegs = 16384;

NFB_SHD int num_runs(const Map& m) {
  if (m.b1 <= m.b0 || m.b3 <= m.b2) return 1;
  return 1 + 2 * (m.b1 - m.b0);
}
// run r of the map in row-major order: leading q_out run, then per box row (q_in run, q_out run up to the next box row / the end)
NFB_SHD void run_extent(const Map& m, int r, long long& k0, long long& len, double& c) {
  const long long N = (long long)m.H * m.W;
  if (m.b1 <= m.b0 || m.b3 <= m.b2) { k0 = 0; len = N; c = m.q_out; return; }
  const long long first_in = (long long)m.b0 * m.W + m.b2;
  if (r == 0) { k0 = 0; len = first_in; c = m.q_out; return; }
  const int row = m.b0 + (r - 1) / 2;
  if ((r - 1) % 2 == 0) { k0 = (long long)row * m.W + m.b2; len = m.b3 - m.b2; c = m.q_in; return; }
  k0 = (long long)row * m.W + m.b3;
  const bool last = (row == m.b1 - 1);
  len = last ? (N - k0) : ((long long)(row + 1) * m.W + m.b2 - k0);
  c = m.q_out;
}

// Add c (> 0) to s, `t` times, each add rounded to nearest-even as np.cumsum does; append the segments that give every
// intermediate value; returns the final s.  t_base = adds already taken inside the current run.
NFB_SHD double seq_add(double s, double c, long long t, long long t_base, Seg* segs, int& nseg, int max_seg) {
  long long done = 0;
  while (done < t) {
    const double s1 = s + c;  // one true add
    bool bulk = false;
    long long k = 0;
    double d = 0.0;
    if (s > 0.0 && ilogb(s1) == ilogb(s)) {
      const int e = ilogb(s1);
      const double ulp = ldexp(1.0, e - 52);
      const double r = fmod(c, ulp);          // exact: the part of c below this binade's ulp
      // Not a tie: the rounding of s' + c is the same for every s' of the binade.  Tie (r == ulp / 2, round-half-even): the sum
      // lands on an EVEN multiple of ulp, and from an even s' every further add moves by the same even-preserving amount —
      // so only an odd s' needs a single step first.
      if (r != 0.5 * ulp || fmod(s, 2.0 * ulp) == 0.0) {
        d = s1 - s;                           // exact (both multiples of ulp, same binade)
        const double top = ldexp(1.0, e + 1);
        const long long room = (long long)((top - s1) / ulp), step = (long long)(d / ulp);  // exact integers < 2^53
        k = step > 0 ? room / step : t - done - 1;  // further adds that stay <= top; absorbed (d = 0): all the rest
        if (k > t - done - 1) k = t - done - 1;
        bulk = true;
      }
    }
    if (nseg < max_seg) {
      Seg& g = segs[nseg];
      g.t0 = t_base + done + 1; g.n = 1 + (bulk ? k : 0); g.v0 = s1; g.d = bulk ? d : 0.0;
    }
    ++nseg;
    s = bulk ? s1 + (double)k * d : s1;       // k * d <= top - s1 is a multiple of ulp: exact
    done += 1 + (bulk ? k : 0);
  }
  return s;
}

// number of entries of the ascending list `z` (n entries) that lie in [a, b]
NFB_SHD long long count_in(const long long* z, int n, long long a, long long b) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (z[mid] < a) lo = mid + 1; else hi = mid; }
  const int first = lo;
  hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (z[mid] <= b) lo = mid + 1; else hi = mid; }
  return lo - first;
}

// Build the run / segment tables of the map with the entries `zeroed` (ascending flat indices) removed.  Returns cdf[-1] (raw).
NFB_SHD double build_tables(const Map& m, const long long* zeroed, int n_zero, Run* runs, int& n_runs, Seg* segs, int& n_segs) {
  n_runs = num_runs(m);
  n_segs = 0;
  double s = 0.0;
  for (int r = 0; r < n_runs && r < kMaxRuns; ++r) {
    Run& R = runs[r];
    run_extent(m, r, R.k0, R.len, R.c);
    R.s_before = s;
    R.seg0 = n_segs;
    R.adds = R.len - (n_zero ? count_in(zeroed, n_zero, R.k0, R.k0 + R.len - 1) : 0);
    int ns = n_segs;
    if (R.adds > 0 && R.c > 0.0) s = seq_add(s, R.c, R.adds, 0, segs, ns, kMaxSegs);
    R.nseg = ns - n_segs;
    n_segs = ns;
  }
  return s;
}

// raw cdf[k] = np.cumsum(p)[k] with p zeroed at `zeroed`
NFB_SHD double cdf_at(long long k, const Run* runs, int n_runs, const Seg* segs, const long long* zeroed, int n_zero) {
  int lo = 0, hi = n_runs - 1;  // last run with k0 <= k
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (runs[mid].k0 <= k) lo = mid; else hi = mid - 1; }
  const Run& R = runs[lo];
  const long long t = (k - R.k0 + 1) - (n_zero ? count_in(zeroed, n_zero, R.k0, k) : 0);
  if (t <= 0) return R.s_before;
  int a = R.seg0, b = R.seg0 + R.nseg - 1;  // last segment with t0 <= t
  while (a < b) { const int mid = (a + b + 1) >> 1; if (segs[mid].t0 <= t) a = mid; else b = mid - 1; }
  const Seg& g = segs[a];
  return g.v0 + (double)(t - g.t0) * g.d;
}

// cdf.searchsorted(x, side='right') on the NORMALISED cdf (cdf /= cdf[-1]): the first k with cdf[k] / total > x
NFB_SHD long long search_right(double x, double total, long long N, const Run* runs, int n_runs, const Seg* segs, const long long* zeroed,
                               int n_zero) {
  long long lo = 0, hi = N;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (cdf_at(mid, runs, n_runs, segs, zeroed, n_zero) / total <= x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

#if defined(__CUDACC__)
// Camera-space direction (cx, cy, -1) of pixel (row, col), as get_ray_bundle (nerf_helpers.py:111-122) forms it in FP32:
// cx = (col - W * cx0) / fx, cy = -(row - H * cy0) / fy, with wcx = W * cx0 and hcy = H * cy0 rounded to FP32 once.  The
// samplers' gathers and the pose-gradient rows of nfb_fit_rows_grad both call it, so the pose gradient multiplies by the very
// bits the rays were built from.
__device__ __forceinline__ void camera_dir(int row, int col, float fx, float fy, float wcx, float hcy, float& cx, float& cy) {
  cx = __fdiv_rn(__fsub_rn((float)col, wcx), fx);
  cy = -__fdiv_rn(__fsub_rn((float)row, hcy), fy);
}
#endif

// Row of pixel (row, col) in an [H][W] table (image, background), row-major.  The samplers' gathers read the target and
// background colours there and nfb_background_rows_grad adds the background's gradient there: one helper, so the scatter
// writes exactly the pixel the gather read (the flat draw index k maps to (row, col) = (k % H, k / H) before this, in the gather).
NFB_SHD size_t pixel_index(int row, int col, int W) { return (size_t)row * W + col; }

}  // namespace smp
}  // namespace nfb
