// yolov3_b200 — validation metrics on the device: the tail of val.run (reference val.py:379-429) that turns matched
// detections into the numbers a user reads.
//   y3_val_prepare      native-space detections / labels of one batch (val.py:394-403) + the accumulator's conf / cls / count
//                       slices; y3_val_match then writes the batch's `correct` rows straight into the accumulator.
//   y3_confusion_update ConfusionMatrix.process_batch (utils/metrics.py:134-178) for a whole batch, integer atomics.
//   y3_ap_per_class     ap_per_class + compute_ap (utils/metrics.py:22-120) over every accumulated row.
// ap_per_class pipeline (work scales with the number of rows, not of classes):
//   count     per-class prediction and label histograms, sort keys (class, ~bits(conf)), "any TP" flag
//   sort      stable LSD radix sort of the keys, 8-bit digits: 4 confidence passes then 1-2 class passes; rows past an image's
//             count carry the class key nc and sort behind every class
//   P         global inclusive prefix of each IoU column's TP bytes in sorted order (tile sums, one-block scan of the tile
//             sums, fix-up): tpc at sorted position k of class c = P[k] - P[start(c) - 1], exact integers
//   S         suffix max of precision = tpc / (k - start + 1) inside each class segment (the envelope of compute_ap): an
//             unsegmented reverse scan of (class, precision) pairs under "smaller class first, then larger precision", whose
//             result at k is k's own class
//   AP        one thread per point of the 101-point grid: binary search of recall, np.interp, np.trapezoid summed in numpy's
//             pairwise order (8 accumulators for n <= 128)
//   curves    one thread per px point: binary search of the confidence, np.interp of recall / precision (left = 0 / 1), F1
//   final     mean F1 over the labelled classes (sequential, numpy's axis-0 reduce), smooth(f, 0.1) as a sequential sum, the
//             first argmax, p / r / f1 / tp / fp at it (rint = numpy's half-to-even)
// Ties in confidence keep the accumulation order (image, NMS row): numpy's argsort(-conf) is unstable there (DESIGN.md §2).
// Compiled without fast math / FMA contraction (build.py EXACT_SOURCES): every fp64 expression is numpy's, op for op.
#include <math.h>

#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {
namespace {

constexpr int kThreads = 256;
constexpr int kItems = 8;
constexpr int kTile = kThreads * kItems;  // rows of one sort tile / scan chunk
constexpr int kNpx = 1000;                // px = linspace(0, 1, 1000)        (utils/metrics.py:50)
constexpr int kNap = 101;                 // x  = linspace(0, 1, 101)         (utils/metrics.py:114)
constexpr int kMaxLabels = 1024;          // labels of one image staged in shared memory (as y3_val_match)
constexpr int kMaxNc = 1024;
constexpr double kEps = 1e-16;            // ap_per_class eps

__device__ __forceinline__ uint32_t conf_desc_key(float c) {  // ascending key order = descending confidence
  const uint32_t u = __float_as_uint(c);
  return ~((u & 0x80000000u) ? ~u : (u | 0x80000000u));
}

struct ApArgs {
  const float* conf;       // [n] (n = n_images * stride)
  const float* cls;        // [n]
  const uint8_t* tp;       // [n, niou]
  const int32_t* counts;   // [n_images] or null
  int n, stride, niou;
  const int32_t* tcls;     // [nl]
  int nl, nc;
  const double* px;        // [1000]
  const double* xap;       // [101]
  // workspace
  unsigned long long* key[2];
  int* idx[2];
  int* tile_hist;          // [256][ntiles]
  int* P;                  // [niou][n]
  double* S;               // [niou][n]
  int* tile_sum;           // [niou][ntiles]
  int* agg_seg;            // [niou][ntiles]
  double* agg_val;         // [niou][ntiles]
  int* start;              // [nc + 2]
  int ntiles;
  // outputs
  int32_t* npred;          // [nc + 1] (the last entry counts the rows that are not predictions of a class < nc)
  int32_t* nt;             // [nc]
  int32_t* info;           // [2] = (max-F1 index, any TP)
  double* ap;              // [nc, niou]
  double* curves;          // [3, nc, 1000] = p, r, f1
  double* best;            // [5, nc] = p, r, f1, tp, fp at the max-F1 index
};

// ------------------------------------------------------------------------------------------------ block scans
// exclusive prefix sum over the block (blockDim.x threads, s: blockDim.x ints); *total = block sum
__device__ int block_excl_sum(int v, int* s, int* total) {
  const int t = threadIdx.x;
  s[t] = v;
  __syncthreads();
  for (int o = 1; o < blockDim.x; o <<= 1) {
    const int add = t >= o ? s[t - o] : 0;
    __syncthreads();
    s[t] += add;
    __syncthreads();
  }
  const int incl = s[t];
  if (total) *total = s[blockDim.x - 1];
  __syncthreads();
  return incl - v;
}

struct SegMax {  // (class segment, precision): a beats b if its segment is smaller, or equal with a larger value
  int seg;
  double v;
};
__device__ __forceinline__ SegMax segmax(const SegMax& a, const SegMax& b) {
  return (a.seg < b.seg || (a.seg == b.seg && a.v > b.v)) ? a : b;
}
__device__ __forceinline__ SegMax segmax_id() { return SegMax{0x7fffffff, 0.0}; }

// exclusive REVERSE scan (combination of the values of threads > t) of SegMax over the block
__device__ SegMax block_rexcl_segmax(SegMax v, int* s_seg, double* s_v) {
  const int t = threadIdx.x, nt = blockDim.x;
  s_seg[t] = v.seg;
  s_v[t] = v.v;
  __syncthreads();
  for (int o = 1; o < nt; o <<= 1) {
    SegMax r = segmax_id();
    if (t + o < nt) r = SegMax{s_seg[t + o], s_v[t + o]};
    __syncthreads();
    const SegMax m = segmax(SegMax{s_seg[t], s_v[t]}, r);
    s_seg[t] = m.seg;
    s_v[t] = m.v;
    __syncthreads();
  }
  const SegMax ex = t + 1 < nt ? SegMax{s_seg[t + 1], s_v[t + 1]} : segmax_id();
  __syncthreads();
  return ex;
}

// ------------------------------------------------------------------------------------------------ ap_per_class kernels
__global__ void __launch_bounds__(kThreads) ap_init_kernel(const ApArgs a) {
  pdl_entry();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= a.nc; i += gridDim.x * blockDim.x) {
    a.npred[i] = 0;
    if (i < a.nc) a.nt[i] = 0;
    if (i < 2) a.info[i] = 0;
  }
}

// histograms (block-local in shared memory, then one global atomic per non-zero bin), sort keys, any-TP flag
__global__ void __launch_bounds__(kThreads) ap_count_kernel(const ApArgs a) {
  __shared__ int s_np[kMaxNc + 1];
  __shared__ int s_nt[kMaxNc];
  __shared__ int s_any;
  pdl_entry();
  for (int i = threadIdx.x; i <= a.nc; i += blockDim.x) {
    s_np[i] = 0;
    if (i < a.nc) s_nt[i] = 0;
  }
  if (threadIdx.x == 0) s_any = 0;
  __syncthreads();
  int any = 0;
  const int total = max(a.n, a.nl);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    if (i < a.n) {
      const int img = i / a.stride, d = i - img * a.stride;
      const bool valid = d < (a.counts ? min(a.counts[img], a.stride) : a.stride);
      int c = a.nc;
      uint32_t ck = 0xffffffffu;
      if (valid) {
        const float cf = a.cls[i];
        if (cf >= 0.0f && cf < static_cast<float>(a.nc)) {  // a class no label can equal (also NaN, 2.5) sorts last
          const int ci = static_cast<int>(cf);
          if (static_cast<float>(ci) == cf) c = ci;
        }
        ck = conf_desc_key(a.conf[i]);
        const uint8_t* t = a.tp + static_cast<size_t>(i) * a.niou;
        for (int j = 0; j < a.niou; ++j) any |= t[j];
      }
      a.key[0][i] = (static_cast<unsigned long long>(c) << 32) | ck;
      a.idx[0][i] = i;
      atomicAdd(&s_np[c], 1);
    }
    if (i < a.nl) {
      const int c = a.tcls[i];
      if (c >= 0 && c < a.nc) atomicAdd(&s_nt[c], 1);
    }
  }
  if (any) s_any = 1;
  __syncthreads();
  for (int i = threadIdx.x; i <= a.nc; i += blockDim.x) {
    if (s_np[i]) atomicAdd(&a.npred[i], s_np[i]);
    if (i < a.nc && s_nt[i]) atomicAdd(&a.nt[i], s_nt[i]);
  }
  if (threadIdx.x == 0 && s_any) atomicOr(&a.info[1], 1);
}

// start[c] = first sorted position of class c (exclusive scan of npred), start[nc + 1] = n
__global__ void __launch_bounds__(1024) ap_start_kernel(const ApArgs a) {
  __shared__ int s[1024];
  pdl_entry();
  int carry = 0;
  for (int base = 0; base <= a.nc; base += blockDim.x) {
    const int i = base + threadIdx.x;
    int tot;
    const int ex = block_excl_sum(i <= a.nc ? a.npred[i] : 0, s, &tot);
    if (i <= a.nc) a.start[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) a.start[a.nc + 1] = carry;
}

// one-block exclusive scan, in place, of `len` ints at data + blockIdx.x * row (each thread owns a contiguous range)
__global__ void __launch_bounds__(1024) scan_rows_kernel(int* data, int len, int row) {
  __shared__ int s[1024];
  pdl_entry();
  int* p = data + static_cast<size_t>(blockIdx.x) * row;
  const int per = (len + blockDim.x - 1) / blockDim.x;
  const int lo = min(len, threadIdx.x * per), hi = min(len, lo + per);
  int sum = 0;
  for (int i = lo; i < hi; ++i) sum += p[i];
  int run = block_excl_sum(sum, s, nullptr);
  for (int i = lo; i < hi; ++i) {
    const int v = p[i];
    p[i] = run;
    run += v;
  }
}

__global__ void __launch_bounds__(kThreads) radix_hist_kernel(const unsigned long long* __restrict__ key, int n, int shift,
                                                              int* __restrict__ tile_hist, int ntiles) {
  __shared__ int h[256];
  pdl_entry();
  h[threadIdx.x] = 0;
  __syncthreads();
  const int base = blockIdx.x * kTile;
  for (int r = 0; r < kItems; ++r) {
    const int i = base + r * kThreads + threadIdx.x;
    if (i < n) atomicAdd(&h[(key[i] >> shift) & 255], 1);
  }
  __syncthreads();
  tile_hist[threadIdx.x * ntiles + blockIdx.x] = h[threadIdx.x];
}

// stable scatter: rounds of 256 rows in index order; inside a round a row's rank = rows of its digit in earlier warps
// (per-warp digit counts) + earlier lanes of its warp with the same digit (__match_any_sync)
__global__ void __launch_bounds__(kThreads) radix_scatter_kernel(const unsigned long long* __restrict__ key_in,
                                                                 const int* __restrict__ idx_in,
                                                                 unsigned long long* __restrict__ key_out,
                                                                 int* __restrict__ idx_out, int n, int shift,
                                                                 const int* __restrict__ tile_hist, int ntiles) {
  __shared__ int s_base[256];
  __shared__ int s_wcnt[kThreads / 32][256];
  pdl_entry();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  s_base[threadIdx.x] = tile_hist[threadIdx.x * ntiles + blockIdx.x];
  const int base = blockIdx.x * kTile;
  for (int r = 0; r < kItems; ++r) {
    for (int w = 0; w < kThreads / 32; ++w) s_wcnt[w][threadIdx.x] = 0;
    __syncthreads();
    const int i = base + r * kThreads + threadIdx.x;
    const bool act = i < n;
    unsigned long long k = 0;
    int dg = 256;
    if (act) {
      k = key_in[i];
      dg = static_cast<int>((k >> shift) & 255);
    }
    const unsigned peers = __match_any_sync(0xffffffffu, dg);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (act && rank == 0) s_wcnt[warp][dg] = __popc(peers);
    __syncthreads();
    {  // thread t owns digit t: warp-exclusive offsets on top of the tile's running offset
      int run = s_base[threadIdx.x];
      for (int w = 0; w < kThreads / 32; ++w) {
        const int c = s_wcnt[w][threadIdx.x];
        s_wcnt[w][threadIdx.x] = run;
        run += c;
      }
      s_base[threadIdx.x] = run;
    }
    __syncthreads();
    if (act) {
      const int pos = s_wcnt[warp][dg] + rank;
      key_out[pos] = k;
      idx_out[pos] = idx_in[i];
    }
    __syncthreads();
  }
}

__device__ __forceinline__ int seg_of(const ApArgs& a, const unsigned long long* key, int k) {
  return static_cast<int>(key[k] >> 32);
}
__device__ __forceinline__ int tp_at(const ApArgs& a, const unsigned long long* key, const int* idx, int k, int j) {
  return seg_of(a, key, k) < a.nc ? a.tp[static_cast<size_t>(idx[k]) * a.niou + j] : 0;
}

// grid (ntiles, niou): TP count of every tile in sorted order
__global__ void __launch_bounds__(kThreads) ap_tile_sum_kernel(const ApArgs a, const unsigned long long* __restrict__ key,
                                                               const int* __restrict__ idx) {
  __shared__ int s[kThreads];
  pdl_entry();
  const int j = blockIdx.y, k0 = blockIdx.x * kTile + threadIdx.x * kItems;
  int sum = 0;
  for (int q = 0; q < kItems; ++q)
    if (k0 + q < a.n) sum += tp_at(a, key, idx, k0 + q, j);
  int tot;
  block_excl_sum(sum, s, &tot);
  if (threadIdx.x == 0) a.tile_sum[j * a.ntiles + blockIdx.x] = tot;
}

// grid (ntiles, niou): P[j][k] = global inclusive prefix of TP column j in sorted order
__global__ void __launch_bounds__(kThreads) ap_prefix_kernel(const ApArgs a, const unsigned long long* __restrict__ key,
                                                             const int* __restrict__ idx) {
  __shared__ int s[kThreads];
  pdl_entry();
  const int j = blockIdx.y, k0 = blockIdx.x * kTile + threadIdx.x * kItems;
  int v[kItems];
  int sum = 0;
  for (int q = 0; q < kItems; ++q) {
    v[q] = k0 + q < a.n ? tp_at(a, key, idx, k0 + q, j) : 0;
    sum += v[q];
  }
  int run = a.tile_sum[j * a.ntiles + blockIdx.x] + block_excl_sum(sum, s, nullptr);
  int* P = a.P + static_cast<size_t>(j) * a.n;
  for (int q = 0; q < kItems; ++q) {
    run += v[q];
    if (k0 + q < a.n) P[k0 + q] = run;
  }
}

__device__ __forceinline__ SegMax prec_at(const ApArgs& a, const unsigned long long* key, int k, int j) {
  const int c = seg_of(a, key, k);
  if (c >= a.nc) return SegMax{c, 0.0};
  const int s0 = a.start[c];
  const int* P = a.P + static_cast<size_t>(j) * a.n;
  const int tpc = P[k] - (s0 > 0 ? P[s0 - 1] : 0);
  return SegMax{c, static_cast<double>(tpc) / static_cast<double>(k - s0 + 1)};  // tpc / (tpc + fpc)
}

// grid (ntiles, niou): the SegMax of every tile
__global__ void __launch_bounds__(kThreads) ap_tile_max_kernel(const ApArgs a, const unsigned long long* __restrict__ key) {
  __shared__ int s_seg[kThreads];
  __shared__ double s_v[kThreads];
  pdl_entry();
  const int j = blockIdx.y, k0 = blockIdx.x * kTile + threadIdx.x * kItems;
  SegMax m = segmax_id();
  for (int q = 0; q < kItems; ++q)
    if (k0 + q < a.n) m = segmax(m, prec_at(a, key, k0 + q, j));
  // the reverse-exclusive value of thread 0 combined with its own = the whole block
  const SegMax rest = block_rexcl_segmax(m, s_seg, s_v);
  if (threadIdx.x == 0) {
    const SegMax all = segmax(m, rest);
    a.agg_seg[j * a.ntiles + blockIdx.x] = all.seg;
    a.agg_val[j * a.ntiles + blockIdx.x] = all.v;
  }
}

// grid (niou), one block: agg[j][t] := combination of the tiles > t (reverse exclusive scan, in place)
__global__ void __launch_bounds__(1024) ap_tile_carry_kernel(const ApArgs a) {
  __shared__ int s_seg[1024];
  __shared__ double s_v[1024];
  pdl_entry();
  int* seg = a.agg_seg + blockIdx.x * a.ntiles;
  double* val = a.agg_val + blockIdx.x * a.ntiles;
  const int per = (a.ntiles + blockDim.x - 1) / blockDim.x;
  const int lo = min(a.ntiles, threadIdx.x * per), hi = min(a.ntiles, lo + per);
  SegMax m = segmax_id();
  for (int i = lo; i < hi; ++i) m = segmax(m, SegMax{seg[i], val[i]});
  SegMax run = block_rexcl_segmax(m, s_seg, s_v);
  for (int i = hi - 1; i >= lo; --i) {
    const SegMax v = SegMax{seg[i], val[i]};
    seg[i] = run.seg;
    val[i] = run.v;
    run = segmax(run, v);
  }
}

// grid (ntiles, niou): S[j][k] = max precision over positions >= k of k's class (the compute_ap envelope)
__global__ void __launch_bounds__(kThreads) ap_suffix_kernel(const ApArgs a, const unsigned long long* __restrict__ key) {
  __shared__ int s_seg[kThreads];
  __shared__ double s_v[kThreads];
  pdl_entry();
  const int j = blockIdx.y, k0 = blockIdx.x * kTile + threadIdx.x * kItems;
  SegMax v[kItems];
  SegMax m = segmax_id();
  for (int q = 0; q < kItems; ++q) {
    v[q] = k0 + q < a.n ? prec_at(a, key, k0 + q, j) : segmax_id();
    m = segmax(m, v[q]);
  }
  SegMax run = segmax(block_rexcl_segmax(m, s_seg, s_v),
                      SegMax{a.agg_seg[j * a.ntiles + blockIdx.x], a.agg_val[j * a.ntiles + blockIdx.x]});
  double* S = a.S + static_cast<size_t>(j) * a.n;
  for (int q = kItems - 1; q >= 0; --q) {
    run = segmax(run, v[q]);
    if (k0 + q < a.n) S[k0 + q] = run.v;
  }
}

// np.interp's rule once the index is known: j = last index with xp[j] <= x (-1: left value), fp[-1] at the end, fp[j] on an
// exact hit, else slope * (x - xp[j]) + fp[j] (no FMA contraction, as numpy on x86-64) with numpy's NaN fallbacks
__device__ __forceinline__ double interp_at(double x, double xj, double xj1, double fj, double fj1) {
  if (xj == x) return fj;
  const double slope = (fj1 - fj) / (xj1 - xj);
  double r = slope * (x - xj) + fj;
  if (isnan(r)) {
    r = slope * (x - xj1) + fj1;
    if (isnan(r) && fj == fj1) r = fj;
  }
  return r;
}

// numpy's pairwise_sum for 8 <= n <= 128: eight strided accumulators, combined as a tree, then the n % 8 tail in order
__device__ double pairwise_sum(const double* t, int n) {
  double r[8];
  for (int q = 0; q < 8; ++q) r[q] = t[q];
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int q = 0; q < 8; ++q) r[q] += t[i + q];
  double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) res += t[i];
  return res;
}

// grid (nc, niou), 128 threads: ap[c][j] = compute_ap(recall[:, j], precision[:, j])
__global__ void __launch_bounds__(128) ap_ap_kernel(const ApArgs a) {
  __shared__ double y[kNap];
  __shared__ double term[kNap - 1];
  pdl_entry();
  const int c = blockIdx.x, j = blockIdx.y;
  const int n = a.npred[c], nl = a.nt[c];
  if (n == 0 || nl == 0) {
    if (threadIdx.x == 0) a.ap[c * a.niou + j] = 0.0;
    return;
  }
  const int s0 = a.start[c];
  const int* P = a.P + static_cast<size_t>(j) * a.n;
  const double* S = a.S + static_cast<size_t>(j) * a.n + s0;
  const int base = s0 > 0 ? P[s0 - 1] : 0;
  const double den = static_cast<double>(nl) + kEps;
  auto recall = [&](int k) { return static_cast<double>(P[s0 + k] - base) / den; };
  // mrec = [0, recall[0..n), 1], mpre (envelope) = [max(1, S[0]), S[0..n), 0]: index i of the n + 2 sentinel arrays
  auto mrec = [&](int i) { return i == 0 ? 0.0 : i <= n ? recall(i - 1) : 1.0; };
  auto mpre = [&](int i) { return i == 0 ? fmax(1.0, S[0]) : i <= n ? S[i - 1] : 0.0; };
  const int q = threadIdx.x;
  if (q < kNap) {
    const double x = a.xap[q];
    int lo = 0, hi = n;  // number of recall values <= x (recall is non-decreasing)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (recall(mid) <= x) lo = mid + 1;
      else hi = mid;
    }
    const int i = lo + ((lo == n && x >= 1.0) ? 1 : 0);  // last index of mrec with mrec[i] <= x (mrec[0] = 0 <= x)
    y[q] = i == n + 1 ? mpre(n + 1) : interp_at(x, mrec(i), mrec(i + 1), mpre(i), mpre(i + 1));
  }
  __syncthreads();
  if (q < kNap - 1) term[q] = (a.xap[q + 1] - a.xap[q]) * (y[q + 1] + y[q]) / 2.0;  // np.trapezoid's terms
  __syncthreads();
  if (q == 0) a.ap[c * a.niou + j] = pairwise_sum(term, kNap - 1);
}

// grid (nc): p, r, f1 curves at px (utils/metrics.py:65,69,78); classes without labels or predictions keep zero rows
__global__ void __launch_bounds__(kThreads) ap_curves_kernel(const ApArgs a, const unsigned long long* __restrict__ key,
                                                             const int* __restrict__ idx) {
  pdl_entry();
  const int c = blockIdx.x;
  const int n = a.npred[c], nl = a.nt[c];
  double* pc = a.curves + static_cast<size_t>(c) * kNpx;
  double* rc = pc + static_cast<size_t>(a.nc) * kNpx;
  double* fc = rc + static_cast<size_t>(a.nc) * kNpx;
  const int s0 = a.start[c];
  const int* P = a.P;  // IoU column 0
  const int base = (n && s0 > 0) ? P[s0 - 1] : 0;
  const double den = static_cast<double>(nl) + kEps;
  auto xp = [&](int k) { return -static_cast<double>(a.conf[idx[s0 + k]]); };  // -conf: non-decreasing
  auto tpc = [&](int k) { return static_cast<double>(P[s0 + k] - base); };
  for (int i = threadIdx.x; i < kNpx; i += blockDim.x) {
    double p = 0.0, r = 0.0;
    if (n > 0 && nl > 0) {
      const double x = -a.px[i];
      int lo = 0, hi = n;  // number of xp values <= x
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (xp(mid) <= x) lo = mid + 1;
        else hi = mid;
      }
      const int jj = lo - 1;
      if (jj < 0) {
        r = 0.0;
        p = 1.0;
      } else if (jj == n - 1) {
        r = tpc(jj) / den;
        p = tpc(jj) / static_cast<double>(jj + 1);
      } else {
        const double x0 = xp(jj), x1 = xp(jj + 1);
        r = interp_at(x, x0, x1, tpc(jj) / den, tpc(jj + 1) / den);
        p = interp_at(x, x0, x1, tpc(jj) / static_cast<double>(jj + 1), tpc(jj + 1) / static_cast<double>(jj + 2));
      }
    }
    pc[i] = p;
    rc[i] = r;
    fc[i] = 2.0 * p * r / (p + r + kEps);
  }
}

// one block: mean F1 over the labelled classes, smooth(., 0.1), first argmax, per-class values at it
__global__ void __launch_bounds__(1024) ap_final_kernel(const ApArgs a) {
  __shared__ double yp[kNpx + 100];
  __shared__ double s_best[1024];
  __shared__ int s_arg[1024];
  pdl_entry();
  const int t = threadIdx.x;
  const double* fc = a.curves + 2 * static_cast<size_t>(a.nc) * kNpx;
  int nu = 0;
  for (int c = 0; c < a.nc; ++c) nu += a.nt[c] > 0;
  for (int i = t; i < kNpx; i += blockDim.x) {
    double s = 0.0;
    for (int c = 0; c < a.nc; ++c)
      if (a.nt[c] > 0) s += fc[static_cast<size_t>(c) * kNpx + i];
    yp[50 + i] = s / static_cast<double>(nu);
  }
  __syncthreads();
  if (t < 50) {  // smooth: nf = round(1000 * 0.1 * 2) // 2 + 1 = 101, 50 copies of each end value on either side
    yp[t] = yp[50];
    yp[50 + kNpx + t] = yp[50 + kNpx - 1];
  }
  __syncthreads();
  const double w = 1.0 / 101.0;  // np.ones(nf) / nf
  double bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = t; i < kNpx; i += blockDim.x) {
    double s = 0.0;
    for (int k = 0; k < 101; ++k) s += yp[i + k] * w;
    if (s > bv) {  // i ascends per thread: the first index of a tie stays
      bv = s;
      bi = i;
    }
  }
  s_best[t] = bv;
  s_arg[t] = bi;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (t < o) {
      const double v2 = s_best[t + o];
      const int i2 = s_arg[t + o];
      if (v2 > s_best[t] || (v2 == s_best[t] && i2 < s_arg[t])) {
        s_best[t] = v2;
        s_arg[t] = i2;
      }
    }
    __syncthreads();
  }
  const int best = nu > 0 && s_arg[0] < kNpx ? s_arg[0] : 0;
  if (t == 0) a.info[0] = best;
  for (int c = t; c < a.nc; c += blockDim.x) {
    const size_t o = static_cast<size_t>(c) * kNpx + best;
    const double p = a.curves[o];
    const double r = a.curves[static_cast<size_t>(a.nc) * kNpx + o];
    const double f = fc[o];
    const double tpv = rint(r * static_cast<double>(a.nt[c]));
    const double fpv = rint(tpv / (p + kEps) - tpv);
    a.best[c] = p;
    a.best[a.nc + c] = r;
    a.best[2 * a.nc + c] = f;
    a.best[3 * a.nc + c] = tpv;
    a.best[4 * a.nc + c] = fpv;
  }
}

// ------------------------------------------------------------------------------------------------ val.py layer
// rows (image, d) of the NMS output -> native space (scale_boxes with the image's ratio_pad, clip to (h0, w0)), single_cls;
// collated targets (image, cls, normalised xywh) -> (image, cls, native xyxy): x (w, h, w, h), xywh2xyxy, scale_boxes
struct PrepArgs {
  const float* det;
  const int32_t* det_count;
  int bs, max_det;
  const float* img;        // [bs, 5] = gain, pad_x, pad_y, h0, w0
  int single_cls;
  const float* targets;
  int nt;
  float img_w, img_h;
  float* det_native;
  float* labels_native;
  float* acc_conf;
  float* acc_cls;
  int32_t* acc_count;
  int32_t* acc_tcls;
};

__device__ __forceinline__ float clamp_like_torch(float v, float hi) { return v != v ? v : fminf(fmaxf(v, 0.0f), hi); }
__device__ __forceinline__ void scale4(float* b, const float* g) {  // y3_scale_boxes' arithmetic
  b[0] = clamp_like_torch(__fdiv_rn(__fsub_rn(b[0], g[1]), g[0]), g[4]);
  b[1] = clamp_like_torch(__fdiv_rn(__fsub_rn(b[1], g[2]), g[0]), g[3]);
  b[2] = clamp_like_torch(__fdiv_rn(__fsub_rn(b[2], g[1]), g[0]), g[4]);
  b[3] = clamp_like_torch(__fdiv_rn(__fsub_rn(b[3], g[2]), g[0]), g[3]);
}

__global__ void __launch_bounds__(kThreads) val_prepare_kernel(const PrepArgs p) {
  pdl_entry();
  const int rows = p.bs * p.max_det;
  const int total = max(rows, p.nt);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    if (i < rows) {
      const int img = i / p.max_det, d = i - img * p.max_det;
      const int n = p.det_count ? min(max(p.det_count[img], 0), p.max_det) : p.max_det;
      if (d == 0) p.acc_count[img] = n;
      float b[6] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
      if (d < n) {
        const float* q = p.det + static_cast<size_t>(i) * 6;
        for (int k = 0; k < 6; ++k) b[k] = q[k];
        if (p.single_cls) b[5] = 0.0f;
        scale4(b, p.img + img * 5);
      }
      float* o = p.det_native + static_cast<size_t>(i) * 6;
      for (int k = 0; k < 6; ++k) o[k] = b[k];
      p.acc_conf[i] = b[4];
      p.acc_cls[i] = b[5];
    }
    if (i < p.nt) {
      const float* q = p.targets + static_cast<size_t>(i) * 6;
      const int img = static_cast<int>(q[0]);
      // targets[:, 2:] *= (w, h, w, h) (val.py:371), then xywh2xyxy: xy -/+ wh / 2
      const float x = __fmul_rn(q[2], p.img_w), y = __fmul_rn(q[3], p.img_h);
      const float hw = __fdiv_rn(__fmul_rn(q[4], p.img_w), 2.0f), hh = __fdiv_rn(__fmul_rn(q[5], p.img_h), 2.0f);
      float b[4] = {__fsub_rn(x, hw), __fsub_rn(y, hh), __fadd_rn(x, hw), __fadd_rn(y, hh)};
      if (img >= 0 && img < p.bs) scale4(b, p.img + img * 5);
      float* o = p.labels_native + static_cast<size_t>(i) * 6;
      o[0] = q[0];
      o[1] = q[1];
      for (int k = 0; k < 4; ++k) o[2 + k] = b[k];
      p.acc_tcls[i] = static_cast<int>(q[1]);  // np.bincount(stats[3].astype(int))
    }
  }
}

// ConfusionMatrix.process_batch for every image of a batch: grid (bs), labels of the image staged in shared memory in index
// order (as val_match_kernel).  Detections with conf > conf_thres keep their best label (IoU > iou_thres, class ignored,
// lower label index on bit-equal IoU); each label keeps its best detection among those (lower detection index on a tie).
struct CmArgs {
  const float* det;
  const int32_t* det_count;
  int max_det;
  const float* labels;
  int nl, nc;
  float conf, iou_thres, eps;
  unsigned long long* matrix;  // [nc + 1, nc + 1], [predicted, true]
};

__global__ void __launch_bounds__(kThreads) confusion_kernel(const CmArgs p) {
  __shared__ float4 s_box[kMaxLabels];
  __shared__ int s_cls[kMaxLabels];
  __shared__ unsigned long long s_win[kMaxLabels];  // (IoU bits << 32) | ~detection of the label's best detection, 0: none
  __shared__ int s_n, s_matched;
  __shared__ int s_wcnt[kThreads / 32];
  pdl_entry();
  const int img = blockIdx.x;
  const int n = p.det_count ? min(max(p.det_count[img], 0), p.max_det) : p.max_det;
  if (threadIdx.x == 0) s_n = s_matched = 0;
  __syncthreads();
  for (int base = 0; base < p.nl; base += blockDim.x) {
    const int l = base + threadIdx.x;
    const bool mine = l < p.nl && static_cast<int>(p.labels[static_cast<size_t>(l) * 6]) == img;
    const unsigned bal = __ballot_sync(0xffffffffu, mine);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) s_wcnt[warp] = __popc(bal);
    __syncthreads();
    int off = s_n;
    for (int w = 0; w < warp; ++w) off += s_wcnt[w];
    const int at = off + __popc(bal & ((1u << lane) - 1u));
    if (mine && at < kMaxLabels) {
      const float* q = p.labels + static_cast<size_t>(l) * 6;
      s_cls[at] = static_cast<int>(q[1]);
      s_box[at] = make_float4(q[2], q[3], q[4], q[5]);
      s_win[at] = 0ull;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < kThreads / 32; ++w) tot += s_wcnt[w];
      s_n += tot;
    }
    __syncthreads();
  }
  const int m = min(s_n, kMaxLabels);
  if (m == 0) return;  // val.py calls process_batch only for images with labels
  const float* det = p.det + static_cast<size_t>(img) * p.max_det * 6;
  const int nc = p.nc, ld = nc + 1;
  auto add = [&](int r, int c) {
    if (r >= 0 && r <= nc && c >= 0 && c <= nc) atomicAdd(p.matrix + static_cast<size_t>(r) * ld + c, 1ull);
  };
  auto best_label = [&](int d, float* iou) -> int {
    const float* q = det + static_cast<size_t>(d) * 6;
    if (!(q[4] > p.conf)) return -1;
    const float4 b = make_float4(q[0], q[1], q[2], q[3]);
    float best = 0.0f;
    int bl = -1;
    for (int l = 0; l < m; ++l) {
      const float v = iou_ld(s_box[l], b, p.eps);
      if (v > p.iou_thres && (bl < 0 || v > best)) {
        best = v;
        bl = l;
      }
    }
    *iou = best;
    return bl;
  };
  for (int d = threadIdx.x; d < n; d += blockDim.x) {
    float v;
    const int bl = best_label(d, &v);
    if (bl >= 0) atomicMax(&s_win[bl], (static_cast<unsigned long long>(__float_as_uint(v)) << 32) | (0xffffffffu - d));
  }
  __syncthreads();
  for (int l = threadIdx.x; l < m; l += blockDim.x) {
    if (s_win[l]) {
      const int d = static_cast<int>(0xffffffffu - static_cast<uint32_t>(s_win[l]));
      add(static_cast<int>(det[static_cast<size_t>(d) * 6 + 5]), s_cls[l]);
      s_matched = 1;
    } else {
      add(nc, s_cls[l]);  // true background
    }
  }
  __syncthreads();
  if (!s_matched) return;  // `if n:` (utils/metrics.py:175): unmatched detections count only when the image has a match
  for (int d = threadIdx.x; d < n; d += blockDim.x) {
    float v;
    const float* q = det + static_cast<size_t>(d) * 6;
    if (!(q[4] > p.conf)) continue;
    const int bl = best_label(d, &v);
    if (bl < 0 || static_cast<int>(0xffffffffu - static_cast<uint32_t>(s_win[bl])) != d) add(static_cast<int>(q[5]), nc);
  }
}

// ------------------------------------------------------------------------------------------------ workspace layout
struct ApLayout {
  size_t key[2], idx[2], tile_hist, P, S, tile_sum, agg_seg, agg_val, start, total;
  int ntiles;
};
inline size_t align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }
ApLayout ap_layout(int n, int nc, int niou) {
  ApLayout L;
  L.ntiles = n > 0 ? (n + kTile - 1) / kTile : 0;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    const size_t at = o;
    o += align256(bytes);
    return at;
  };
  const size_t nn = static_cast<size_t>(n), nt = static_cast<size_t>(L.ntiles), ni = static_cast<size_t>(niou);
  L.key[0] = take(nn * 8);
  L.key[1] = take(nn * 8);
  L.idx[0] = take(nn * 4);
  L.idx[1] = take(nn * 4);
  L.tile_hist = take(256 * nt * 4);
  L.P = take(ni * nn * 4);
  L.S = take(ni * nn * 8);
  L.tile_sum = take(ni * nt * 4);
  L.agg_seg = take(ni * nt * 4);
  L.agg_val = take(ni * nt * 8);
  L.start = take((static_cast<size_t>(nc) + 2) * 4);
  L.total = o;
  return L;
}

}  // namespace
}  // namespace y3

#define Y3_LAUNCH(kern, grid, block, stream, ...) \
  Y3_CHECK_CUDA(::y3::launch_pdl(kern, grid, block, 0, stream, __VA_ARGS__))

extern "C" int64_t y3_ap_workspace_bytes(int32_t n_rows, int32_t nc, int32_t niou) {
  if (n_rows < 0 || nc < 1 || nc > y3::kMaxNc || niou < 1 || niou > 64) return -1;
  return static_cast<int64_t>(y3::ap_layout(n_rows, nc, niou).total);
}

extern "C" int y3_ap_per_class(const float* conf, const float* cls, const uint8_t* tp, const int32_t* counts, int32_t n_images,
                               int32_t stride, int32_t niou, const int32_t* tcls, int32_t n_labels, int32_t nc, const double* px,
                               const double* xap, void* workspace, int64_t workspace_bytes, int32_t* npred, int32_t* nt,
                               int32_t* info, double* ap, double* curves, double* best, y3_stream_t stream) {
  Y3_REQUIRE(n_images >= 0 && stride >= 0 && n_labels >= 0 && nc >= 1 && nc <= y3::kMaxNc && niou >= 1 && niou <= 64,
             "ap_per_class: bad shape (images %d, stride %d, labels %d, nc %d, niou %d)", n_images, stride, n_labels, nc, niou);
  const long long n64 = static_cast<long long>(n_images) * stride;
  Y3_REQUIRE(n64 < (1ll << 30), "ap_per_class: %lld rows (limit 2^30)", n64);
  const int n = static_cast<int>(n64);
  Y3_REQUIRE(px && xap && npred && nt && info && ap && curves && best, "ap_per_class: null pointer");
  Y3_REQUIRE(n == 0 || (conf && cls && tp), "ap_per_class: null row pointer");
  Y3_REQUIRE(n_labels == 0 || tcls, "ap_per_class: null label pointer");
  const y3::ApLayout L = y3::ap_layout(n, nc, niou);
  Y3_REQUIRE(workspace && workspace_bytes >= static_cast<int64_t>(L.total), "ap_per_class: workspace too small (%lld < %lld)",
             static_cast<long long>(workspace_bytes), static_cast<long long>(L.total));
  char* ws = static_cast<char*>(workspace);
  y3::ApArgs a;
  a.conf = conf;
  a.cls = cls;
  a.tp = tp;
  a.counts = counts;
  a.n = n;
  a.stride = stride;
  a.niou = niou;
  a.tcls = tcls;
  a.nl = n_labels;
  a.nc = nc;
  a.px = px;
  a.xap = xap;
  for (int b = 0; b < 2; ++b) {
    a.key[b] = reinterpret_cast<unsigned long long*>(ws + L.key[b]);
    a.idx[b] = reinterpret_cast<int*>(ws + L.idx[b]);
  }
  a.tile_hist = reinterpret_cast<int*>(ws + L.tile_hist);
  a.P = reinterpret_cast<int*>(ws + L.P);
  a.S = reinterpret_cast<double*>(ws + L.S);
  a.tile_sum = reinterpret_cast<int*>(ws + L.tile_sum);
  a.agg_seg = reinterpret_cast<int*>(ws + L.agg_seg);
  a.agg_val = reinterpret_cast<double*>(ws + L.agg_val);
  a.start = reinterpret_cast<int*>(ws + L.start);
  a.ntiles = L.ntiles;
  a.npred = npred;
  a.nt = nt;
  a.info = info;
  a.ap = ap;
  a.curves = curves;
  a.best = best;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int T = y3::kThreads;
  Y3_LAUNCH(y3::ap_init_kernel, dim3((nc + T) / T), dim3(T), st, a);
  const int work = n > n_labels ? n : n_labels;
  const int cap = y3::num_sms() * 4;
  const int cblocks = work > 0 ? ((work + T - 1) / T < cap ? (work + T - 1) / T : cap) : 1;
  Y3_LAUNCH(y3::ap_count_kernel, dim3(cblocks), dim3(T), st, a);
  Y3_LAUNCH(y3::ap_start_kernel, dim3(1), dim3(1024), st, a);
  int cur = 0;
  if (n > 0) {
    // 32 confidence bits, then the class (values 0..nc, nc = "no class"): one 8-bit digit below 256, else two
    const int passes = 4 + (nc < 256 ? 1 : 2);
    for (int ps = 0; ps < passes; ++ps) {
      const int shift = 8 * ps;
      Y3_LAUNCH(y3::radix_hist_kernel, dim3(L.ntiles), dim3(T), st, static_cast<const unsigned long long*>(a.key[cur]), n, shift,
                a.tile_hist, L.ntiles);
      Y3_LAUNCH(y3::scan_rows_kernel, dim3(1), dim3(1024), st, a.tile_hist, 256 * L.ntiles, 0);
      Y3_LAUNCH(y3::radix_scatter_kernel, dim3(L.ntiles), dim3(T), st, static_cast<const unsigned long long*>(a.key[cur]),
                static_cast<const int*>(a.idx[cur]), a.key[cur ^ 1], a.idx[cur ^ 1], n, shift,
                static_cast<const int*>(a.tile_hist), L.ntiles);
      cur ^= 1;
    }
    const unsigned long long* key = a.key[cur];
    const int* idx = a.idx[cur];
    Y3_LAUNCH(y3::ap_tile_sum_kernel, dim3(L.ntiles, niou), dim3(T), st, a, key, idx);
    Y3_LAUNCH(y3::scan_rows_kernel, dim3(niou), dim3(1024), st, a.tile_sum, L.ntiles, L.ntiles);
    Y3_LAUNCH(y3::ap_prefix_kernel, dim3(L.ntiles, niou), dim3(T), st, a, key, idx);
    Y3_LAUNCH(y3::ap_tile_max_kernel, dim3(L.ntiles, niou), dim3(T), st, a, key);
    Y3_LAUNCH(y3::ap_tile_carry_kernel, dim3(niou), dim3(1024), st, a);
    Y3_LAUNCH(y3::ap_suffix_kernel, dim3(L.ntiles, niou), dim3(T), st, a, key);
  }
  Y3_LAUNCH(y3::ap_ap_kernel, dim3(nc, niou), dim3(128), st, a);
  Y3_LAUNCH(y3::ap_curves_kernel, dim3(nc), dim3(T), st, a, static_cast<const unsigned long long*>(a.key[cur]),
            static_cast<const int*>(a.idx[cur]));
  Y3_LAUNCH(y3::ap_final_kernel, dim3(1), dim3(1024), st, a);
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_val_prepare(const float* det, const int32_t* det_count, int32_t bs, int32_t max_det, const float* img_params,
                              int32_t single_cls, const float* targets, int32_t nt, float img_w, float img_h,
                              float* det_native, float* labels_native, float* acc_conf, float* acc_cls, int32_t* acc_count,
                              int32_t* acc_tcls, y3_stream_t stream) {
  Y3_REQUIRE(bs >= 1 && max_det >= 1 && nt >= 0, "val_prepare: bad shape (bs %d, max_det %d, nt %d)", bs, max_det, nt);
  const long long rows = static_cast<long long>(bs) * max_det;
  Y3_REQUIRE(rows < (1ll << 31), "val_prepare: %lld rows", rows);
  const long long total = rows > nt ? rows : nt;
  Y3_REQUIRE(det && img_params && acc_count && det_native && acc_conf && acc_cls && (nt == 0 || (targets && labels_native && acc_tcls)),
             "val_prepare: null pointer");
  y3::PrepArgs p;
  p.det = det;
  p.det_count = det_count;
  p.bs = bs;
  p.max_det = max_det;
  p.img = img_params;
  p.single_cls = single_cls;
  p.targets = targets;
  p.nt = nt;
  p.img_w = img_w;
  p.img_h = img_h;
  p.det_native = det_native;
  p.labels_native = labels_native;
  p.acc_conf = acc_conf;
  p.acc_cls = acc_cls;
  p.acc_count = acc_count;
  p.acc_tcls = acc_tcls;
  long long blocks = (total + y3::kThreads - 1) / y3::kThreads;
  const long long cap = static_cast<long long>(y3::num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  Y3_LAUNCH(y3::val_prepare_kernel, dim3(static_cast<unsigned>(blocks)), dim3(y3::kThreads), static_cast<cudaStream_t>(stream), p);
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_confusion_update(const float* det, const int32_t* det_count, int32_t bs, int32_t max_det, const float* labels,
                                   int32_t nl, int32_t nc, float conf_thres, float iou_thres, float eps,
                                   unsigned long long* matrix, y3_stream_t stream) {
  Y3_REQUIRE(bs >= 0 && max_det >= 0 && nl >= 0 && nc >= 1 && nc <= y3::kMaxNc, "confusion_update: bad shape");
  if (bs == 0 || nl == 0) return Y3_OK;
  Y3_REQUIRE(labels && matrix && (max_det == 0 || det), "confusion_update: null pointer");
  y3::CmArgs p;
  p.det = det;
  p.det_count = det_count;
  p.max_det = max_det;
  p.labels = labels;
  p.nl = nl;
  p.nc = nc;
  p.conf = conf_thres;
  p.iou_thres = iou_thres;
  p.eps = eps;
  p.matrix = matrix;
  Y3_LAUNCH(y3::confusion_kernel, dim3(bs), dim3(y3::kThreads), static_cast<cudaStream_t>(stream), p);
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
