// yolov3_b200 — AutoAnchor (utils/autoanchor.py:26-164, train.py:316) on the device: the anchor metric of check_anchors and
// print_results, scipy.cluster.vq.kmeans with all restarts run at once, and kmean_anchors' genetic evolution.
//   metric:    r = wh / k, x = min(r, 1 / r).min(coords), best = x.max(anchors): NaN-propagating like torch, fp32 or fp64,
//              the threshold compared in the same precision (torch rounds a Python float to the tensor's dtype);
//              the counts BPR and AAT rest on are exact integers, the sums print_results logs are fp64.
//   k-means:   vq, update_cluster_means and numpy's fp32 mean of the distortions, bit for bit: the codebook, distortion,
//              iteration count and dropped clusters of every restart are scipy's.  One pass = assignment + leaf sums of
//              numpy's pairwise tree (one thread per leaf, all restarts) and one block per restart for the rest.
//   evolution: the fitness mean(best * (best > fp32(thr))) summed exactly in fixed point (uint64 in units of 2^-32,
//              exact for fp32(thr) >= 2^-9 because every fp32 above 2^-9 is a multiple of 2^-32), rounded to fp32 once and
//              divided by N;
//              the generations run in order on the stream, each a fitness launch and a one-thread accept launch.
// Separately rounded IEEE operations throughout (compiled with -fmad=false, no fast math).
#include "y3_common.cuh"
#include "y3_internal.h"

#include <algorithm>
#include <vector>

namespace y3 {
namespace {

constexpr int kMaxAnchors = 32;   // anchors of the metric / evolution, codes of the k-means
constexpr int kMaxRestarts = 64;
constexpr int kLeaf = 128;        // numpy's PW_BLOCKSIZE
constexpr int kRunning = 0, kFinal = 1, kDone = 2;

template <typename T>
__device__ __forceinline__ T nan_min(T a, T b) { return a != a ? a : (b != b ? b : (b < a ? b : a)); }
template <typename T>
__device__ __forceinline__ T nan_max(T a, T b) { return a != a ? a : (b != b ? b : (b > a ? b : a)); }
__device__ __forceinline__ float rdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double rdiv(double a, double b) { return __ddiv_rn(a, b); }

// x of one anchor: min(r, 1 / r) over both coordinates, r = wh / k (torch.min(r, 1 / r).min(2))
template <typename T>
__device__ __forceinline__ T ratio_x(T w, T h, T kw, T kh) {
  const T rw = rdiv(w, kw), rh = rdiv(h, kh);
  return nan_min(nan_min(rw, rdiv(T(1), rw)), nan_min(rh, rdiv(T(1), rh)));
}

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[w] = v;
  __syncthreads();
  T s = T(0);
  if (threadIdx.x == 0)
    for (int i = 0; i < nw; ++i) s += sh[i];
  return s;  // thread 0 only
}

// ---------------------------------------------------------------------------------------------------------- metric
// counts[0] += #(best > thr), counts[1] += #(x > thr) over every anchor; sums[0..2] += sum x, sum best, sum of x > thr
template <typename T>
__global__ void __launch_bounds__(256) metric_kernel(const float2* __restrict__ wh, long long n, const double* __restrict__ k,
                                                     int na, double thr, unsigned long long* counts, double* sums) {
  __shared__ T sk[2 * kMaxAnchors];
  __shared__ unsigned long long shu[8];
  __shared__ double shd[8];
  for (int t = threadIdx.x; t < 2 * na; t += blockDim.x) sk[t] = static_cast<T>(k[t]);
  __syncthreads();
  const T t_thr = static_cast<T>(thr);
  unsigned long long c_best = 0, c_x = 0;
  double s_x = 0, s_best = 0, s_past = 0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float2 p = wh[i];
    T best = T(0);
    for (int a = 0; a < na; ++a) {
      const T x = ratio_x(static_cast<T>(p.x), static_cast<T>(p.y), sk[2 * a], sk[2 * a + 1]);
      best = a == 0 ? x : nan_max(best, x);
      s_x += static_cast<double>(x);
      if (x > t_thr) {
        ++c_x;
        s_past += static_cast<double>(x);
      }
    }
    s_best += static_cast<double>(best);
    if (best > t_thr) ++c_best;
  }
  const unsigned long long b0 = block_sum(c_best, shu), b1 = block_sum(c_x, shu);
  const double d0 = block_sum(s_x, shd), d1 = block_sum(s_best, shd), d2 = block_sum(s_past, shd);
  if (threadIdx.x == 0) {
    atomicAdd(counts, b0);
    atomicAdd(counts + 1, b1);
    atomicAdd(sums, d0);
    atomicAdd(sums + 1, d1);
    atomicAdd(sums + 2, d2);
  }
}

// ---------------------------------------------------------------------------------------------------------- evolution
struct EvolveState {
  unsigned long long acc[2];  // fixed-point sum of best * (best > thr) (units of 2^-32), NaN count
  double k[2 * kMaxAnchors];  // current anchors (fp64, as kmean_anchors keeps k after the first acceptance)
  double kg[2 * kMaxAnchors]; // candidate
  float kg32[2 * kMaxAnchors];  // candidate rounded to fp32 (torch.tensor(kg, dtype=torch.float32))
  float f;                    // current fitness
};

__global__ void __launch_bounds__(256) fitness_kernel(const float2* __restrict__ wh, long long n, int na, double thr,
                                                      EvolveState* st) {
  __shared__ float sk[2 * kMaxAnchors];
  __shared__ unsigned long long sh[8];
  for (int t = threadIdx.x; t < 2 * na; t += blockDim.x) sk[t] = st->kg32[t];
  __syncthreads();
  const float t_thr = static_cast<float>(thr);  // best > thr: torch compares an fp32 tensor in fp32
  unsigned long long s = 0, nan = 0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float2 p = wh[i];
    float best = ratio_x(p.x, p.y, sk[0], sk[1]);
    for (int a = 1; a < na; ++a) best = nan_max(best, ratio_x(p.x, p.y, sk[2 * a], sk[2 * a + 1]));
    if (best != best) ++nan;
    else if (best > t_thr) s += __float2ull_rn(__fmul_rn(best, 4294967296.0f));  // exact: best > 2^-9
  }
  const unsigned long long bs = block_sum(s, sh), bn = block_sum(nan, sh);
  if (threadIdx.x == 0) {
    if (bs) atomicAdd(&st->acc[0], bs);
    if (bn) atomicAdd(&st->acc[1], bn);
  }
}

__device__ __forceinline__ void set_candidate(EvolveState* st, int i, double kg) {
  st->kg[i] = kg;
  st->kg32[i] = __double2float_rn(kg);
}

__global__ void evolve_init_kernel(EvolveState* st, const double* __restrict__ k0, int na) {
  st->acc[0] = st->acc[1] = 0;
  for (int i = 0; i < 2 * na; ++i) {
    st->k[i] = k0[i];
    set_candidate(st, i, k0[i]);
  }
}

// decides generation g (g = -1: the initial fitness) from the fitness just summed, then forms generation g + 1's
// candidate kg = (k * v).clip(min=2.0) (np.clip propagates NaN)
__global__ void evolve_step_kernel(EvolveState* st, const double* __restrict__ v, int g, int gen, int na, long long n,
                                   float* __restrict__ fit, uint8_t* __restrict__ accepted) {
  const unsigned long long s = st->acc[0], nan = st->acc[1];
  st->acc[0] = st->acc[1] = 0;
  const float fg = nan ? __int_as_float(0x7fc00000)
                       : __fdiv_rn(__fmul_rn(__ull2float_rn(s), 2.3283064365386963e-10f), __ll2float_rn(n));
  fit[g + 1] = fg;
  if (g < 0) {
    st->f = fg;
  } else {
    const bool acc = fg > st->f;
    accepted[g] = acc;
    if (acc) {
      st->f = fg;
      for (int i = 0; i < 2 * na; ++i) st->k[i] = st->kg[i];
    }
  }
  if (g + 1 < gen) {
    const double* vg = v + static_cast<size_t>(g + 1) * 2 * na;
    for (int i = 0; i < 2 * na; ++i) {
      const double kg = __dmul_rn(st->k[i], vg[i]);
      set_candidate(st, i, kg < 2.0 ? 2.0 : kg);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- k-means
// numpy's pairwise_sum over n fp32 values: n < 8 summed in order from 0; n <= 128 in eight strided accumulators combined as
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the n % 8 tail in order; larger n split at n2 = n / 2 - (n / 2) % 8.
// The tree depends on n alone: node j of depth d is heap slot 2^d - 1 + j.  Every leaf starts at a multiple of 8.
__host__ __device__ __forceinline__ long long pw_split(long long n) { return n / 2 - (n / 2) % 8; }

// depth of the deepest leaf, level by level over the few distinct node sizes of each level
int pw_depth(long long n) {
  std::vector<long long> level{n};
  int d = 0;
  for (;; ++d) {
    std::vector<long long> next;
    for (long long m : level)
      if (m > kLeaf) {
        next.push_back(pw_split(m));
        next.push_back(m - pw_split(m));
      }
    if (next.empty()) return d;
    std::sort(next.begin(), next.end());
    next.erase(std::unique(next.begin(), next.end()), next.end());
    level.swap(next);
  }
}

// the node of heap path `path` (depth `d`, bits read from the top) if it exists: its start and size; false if an ancestor
// is a leaf
__device__ __forceinline__ bool pw_node(long long n, int d, long long path, long long* start, long long* size) {
  long long s = 0, m = n;
  for (int q = d - 1; q >= 0; --q) {
    if (m <= kLeaf) return false;
    const long long m2 = pw_split(m);
    if ((path >> q) & 1) {
      s += m2;
      m -= m2;
    } else {
      m = m2;
    }
  }
  *start = s;
  *size = m;
  return true;
}

// node kinds of the heap: 0 absent, 1 leaf, 2 internal
__global__ void __launch_bounds__(256) pw_kinds_kernel(long long n, int depth, uint8_t* __restrict__ kind) {
  const long long slots = (2LL << depth) - 1;
  for (long long h = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; h < slots;
       h += static_cast<long long>(gridDim.x) * blockDim.x) {
    int d = 0;
    while ((2LL << d) - 1 <= h) ++d;
    long long s, m;
    kind[h] = pw_node(n, d, h - ((1LL << d) - 1), &s, &m) ? (m <= kLeaf ? 1 : 2) : 0;
  }
}

struct KmArgs {
  const float2* obs;
  long long n;
  int restarts, k, depth;
  float2* book;       // [restarts][k]: the current codebook, its first ncode[r] codes valid
  int* ncode;         // [restarts]
  int* status;        // [restarts]: kRunning, kFinal (the codebook has converged: one more vq for the final distortion), kDone
  float* dist;        // [restarts]: mean distortion of the final vq
  float* prev;        // [restarts]: mean distortion of the previous pass (+inf before the first)
  int* passes;        // [restarts]: vq passes run, the final one included
  uint8_t* code;      // [restarts][n]
  float* heap;        // [restarts][2^(depth+1) - 1]: pairwise-tree node sums
  const uint8_t* kind;  // [2^(depth+1) - 1]
};

__global__ void km_init_kernel(KmArgs a, const long long* __restrict__ idx) {
  const int r = blockIdx.x;
  for (int j = threadIdx.x; j < a.k; j += blockDim.x) a.book[r * a.k + j] = a.obs[idx[r * a.k + j]];
  if (threadIdx.x == 0) {
    a.ncode[r] = a.k;
    a.status[r] = kRunning;
    a.prev[r] = __int_as_float(0x7f800000);
    a.passes[r] = 0;
  }
}

// vq of one point: first code of the strictly smallest (c0 - o0)^2 + (c1 - o1)^2, distance sqrt of it
__device__ __forceinline__ float vq_point(const float2 o, const float2* cb, int nc, uint8_t* code) {
  float low = __int_as_float(0x7f800000);
  int c = 0;
  for (int j = 0; j < nc; ++j) {
    const float dx = __fsub_rn(cb[j].x, o.x), dy = __fsub_rn(cb[j].y, o.y);
    const float d = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
    if (d < low) {
      low = d;
      c = j;
    }
  }
  *code = static_cast<uint8_t>(c);
  return __fsqrt_rn(low);
}

// one thread per heap slot of the deepest level; the first slot under each leaf assigns the leaf's points for every live
// restart and stores the leaf's pairwise sum of the distances
__global__ void __launch_bounds__(128) km_assign_kernel(KmArgs a) {
  extern __shared__ float2 s_book[];  // [restarts][k]
  __shared__ int s_nc[kMaxRestarts], s_live[kMaxRestarts];
  for (int t = threadIdx.x; t < a.restarts * a.k; t += blockDim.x) s_book[t] = a.book[t];
  for (int t = threadIdx.x; t < a.restarts; t += blockDim.x) {
    s_nc[t] = a.ncode[t];
    s_live[t] = a.status[t] != kDone;
  }
  __syncthreads();
  const long long path = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (path >= (1LL << a.depth)) return;
  // the leaf above this slot, owned by its leftmost slot
  long long s = 0, m = a.n, node = 0;
  int d = 0;
  for (; d < a.depth && m > kLeaf; ++d) {
    const long long m2 = pw_split(m);
    const int bit = (path >> (a.depth - 1 - d)) & 1;
    if (bit) {
      s += m2;
      m -= m2;
    } else {
      m = m2;
    }
    node = 2 * node + 1 + bit;
  }
  if (path & ((1LL << (a.depth - d)) - 1)) return;
  const size_t hslots = (2ull << a.depth) - 1;
  for (int r = 0; r < a.restarts; ++r) {
    if (!s_live[r]) continue;
    const float2* cb = s_book + r * a.k;
    const int nc = s_nc[r];
    uint8_t* code = a.code + static_cast<size_t>(r) * a.n + s;
    const float2* o = a.obs + s;
    const int len = static_cast<int>(m);
    float res;
    if (len < 8) {
      res = 0.f;
      for (int i = 0; i < len; ++i) res = __fadd_rn(res, vq_point(o[i], cb, nc, code + i));
    } else {
      float acc[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[q] = vq_point(o[q], cb, nc, code + q);
      int i = 8;
      for (; i < len - (len % 8); i += 8) {
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = __fadd_rn(acc[q], vq_point(o[i + q], cb, nc, code + i + q));
      }
      res = __fadd_rn(__fadd_rn(__fadd_rn(acc[0], acc[1]), __fadd_rn(acc[2], acc[3])),
                      __fadd_rn(__fadd_rn(acc[4], acc[5]), __fadd_rn(acc[6], acc[7])));
      for (; i < len; ++i) res = __fadd_rn(res, vq_point(o[i], cb, nc, code + i));
    }
    a.heap[r * hslots + node] = res;
  }
}

// one block (32 warps) per live restart: the pairwise tree's internal nodes, then (when the restart is still running) the
// cluster means — warp c walks the points in order and adds the members of cluster c to one serial fp32 chain per
// coordinate, as update_cluster_means does — then the dropped clusters, the distortion-change test and the status
constexpr int kUpdThreads = 1024;
__global__ void __launch_bounds__(kUpdThreads) km_update_kernel(KmArgs a, float thresh) {
  const int r = blockIdx.x;
  if (a.status[r] == kDone) return;
  const size_t hslots = (2ull << a.depth) - 1;
  float* heap = a.heap + r * hslots;
  for (int d = a.depth - 1; d >= 0; --d) {
    const long long lo = (1LL << d) - 1, hi = (2LL << d) - 1;
    for (long long h = lo + threadIdx.x; h < hi; h += blockDim.x)
      if (a.kind[h] == 2) heap[h] = __fadd_rn(heap[2 * h + 1], heap[2 * h + 2]);
    __syncthreads();
  }
  __shared__ float s_mean;
  __shared__ int s_conv;
  __shared__ float2 s_sum[kMaxAnchors];
  __shared__ long long s_cnt[kMaxAnchors];
  const int status = a.status[r];
  if (threadIdx.x == 0) {
    const float mean = __fdiv_rn(heap[0], __ll2float_rn(a.n));
    s_mean = mean;
    a.passes[r] += 1;
    if (status == kRunning) {
      const float diff = fabsf(__fsub_rn(a.prev[r], mean));
      s_conv = !(diff > thresh);
      a.prev[r] = mean;
    }
  }
  __syncthreads();
  if (status == kFinal) {
    if (threadIdx.x == 0) {
      a.dist[r] = s_mean;
      a.status[r] = kDone;
    }
    return;
  }
  const int nc = a.ncode[r], warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < nc) {
    const uint8_t* code = a.code + static_cast<size_t>(r) * a.n;
    float sx = 0.f, sy = 0.f;
    long long cnt = 0;
    for (long long base = 0; base < a.n; base += 32) {
      const long long i = base + lane;
      const bool in = i < a.n;
      const float2 o = in ? a.obs[i] : make_float2(0.f, 0.f);
      unsigned mask = __ballot_sync(0xffffffffu, in && code[in ? i : 0] == warp);
      cnt += __popc(mask);
      while (mask) {  // the members in point order, eight shuffles in flight
        int j[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          j[q] = mask ? __ffs(mask) - 1 : -1;
          mask &= mask - 1;
        }
        float vx[8], vy[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          vx[q] = __shfl_sync(0xffffffffu, o.x, j[q] < 0 ? 0 : j[q]);
          vy[q] = __shfl_sync(0xffffffffu, o.y, j[q] < 0 ? 0 : j[q]);
        }
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (j[q] >= 0) {
            sx = __fadd_rn(sx, vx[q]);
            sy = __fadd_rn(sy, vy[q]);
          }
      }
    }
    if (lane == 0) {
      s_sum[warp] = make_float2(sx, sy);
      s_cnt[warp] = cnt;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int kept = 0;
    for (int c = 0; c < nc; ++c) {
      if (s_cnt[c] == 0) continue;
      const float cf = __ll2float_rn(s_cnt[c]);
      a.book[r * a.k + kept++] = make_float2(__fdiv_rn(s_sum[c].x, cf), __fdiv_rn(s_sum[c].y, cf));
    }
    a.ncode[r] = kept;
    if (s_conv) a.status[r] = kFinal;
  }
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

struct KmLayout {
  size_t code, heap, kind, prev, total;
};
KmLayout km_layout(long long n, int restarts, int depth) {
  const size_t hslots = (2ull << depth) - 1;
  KmLayout l;
  l.code = 0;
  l.heap = l.code + align256(static_cast<size_t>(restarts) * n);
  l.kind = l.heap + align256(sizeof(float) * restarts * hslots);
  l.prev = l.kind + align256(hslots);
  l.total = l.prev + align256(sizeof(float) * restarts);
  return l;
}

int grid_for(long long work, int threads) {
  long long b = (work + threads - 1) / threads;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  return static_cast<int>(std::max(1LL, std::min(b, cap)));
}

int km_args(KmArgs* a, const float* obs, int64_t n, int32_t restarts, int32_t k, float* book, int32_t* ncode,
            int32_t* status, float* dist, int32_t* passes, void* ws, int64_t ws_bytes) {
  Y3_REQUIRE(n >= 1 && n < (1LL << 40), "kmeans: bad point count %lld", static_cast<long long>(n));
  Y3_REQUIRE(restarts >= 1 && restarts <= kMaxRestarts, "kmeans: restarts %d not in [1, %d]", restarts, kMaxRestarts);
  Y3_REQUIRE(k >= 1 && k <= kMaxAnchors && k <= n, "kmeans: k %d not in [1, min(%d, n)]", k, kMaxAnchors);
  Y3_REQUIRE(obs && book && ncode && status && dist && passes && ws, "kmeans: null pointer");
  Y3_REQUIRE((reinterpret_cast<uintptr_t>(obs) & 7) == 0 && (reinterpret_cast<uintptr_t>(book) & 7) == 0 &&
                 (reinterpret_cast<uintptr_t>(ws) & 255) == 0,
             "kmeans: obs and book must be 8-byte aligned [., 2] fp32, the workspace 256-byte aligned");
  const int depth = pw_depth(n);
  const KmLayout l = km_layout(n, restarts, depth);
  Y3_REQUIRE(ws_bytes >= static_cast<int64_t>(l.total), "kmeans: workspace of %lld bytes, %lld needed",
             static_cast<long long>(ws_bytes), static_cast<long long>(l.total));
  char* w = static_cast<char*>(ws);
  *a = KmArgs{reinterpret_cast<const float2*>(obs), n, restarts, k, depth, reinterpret_cast<float2*>(book), ncode, status,
              dist, reinterpret_cast<float*>(w + l.prev), passes, reinterpret_cast<uint8_t*>(w + l.code),
              reinterpret_cast<float*>(w + l.heap), reinterpret_cast<const uint8_t*>(w + l.kind)};
  return Y3_OK;
}

}  // namespace
}  // namespace y3

extern "C" int y3_anchor_metric(const float* wh, int64_t n, const double* k, int32_t na, double thr, int32_t fp64,
                                uint64_t* counts, double* sums, y3_stream_t stream) {
  Y3_REQUIRE(n >= 0 && na >= 1 && na <= y3::kMaxAnchors, "anchor_metric: bad shape (n=%lld, anchors=%d)",
             static_cast<long long>(n), na);
  Y3_REQUIRE(wh && k && counts && sums, "anchor_metric: null pointer");
  Y3_REQUIRE((reinterpret_cast<uintptr_t>(wh) & 7) == 0, "anchor_metric: wh must be 8-byte aligned [n, 2] fp32");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Y3_CHECK_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(uint64_t), s));
  Y3_CHECK_CUDA(cudaMemsetAsync(sums, 0, 3 * sizeof(double), s));
  if (n == 0) return Y3_OK;
  const int g = y3::grid_for(n, 256);
  auto* c = reinterpret_cast<unsigned long long*>(counts);
  if (fp64) y3::metric_kernel<double><<<g, 256, 0, s>>>(reinterpret_cast<const float2*>(wh), n, k, na, thr, c, sums);
  else y3::metric_kernel<float><<<g, 256, 0, s>>>(reinterpret_cast<const float2*>(wh), n, k, na, thr, c, sums);
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int64_t y3_anchor_evolve_workspace_bytes(void) { return static_cast<int64_t>(sizeof(y3::EvolveState)); }

extern "C" int y3_anchor_evolve(const float* wh, int64_t n, int32_t na, double thr, const double* k0, const double* v,
                                int32_t gen, double* k_out, float* fit, uint8_t* accepted, void* ws, int64_t ws_bytes,
                                y3_stream_t stream) {
  Y3_REQUIRE(n >= 1 && na >= 1 && na <= y3::kMaxAnchors && gen >= 0, "anchor_evolve: bad shape (n=%lld, anchors=%d, gen=%d)",
             static_cast<long long>(n), na, gen);
  Y3_REQUIRE(n <= (1LL << 31), "anchor_evolve: %lld labels: the fixed-point fitness sum holds at most 2^31",
             static_cast<long long>(n));
  Y3_REQUIRE(static_cast<float>(thr) >= 1.0f / 512 && thr <= 1.0, "anchor_evolve: 1 / anchor_t = %g outside [2^-9, 1]", thr);
  Y3_REQUIRE(wh && k0 && k_out && fit && ws && (gen == 0 || (v && accepted)), "anchor_evolve: null pointer");
  Y3_REQUIRE((reinterpret_cast<uintptr_t>(wh) & 7) == 0 && (reinterpret_cast<uintptr_t>(ws) & 15) == 0,
             "anchor_evolve: wh must be 8-byte aligned [n, 2] fp32, the workspace 16-byte aligned");
  Y3_REQUIRE(ws_bytes >= static_cast<int64_t>(sizeof(y3::EvolveState)), "anchor_evolve: workspace too small");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  auto* st = static_cast<y3::EvolveState*>(ws);
  const auto* p = reinterpret_cast<const float2*>(wh);
  const int g = y3::grid_for(n, 256);
  y3::evolve_init_kernel<<<1, 1, 0, s>>>(st, k0, na);
  for (int i = -1; i < gen; ++i) {
    y3::fitness_kernel<<<g, 256, 0, s>>>(p, n, na, thr, st);
    y3::evolve_step_kernel<<<1, 1, 0, s>>>(st, v, i, gen, na, n, fit, accepted);
  }
  Y3_CHECK_CUDA(cudaGetLastError());
  Y3_CHECK_CUDA(cudaMemcpyAsync(k_out, st->k, 2 * na * sizeof(double), cudaMemcpyDeviceToDevice, s));
  return Y3_OK;
}

extern "C" int64_t y3_kmeans_workspace_bytes(int64_t n, int32_t restarts) {
  if (n < 1 || restarts < 1 || restarts > y3::kMaxRestarts) return -1;
  return static_cast<int64_t>(y3::km_layout(n, restarts, y3::pw_depth(n)).total);
}

extern "C" int y3_kmeans_init(const float* obs, int64_t n, int32_t restarts, int32_t k, const int64_t* init_idx, float* book,
                              int32_t* ncode, int32_t* status, float* dist, int32_t* passes, void* ws, int64_t ws_bytes,
                              y3_stream_t stream) {
  y3::KmArgs a;
  if (int rc = y3::km_args(&a, obs, n, restarts, k, book, ncode, status, dist, passes, ws, ws_bytes)) return rc;
  Y3_REQUIRE(init_idx, "kmeans: null pointer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long slots = (2LL << a.depth) - 1;
  y3::pw_kinds_kernel<<<y3::grid_for(slots, 256), 256, 0, s>>>(n, a.depth, const_cast<uint8_t*>(a.kind));
  y3::km_init_kernel<<<restarts, 32, 0, s>>>(a, reinterpret_cast<const long long*>(init_idx));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_kmeans_pass(const float* obs, int64_t n, int32_t restarts, int32_t k, float thresh, float* book,
                              int32_t* ncode, int32_t* status, float* dist, int32_t* passes, void* ws, int64_t ws_bytes,
                              y3_stream_t stream) {
  y3::KmArgs a;
  if (int rc = y3::km_args(&a, obs, n, restarts, k, book, ncode, status, dist, passes, ws, ws_bytes)) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long slots = 1LL << a.depth;
  const size_t smem = sizeof(float2) * restarts * k;
  y3::km_assign_kernel<<<static_cast<unsigned>((slots + 127) / 128), 128, smem, s>>>(a);
  y3::km_update_kernel<<<restarts, y3::kUpdThreads, 0, s>>>(a, thresh);
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
