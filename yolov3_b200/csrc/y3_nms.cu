// yolov3_b200 — batched non-maximum suppression entirely on the device, no host synchronisation.
// Replaces non_max_suppression (reference utils/general.py:630-750) together with torchvision.ops.nms (:733):
//   candidates : obj > thr, conf = obj*cls, best class (or every class > thr when multi_label), class filter
//                -> 64-bit key (conf bits | ~candidate id) and the row's xywh, appended per image (general.py:669-718)
//   bucket     : max_nms cut by key (general.py:728), xywh -> xyxy (general.py:705), counting sort by class into
//                per-(image, class) segments
//   segments   : rank each segment's members by key, greedy suppression of class-offset boxes, strict IoU > thr
//                (general.py:731-732, torchvision nms); segment mask for <= 512 members, segment block above
//   output     : the max_det largest survivor keys in confidence order -> out rows + sources + counts (general.py:734,743)
// Exactness: every floating-point step is a separately rounded fp32 operation in the reference's order (this file is
// compiled with -fmad=false and without fast-math), so kept sets and output rows are bit-identical to the reference on
// identical inputs whenever confidences are tie-free (ties: lower candidate index first, i.e. a stable sort; the
// reference's argsort is unstable there).  Splitting the greedy pass by class is exact because boxes offset by
// class*max_wh cannot intersect across classes while all coordinates lie inside (-max_wh/2, max_wh/2); images that
// violate that bound (or agnostic=True) take the single-segment path over all candidates.
// The reference's wall-clock time_limit break (general.py:675,746-748) is deliberately not reproduced.
#include <cmath>
#include <cstring>

#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {
namespace {

constexpr int kMinCap = 4096;     // smallest candidate capacity per image
constexpr int kRankCap = 32768;   // >= max_nms (30000), power of two
constexpr int kSegSmemBoxes = 2048;

struct NmsArgs {
  const float* pred;  // [bs, n_rows, no]
  int bs, n_rows, nc, no;
  float conf_thres, iou_thres, max_wh;
  double iou_mid;  // midpoint between iou_thres and the next float above it (division-free exact IoU test)
  int iou_odd;     // mantissa LSB of iou_thres: where a quotient exactly at the midpoint rounds to
  int multi_label, agnostic, max_det, max_nms;
  int cap;  // candidate capacity per image (power of two >= kMinCap)
  uint32_t cls_mask[32];
  int use_mask;
  // workspace
  unsigned long long* keys;  // [bs, cap]
  float4* cand_box;          // [bs, cap] (cx, cy, w, h) of the candidate's row, written beside its key (bucketing reads no pred row)
  int* count;                // [bs] candidates found (may exceed cap)
  int* flags;                // [bs] bit0: needs single-segment path
  int* seg_off;                  // [bs, nc + 1] first member of every class segment (conf-unordered members)
  unsigned long long* seg_key2;  // [bs, kRankCap] candidate keys grouped by class
  float4* box4;                  // [bs, kRankCap] xyxy of the member at the same position
  int* surv_cnt;                 // [bs] members that survived the greedy pass
  unsigned long long* surv_key;  // [bs, kRankCap]
  int* surv_pos;                 // [bs, kRankCap] position of the survivor in seg_key2 / box4
  int* done_cnt;                 // [bs] blocks that finished ranking a single-segment image (last one runs the greedy pass)
  uint16_t* ord;                 // [bs, kRankCap] large segments: member index by confidence rank
  // outputs
  float* out;     // [bs, max_det, 6]
  int* out_src;   // [bs, max_det, 2] or null
  int* out_count; // [bs]
  int* overflow;  // [bs] or null
};

__device__ __forceinline__ int next_pow2(int v) { return v <= 1 ? 1 : 1 << (32 - __clz(v - 1)); }

// ------------------------------------------------------------------------------------------------ candidates
// One warp per 32 consecutive prediction rows: the lanes test obj of 32 rows with one strided load, then the warp visits
// only the rows that passed (85 contiguous floats each), and one atomic per warp reserves the key slots.  The first
// version spent a warp, two block barriers and a share of a block atomic on EVERY row and was bound by those serial
// latencies (64 rows in flight per SM).
constexpr int kCandWarps = 8;

__global__ void __launch_bounds__(32 * kCandWarps) nms_candidates_kernel(const NmsArgs p) {
  pdl_entry();
  const unsigned full = 0xffffffffu;
  const int img = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = (blockIdx.x * kCandWarps + warp) * 32;
  if (row0 >= p.n_rows) return;
  const float* base = p.pred + static_cast<size_t>(img) * p.n_rows * p.no;
  const int my_row = row0 + lane;
  float my_obj = 0.f;
  bool pass = false;
  if (my_row < p.n_rows) {
    my_obj = __ldg(base + static_cast<size_t>(my_row) * p.no + 4);
    pass = my_obj > p.conf_thres;
  }
  const unsigned todo = __ballot_sync(full, pass);
  if (todo == 0u) return;
  const unsigned lt_mask = (1u << lane) - 1u;
  int my_cnt = 0;      // candidates of row `lane`
  float my_best = 0.f; // single-label: best conf / class of row `lane`
  int my_c = 0;
  if (p.multi_label) {
    for (unsigned rem = todo; rem; rem &= rem - 1u) {
      const int r = __ffs(rem) - 1;
      const float obj = __shfl_sync(full, my_obj, r);
      const float* x = base + static_cast<size_t>(row0 + r) * p.no + 5;
      int cnt = 0;
      for (int c0 = 0; c0 < p.nc; c0 += 32) {
        const int c = c0 + lane;
        bool ok = false;
        if (c < p.nc) {
          const float conf = __fmul_rn(__ldg(x + c), obj);
          ok = (conf > p.conf_thres) && (!p.use_mask || ((p.cls_mask[c >> 5] >> (c & 31)) & 1u));
        }
        cnt += __popc(__ballot_sync(full, ok));
      }
      if (lane == r) my_cnt = cnt;
    }
  } else {
    // single label: FOUR passing rows per iteration — their class loads are issued back to back before any of the shuffle
    // reductions starts.  One row at a time left a warp with a single 340-byte row in flight and the kernel latency-bound.
    constexpr int kRows = 4;
    for (unsigned rem = todo; rem;) {
      int rr[kRows];
      float obj[kRows], bv[kRows];
      int bc[kRows];
      bool nanv[kRows];
#pragma unroll
      for (int q = 0; q < kRows; ++q) {
        rr[q] = rem ? __ffs(rem) - 1 : -1;
        if (rem) rem &= rem - 1u;
        obj[q] = __shfl_sync(full, my_obj, rr[q] < 0 ? 0 : rr[q]);
        bv[q] = -INFINITY;
        bc[q] = 0x7fffffff;
        nanv[q] = false;
      }
      for (int c = lane; c < p.nc; c += 32) {
        float v[kRows];
#pragma unroll
        for (int q = 0; q < kRows; ++q)
          v[q] = rr[q] >= 0 ? __ldg(base + static_cast<size_t>(row0 + rr[q]) * p.no + 5 + c) : 0.f;
#pragma unroll
        for (int q = 0; q < kRows; ++q) {
          const float conf = __fmul_rn(v[q], obj[q]);
          nanv[q] |= (conf != conf);
          if (conf > bv[q]) {  // first maximum wins inside a lane (ascending c)
            bv[q] = conf;
            bc[q] = c;
          }
        }
      }
      // warp arg-max with two redux.sync per row (value as an order-preserving unsigned key, then the smallest class among the
      // lanes that hold it) instead of a 5-step butterfly of (value, class) shuffle pairs: at conf 0.001 every row comes through
      // here and the 10 shuffles per row were a third of the kernel (one warp shuffle per clock and SM)
#pragma unroll
      for (int q = 0; q < kRows; ++q) {
        uint32_t u = __float_as_uint(bv[q] + 0.0f);  // -0 -> +0: equal as floats, equal as keys
        u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
        const uint32_t umax = __reduce_max_sync(full, u);
        bc[q] = __reduce_min_sync(full, u == umax ? bc[q] : 0x7fffffff);  // first maximum (lowest class) wins, like torch.max
        bv[q] = __uint_as_float((umax & 0x80000000u) ? (umax & 0x7fffffffu) : ~umax);
      }
#pragma unroll
      for (int q = 0; q < kRows; ++q) {
        const float best = __any_sync(full, nanv[q]) ? __int_as_float(0x7fc00000) : bv[q];  // torch.max propagates NaN
        const bool in_set = !p.use_mask || ((p.cls_mask[(bc[q] & 1023) >> 5] >> (bc[q] & 31)) & 1u);
        if (rr[q] >= 0 && lane == rr[q]) {
          my_best = best;
          my_c = bc[q];
          my_cnt = (best > p.conf_thres && in_set) ? 1 : 0;
        }
      }
    }
  }
  // exclusive prefix of my_cnt over the lanes, one atomic for the warp
  int incl = my_cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(full, incl, o);
    if (lane >= o) incl += t;
  }
  const int warp_total = __shfl_sync(full, incl, 31);
  if (warp_total == 0) return;
  int slot0 = 0;
  if (lane == 0) slot0 = atomicAdd(&p.count[img], warp_total);
  slot0 = __shfl_sync(full, slot0, 0);
  const int my_slot = slot0 + incl - my_cnt;
  unsigned long long* keys = p.keys + static_cast<size_t>(img) * p.cap;
  float4* cbox = p.cand_box + static_cast<size_t>(img) * p.cap;
  if (!p.multi_label) {
    if (my_cnt && my_slot < p.cap) {
      const uint32_t id = static_cast<uint32_t>(my_row) * p.nc + my_c;
      keys[my_slot] = (static_cast<unsigned long long>(__float_as_uint(my_best)) << 32) | (0xFFFFFFFFu - id);
      const float* x = base + static_cast<size_t>(my_row) * p.no;  // the row was just read by the warp: L1 / L2 hits
      cbox[my_slot] = make_float4(__ldg(x), __ldg(x + 1), __ldg(x + 2), __ldg(x + 3));
    }
    return;
  }
  for (unsigned rem = __ballot_sync(full, my_cnt > 0); rem; rem &= rem - 1u) {
    const int r = __ffs(rem) - 1;
    const float obj = __shfl_sync(full, my_obj, r);
    int slot = __shfl_sync(full, my_slot, r);
    const float* x = base + static_cast<size_t>(row0 + r) * p.no + 5;
    const float xv = lane < 4 ? __ldg(x - 5 + lane) : 0.f;
    const float4 rbox = make_float4(__shfl_sync(full, xv, 0), __shfl_sync(full, xv, 1), __shfl_sync(full, xv, 2), __shfl_sync(full, xv, 3));
    for (int c0 = 0; c0 < p.nc; c0 += 32) {
      const int c = c0 + lane;
      bool ok = false;
      float conf = 0.f;
      if (c < p.nc) {
        conf = __fmul_rn(__ldg(x + c), obj);
        ok = (conf > p.conf_thres) && (!p.use_mask || ((p.cls_mask[c >> 5] >> (c & 31)) & 1u));
      }
      const unsigned b = __ballot_sync(full, ok);
      const int at = slot + __popc(b & lt_mask);
      if (ok && at < p.cap) {
        const uint32_t id = static_cast<uint32_t>(row0 + r) * p.nc + c;
        keys[at] = (static_cast<unsigned long long>(__float_as_uint(conf)) << 32) | (0xFFFFFFFFu - id);
        cbox[at] = rbox;
      }
      slot += __popc(b);
    }
  }
}

// fdiv_rn(inter, uni) > thr  without the division: the correctly rounded quotient exceeds thr iff the exact quotient lies
// above the midpoint `mid` of thr and its successor (or exactly on it when round-to-nearest-even picks the successor).
// uni has 24 and mid at most 25 significant bits, so uni * mid is exact in double.  Degenerate operands (uni <= 0, NaN,
// infinities) take the IEEE division, which is what torchvision's kernel evaluates.
__device__ __forceinline__ bool iou_exceeds(float inter, float uni, const NmsArgs& p) {
  if (uni > 0.0f && uni < INFINITY && inter < INFINITY) {
    const double a = static_cast<double>(inter), d = __dmul_rn(static_cast<double>(uni), p.iou_mid);
    return a > d || (a == d && p.iou_odd);
  }
  return __fdiv_rn(inter, uni) > p.iou_thres;
}

__device__ __forceinline__ bool box_suppresses(const float4& bi, float ai, const float4& bj, const NmsArgs& p) {
  // disjoint boxes (most pairs) leave after 3-4 instructions per axis: inter = w * h = 0 can never exceed a threshold >= 0,
  // and NaN coordinates do not take these exits (comparisons with NaN are false)
  const float w = fmaxf(0.0f, __fsub_rn(fminf(bi.z, bj.z), fmaxf(bi.x, bj.x)));
  if (w == 0.0f) return false;
  const float h = fmaxf(0.0f, __fsub_rn(fminf(bi.w, bj.w), fmaxf(bi.y, bj.y)));
  if (h == 0.0f) return false;
  const float inter = __fmul_rn(w, h);
  if (inter == 0.0f) return false;  // underflow of w * h
  const float aj = __fmul_rn(__fsub_rn(bj.z, bj.x), __fsub_rn(bj.w, bj.y));
  return iou_exceeds(inter, __fsub_rn(__fadd_rn(ai, aj), inter), p);
}

// ================================================================================================ bucket, segments, output
// No candidate is ever sorted globally: nothing needs a global order except the <= max_det rows that are returned.
//   nms_bucket_kernel    1 CTA/image  max_nms cut (exact radix select, only when count > max_nms), xywh -> xyxy, counting
//                                     sort of the candidates by class (shared-memory histogram + scan + scatter)
//   nms_seg_mask_kernel  1 CTA/(image,class), <= 128 and <= 512 members: rank the members by key (counting in shared memory),
//                                     suppression matrix (intersection bits by ballot, exact division-free IoU on the
//                                     intersecting pairs), one warp resolves the greedy order with bit operations, survivors
//                                     appended to the image's survivor list
//   nms_seg_block_kernel              segments > 512 members (multi-label at low conf; agnostic / out-of-range images, whose
//                                     single segment is ranked by all the image's CTAs and finished by the last one)
//   nms_output_kernel    1 CTA/image  top max_det survivors by key: shared-memory bitonic sort (<= 8192 survivors) or exact
//                                     radix select + sort of the selected, rows + (row, class) sources + counts
// All arithmetic in the reference's order, ties broken by candidate id (stable).
constexpr int kBucketThreads = 1024;
constexpr int kOutSortMax = 8192;  // survivors sorted in shared memory (64 KB keys + 16 KB positions, dynamic)

__device__ __forceinline__ void key_to_rowcls(unsigned long long key, int nc, int& row, int& cls) {
  const uint32_t id = 0xFFFFFFFFu - static_cast<uint32_t>(key & 0xFFFFFFFFull);
  row = static_cast<int>(id / static_cast<uint32_t>(nc));
  cls = static_cast<int>(id - static_cast<uint32_t>(row) * nc);
}

// k-th largest (k >= 1) of n UNIQUE 64-bit keys in global memory, by one CTA: 8 passes over 8-bit digits, MSB first.
// Returns the key itself: exactly k keys are >= it.
__device__ unsigned long long block_select_kth(const unsigned long long* keys, int n, int k, int* s_hist, unsigned long long* s_prefix,
                                               int* s_k) {
  if (threadIdx.x == 0) {
    *s_prefix = 0ull;
    *s_k = k;
  }
  __syncthreads();
  for (int pass = 7; pass >= 0; --pass) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const unsigned long long prefix = *s_prefix;
    const int shift = pass * 8;
    const unsigned long long hi_mask = pass == 7 ? 0ull : (~0ull << (shift + 8));
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned long long v = keys[i];
      if ((v & hi_mask) == prefix) atomicAdd(&s_hist[static_cast<int>((v >> shift) & 0xFFull)], 1);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      // walk down from the largest digit, one warp: lane l owns bins [8l, 8l+8); suffix sums over lanes by shuffle
      const int lane = threadIdx.x;
      int mine = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) mine += s_hist[lane * 8 + q];
      int incl = mine;  // inclusive suffix sum: keys in my bins and in the bins of higher lanes
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_down_sync(0xffffffffu, incl, o);
        if (lane + o < 32) incl += t;
      }
      const int above = incl - mine;
      const int kk0 = *s_k;
      const bool here = above < kk0 && kk0 <= incl;  // the k-th largest falls into my 8 bins (exactly one lane)
      if (here) {
        int kk = kk0 - above, d = lane * 8 + 7;
        for (; d > lane * 8; --d) {
          if (s_hist[d] >= kk) break;
          kk -= s_hist[d];
        }
        *s_k = kk;
        *s_prefix = prefix | (static_cast<unsigned long long>(d) << shift);
      }
    }
    __syncthreads();
  }
  return *s_prefix;
}

__global__ void __launch_bounds__(kBucketThreads) nms_bucket_kernel(const NmsArgs p) {
  pdl_entry();
  __shared__ int s_hist[1024];   // class histogram, then exclusive offsets
  __shared__ int s_cur[1024];    // scatter cursors
  __shared__ int s_sel[256];
  __shared__ int s_warp[32];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_k, s_outside;
  const int img = blockIdx.x;
  int c = p.count[img];
  c = c < p.cap ? c : p.cap;
  const int n = c < p.max_nms ? c : p.max_nms;
  const unsigned long long* keys = p.keys + static_cast<size_t>(img) * p.cap;
  int* off = p.seg_off + static_cast<size_t>(img) * (p.nc + 1);
  if (threadIdx.x == 0) {
    s_outside = 0;
    p.surv_cnt[img] = 0;
    p.done_cnt[img] = 0;
  }
  unsigned long long thr = 0ull;  // candidates below the max_nms-th key are dropped (general.py:728)
  if (c > p.max_nms) thr = block_select_kth(keys, c, p.max_nms, s_sel, &s_prefix, &s_k);
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) {
    s_hist[i] = 0;
    s_cur[i] = 0;
  }
  __syncthreads();
  const float lim = p.max_wh * 0.5f;
  const float4* cb = p.cand_box + static_cast<size_t>(img) * p.cap;
  constexpr int kIlp = 4;  // candidates per thread and iteration: their loads are issued together (one CTA per image: latency-bound)
  // pass A: class histogram + "class-split is exact" check (offset boxes of different classes cannot intersect)
  for (int i0 = threadIdx.x; i0 < c; i0 += kIlp * blockDim.x) {
    unsigned long long kq[kIlp];
    float4 bq[kIlp];
#pragma unroll
    for (int q = 0; q < kIlp; ++q) {
      const int i = i0 + q * blockDim.x;
      kq[q] = i < c ? keys[i] : 0ull;
      bq[q] = i < c ? cb[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int q = 0; q < kIlp; ++q) {
      if (i0 + q * static_cast<int>(blockDim.x) >= c || kq[q] < thr) continue;
      int row, cls;
      key_to_rowcls(kq[q], p.nc, row, cls);
      const float hw = __fdiv_rn(bq[q].z, 2.0f);
      const float x1 = __fsub_rn(bq[q].x, hw), x2 = __fadd_rn(bq[q].x, hw);
      if (!((x1 > -lim) && (x2 < lim) && (x1 <= x2))) s_outside = 1;
      atomicAdd(&s_hist[cls], 1);
    }
  }
  __syncthreads();
  const bool single = p.agnostic || s_outside;
  // exclusive scan of the class counts (nc <= 1024 = one per thread)
  {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int v = (threadIdx.x < p.nc && !single) ? s_hist[threadIdx.x] : 0;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += t;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    const int excl = incl - v + (warp ? s_warp[warp - 1] : 0);
    __syncthreads();
    if (threadIdx.x < p.nc) {
      const int o = single ? (threadIdx.x == 0 ? 0 : n) : excl;
      s_hist[threadIdx.x] = o;
      off[threadIdx.x] = o;
    }
    if (threadIdx.x == 0) {
      off[p.nc] = n;
      p.flags[img] = single ? 1 : 0;
    }
  }
  __syncthreads();
  // pass B: scatter (order inside a segment is arbitrary: the segment kernels rank by key)
  unsigned long long* k2 = p.seg_key2 + static_cast<size_t>(img) * kRankCap;
  float4* b4 = p.box4 + static_cast<size_t>(img) * kRankCap;
  for (int i0 = threadIdx.x; i0 < c; i0 += kIlp * blockDim.x) {
    unsigned long long kq[kIlp];
    float4 bq[kIlp];
#pragma unroll
    for (int q = 0; q < kIlp; ++q) {
      const int i = i0 + q * blockDim.x;
      kq[q] = i < c ? keys[i] : 0ull;
      bq[q] = i < c ? cb[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int q = 0; q < kIlp; ++q) {
      if (i0 + q * static_cast<int>(blockDim.x) >= c || kq[q] < thr) continue;
      int row, cls;
      key_to_rowcls(kq[q], p.nc, row, cls);
      const int seg = single ? 0 : cls;
      const int pos = s_hist[seg] + atomicAdd(&s_cur[seg], 1);
      const float hw = __fdiv_rn(bq[q].z, 2.0f), hh = __fdiv_rn(bq[q].w, 2.0f);
      k2[pos] = kq[q];
      b4[pos] = make_float4(__fsub_rn(bq[q].x, hw), __fsub_rn(bq[q].y, hh), __fadd_rn(bq[q].x, hw), __fadd_rn(bq[q].y, hh));
    }
  }
}

__device__ __forceinline__ float4 offset_box(const float4& b, int cls, const NmsArgs& p) {
  const float off = p.agnostic ? 0.0f : __fmul_rn(static_cast<float>(cls), p.max_wh);  // general.py:731-732
  return make_float4(__fadd_rn(b.x, off), __fadd_rn(b.y, off), __fadd_rn(b.z, off), __fadd_rn(b.w, off));
}

__device__ __forceinline__ void append_survivors(const NmsArgs& p, int img, bool kept, unsigned long long key, int pos, int lane) {
  const unsigned full = 0xffffffffu;
  const unsigned b = __ballot_sync(full, kept);
  if (b == 0u) return;
  int base = 0;
  if (lane == 0) base = atomicAdd(&p.surv_cnt[img], __popc(b));
  base = __shfl_sync(full, base, 0);
  if (kept) {
    const int at = base + __popc(b & ((1u << lane) - 1u));
    p.surv_key[static_cast<size_t>(img) * kRankCap + at] = key;
    p.surv_pos[static_cast<size_t>(img) * kRankCap + at] = pos;
  }
}

constexpr int kMaskSmall = 128;  // segments up to this size: nms_seg_mask_kernel<128, 128> (4 warps, 12 KB of shared memory)
constexpr int kMaskLarge = 512;  // ... up to this size: nms_seg_mask_kernel<512, 256> (46 KB); larger: nms_seg_block_kernel

// One CTA per (image, class) segment, suppression-matrix form: (1) rank the members by key (counting, keys in shared memory),
// (2) boxes to shared memory in confidence order, (3) ALL pair tests in parallel — thread (i, w) builds the 32-bit word "which of
// members 32w..32w+31 does member i suppress" with no dependency between pairs — (4) one warp resolves the greedy order with
// bit operations only: walk i upward, skip removed members, OR row i into the removed set.  The per-keeper formulations (a warp
// with boxes in registers, or a block with a barrier per keeper) serialise m dependent rounds, several times
// the pair-test work at a few hundred members per class.
template <int MAXM, int THREADS>
__global__ void __launch_bounds__(THREADS) nms_seg_mask_kernel(const NmsArgs p, int m_lo) {
  pdl_entry();
  constexpr int W = MAXM / 32;  // mask words per row
  extern __shared__ unsigned long long s_dyn[];
  unsigned long long* s_key = s_dyn;                                   // [MAXM]
  float4* s_box = reinterpret_cast<float4*>(s_key + MAXM);             // [MAXM] in confidence order
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(s_box + MAXM);        // [MAXM][W]
  uint16_t* s_ord = reinterpret_cast<uint16_t*>(s_mask + MAXM * W);    // [MAXM] rank -> member
  constexpr int kList = MAXM * 4;                                      // intersecting pairs tested from a compact list
  uint32_t* s_list = reinterpret_cast<uint32_t*>(s_ord + MAXM);        // [kList] (i << 16 | j)
  __shared__ int s_pairs;
  const int img = blockIdx.y, seg = blockIdx.x;
  const int* off = p.seg_off + static_cast<size_t>(img) * (p.nc + 1);
  const int lo = off[seg], m = off[seg + 1] - lo;
  if (m <= m_lo || m > MAXM) return;  // other instantiations / the serial block kernel own the other sizes
  if (threadIdx.x == 0) s_pairs = 0;
  const unsigned long long* k2 = p.seg_key2 + static_cast<size_t>(img) * kRankCap + lo;
  const float4* b4 = p.box4 + static_cast<size_t>(img) * kRankCap + lo;
  for (int j = threadIdx.x; j < m; j += THREADS) s_key[j] = k2[j];
  __syncthreads();
  for (int j = threadIdx.x; j < m; j += THREADS) {
    const unsigned long long kj = s_key[j];
    int r = 0;
    for (int t = 0; t < m; ++t) r += (s_key[t] > kj) ? 1 : 0;  // broadcast reads
    s_ord[r] = static_cast<uint16_t>(j);
  }
  __syncthreads();
  for (int q = threadIdx.x; q < m; q += THREADS) {
    const int j = s_ord[q];
    int row, cls;
    key_to_rowcls(s_key[j], p.nc, row, cls);
    s_box[q] = offset_box(b4[j], cls, p);
  }
  __syncthreads();
  const int words = (m + 31) >> 5;
  // (3a) intersection bits.  Only "the boxes may intersect" is decided here — two comparisons per axis, a superset of the
  // pairs that pass the first two exits of box_suppresses (NaN coordinates compare false and stay in) — and ~9 in 10 pairs of
  // one class leave at this point, every lane of the warp with them; a per-thread loop over the 32 pairs of a word ran the full
  // exact test (division-free IoU in double) on every pair as soon as one lane needed it.
  // Work = the upper triangle, word column by word column: lane = member j = 32 w + lane (its box stays in registers), rows
  // i < min(m, 32 w + 31), one ballot per (i, w); the flattened (w, i) list is cut into equal ranges, one per warp.
  for (int t = threadIdx.x; t < m * W; t += THREADS) s_mask[t] = 0u;  // rows below the diagonal / words past `words` stay zero
  __syncthreads();
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int kWarps = THREADS / 32;
    auto rows_of = [&](int w) { return min(m, (w << 5) + 31); };
    int total = 0;
    for (int w = 0; w < words; ++w) total += rows_of(w);
    const int per = (total + kWarps - 1) / kWarps;
    int t = warp * per;
    const int t_end = min(total, t + per);
    int w = 0, acc = 0;
    while (w < words && t >= acc + rows_of(w)) acc += rows_of(w++);
    int i = t - acc;
    const float inf = __int_as_float(0x7f800000);
    while (t < t_end) {
      const int j = (w << 5) + lane;
      const float4 bj = j < m ? s_box[j] : make_float4(inf, inf, inf, inf);  // x1 = +inf: intersects nothing
      const int i_end = min(rows_of(w), i + (t_end - t));
      t += i_end - i;
      for (; i < i_end; ++i) {
        const float4 bi = s_box[i];  // broadcast
        uint32_t bits = __ballot_sync(0xffffffffu, j < m && !(bi.z <= bj.x) && !(bj.z <= bi.x) && !(bi.w <= bj.y) && !(bj.w <= bi.y));
        if ((i >> 5) == w) bits &= ~((2u << (i & 31)) - 1u);  // diagonal word: only j > i
        if (lane == 0) s_mask[i * W + w] = bits;
      }
      ++w;
      i = 0;
    }
  }
  __syncthreads();
  {
    // (3b) the exact test on the intersecting pairs only.  The set bits are first compacted into a list of (i, j) pairs — one
    // shared-memory atomic per non-empty word — and the list is then tested one pair per thread: every lane of a warp runs the
    // long path (~40 instructions, double multiply) on a pair that needs it.  Looping over the bits of its own word, a thread
    // dragged its warp through max-popcount-of-32-words rounds (~8 for ~3 useful ones).  A word that does not fit the list any
    // more is tested in place by its owner (same result, slower).
    int i = threadIdx.x / words, w = threadIdx.x - i * words;
    const int di = THREADS / words, dw = THREADS - di * words;
    for (; i < m; i += di, w += dw) {
      if (w >= words) {
        w -= words;
        if (++i >= m) break;
      }
      if ((w << 5) + 31 <= i) continue;  // below the diagonal: zero
      uint32_t bits = s_mask[i * W + w];
      if (!bits) continue;
      const int at = atomicAdd(&s_pairs, __popc(bits));
      if (at + __popc(bits) <= kList) {
        s_mask[i * W + w] = 0u;  // the hits come back through atomicOr below
        int k = at;
        while (bits) {
          const int b = __ffs(bits) - 1;
          bits &= bits - 1;
          s_list[k++] = (static_cast<uint32_t>(i) << 16) | static_cast<uint32_t>((w << 5) + b);
        }
      } else {
        for (int k = at; k < kList; ++k) s_list[k] = 0xFFFFFFFFu;  // reserved, not used (at most one word straddles the end)
        const float4 bi = s_box[i];
        const float ai = __fmul_rn(__fsub_rn(bi.z, bi.x), __fsub_rn(bi.w, bi.y));
        uint32_t keep = 0;
        while (bits) {
          const int b = __ffs(bits) - 1;
          bits &= bits - 1;
          if (box_suppresses(bi, ai, s_box[(w << 5) + b], p)) keep |= 1u << b;
        }
        s_mask[i * W + w] = keep;
      }
    }
    __syncthreads();
    const int n_pairs = min(s_pairs, kList);
    for (int k = threadIdx.x; k < n_pairs; k += THREADS) {
      const uint32_t e = s_list[k];
      if (e == 0xFFFFFFFFu) continue;  // slot reserved by a word that went the in-place way
      const int pi = static_cast<int>(e >> 16), pj = static_cast<int>(e & 0xFFFFu);
      const float4 bi = s_box[pi];
      const float ai = __fmul_rn(__fsub_rn(bi.z, bi.x), __fsub_rn(bi.w, bi.y));
      if (box_suppresses(bi, ai, s_box[pj], p)) atomicOr(&s_mask[pi * W + (pj >> 5)], 1u << (pj & 31));
    }
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    // (4) greedy order, one warp, bit operations only.  Lane l keeps word l of the removed set; `cur` (all lanes) is the word
    // the walk is in.  Both mask words of row i are loaded whether or not the row is alive, so the loads run ahead of the
    // 3-instruction dependency chain (test bit, OR, OR); the first version shuffled the current word out of its lane for every
    // row and waited for each row's load: ~60 clk x m with a single warp active — with the per-32-member atomics below, most of
    // the kernel's critical path.
    const int lane = threadIdx.x;
    uint32_t removed = 0;  // lane w holds word w of the removed set (W <= 32)
    for (int wb = 0; wb < words; ++wb) {
      uint32_t cur = __shfl_sync(0xffffffffu, removed, wb);
      const int i_end = min(m, (wb << 5) + 32);
#pragma unroll 8
      for (int i = wb << 5; i < i_end; ++i) {
        const uint32_t v_own = lane < words ? s_mask[i * W + lane] : 0u;
        const uint32_t v_cur = s_mask[i * W + wb];  // broadcast
        if (!((cur >> (i & 31)) & 1u)) {            // uniform: member i is kept
          removed |= v_own;
          cur |= v_cur;
        }
      }
    }
    // survivors, in rank order: ONE atomic reserves the segment's range (a dependent global round trip per 32 members before)
    int kept_before = 0, total = 0;
    {
      const uint32_t valid = lane < words ? (lane == words - 1 && (m & 31) ? (1u << (m & 31)) - 1u : 0xffffffffu) : 0u;
      const int mine = __popc(~removed & valid);
      int incl = mine;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      kept_before = incl - mine;  // survivors in the words before mine
      total = __shfl_sync(0xffffffffu, incl, 31);
    }
    int base = 0;
    if (lane == 0 && total) base = atomicAdd(&p.surv_cnt[img], total);
    base = __shfl_sync(0xffffffffu, base, 0);
    for (int q0 = 0; q0 < m; q0 += 32) {
      const int q = q0 + lane;
      const uint32_t wq = __shfl_sync(0xffffffffu, removed, q0 >> 5);
      const int before = __shfl_sync(0xffffffffu, kept_before, q0 >> 5);
      const uint32_t alive = ~wq & (q0 + 32 <= m ? 0xffffffffu : (1u << (m & 31)) - 1u);
      if ((alive >> lane) & 1u) {
        const int j = s_ord[q];
        const int at = base + before + __popc(alive & ((1u << lane) - 1u));
        p.surv_key[static_cast<size_t>(img) * kRankCap + at] = s_key[j];
        p.surv_pos[static_cast<size_t>(img) * kRankCap + at] = lo + j;
      }
    }
  }
}

template <int MAXM, int THREADS>
int launch_seg_mask(const NmsArgs& a, int m_lo, cudaStream_t stream) {
  constexpr int W = MAXM / 32;
  constexpr int kSmem = MAXM * (8 + 16 + 4 * W + 2 + 4 * 4);
  auto kern = nms_seg_mask_kernel<MAXM, THREADS>;
  static bool attr_set = false;
  if (!attr_set) {
    Y3_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    attr_set = true;
  }
  Y3_CHECK_CUDA(::y3::launch_pdl(kern, dim3(a.nc, a.bs), dim3(THREADS), kSmem, stream, a, m_lo));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}


// Segments with more than kMaskLarge members.  Class segments: one CTA ranks its members (keys tiled through shared memory) and runs
// the greedy pass.  Single-segment images (agnostic, or boxes outside the class-offset bound): every CTA of the image ranks a
// share of the members; the last one to finish (atomic ticket, no waiting) runs the greedy pass over the whole segment.
constexpr int kRankTile = 1024;

__global__ void __launch_bounds__(256) nms_seg_block_kernel(const NmsArgs p) {
  pdl_entry();
  __shared__ unsigned long long s_tile[kRankTile];
  __shared__ float4 s_box[kSegSmemBoxes];
  __shared__ uint32_t s_supp[(kRankCap + 31) / 32];
  __shared__ int s_last;
  const int img = blockIdx.y, seg = blockIdx.x;
  const int* off = p.seg_off + static_cast<size_t>(img) * (p.nc + 1);
  const bool single = p.flags[img] & 1;
  const int lo = single ? 0 : off[seg], hi = single ? off[p.nc] : off[seg + 1];
  const int m = hi - lo;
  if (m <= kMaskLarge) return;  // empty, or done by the matrix kernels (a single segment sits in class slot 0 there)
  const unsigned long long* k2 = p.seg_key2 + static_cast<size_t>(img) * kRankCap + lo;
  const float4* b4 = p.box4 + static_cast<size_t>(img) * kRankCap + lo;
  uint16_t* ord = p.ord + static_cast<size_t>(img) * kRankCap + lo;
  // ---- rank my share of the members: rank = number of larger keys
  const int share = single ? gridDim.x : 1, me = single ? seg : 0;
  for (int j0 = me * blockDim.x; j0 < m; j0 += share * blockDim.x) {
    const int j = j0 + threadIdx.x;
    const unsigned long long kj = j < m ? k2[j] : ~0ull;
    int r = 0;
    for (int t0 = 0; t0 < m; t0 += kRankTile) {
      __syncthreads();
      for (int t = threadIdx.x; t < kRankTile && t0 + t < m; t += blockDim.x) s_tile[t] = k2[t0 + t];
      __syncthreads();
      const int tn = min(kRankTile, m - t0);
      for (int t = 0; t < tn; ++t) r += (s_tile[t] > kj) ? 1 : 0;
    }
    if (j < m) ord[r] = static_cast<uint16_t>(j);
  }
  if (single) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&p.done_cnt[img], 1) == static_cast<int>(gridDim.x) - 1) ? 1 : 0;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
  } else {
    __syncthreads();
  }
  // ---- greedy pass in confidence order
  auto load_box = [&](int q) -> float4 {
    const int j = ord[q];
    int row, cls;
    key_to_rowcls(k2[j], p.nc, row, cls);
    return offset_box(b4[j], cls, p);
  };
  const bool in_smem = m <= kSegSmemBoxes;
  for (int q = threadIdx.x; q < (m + 31) / 32; q += blockDim.x) s_supp[q] = 0;
  if (in_smem)
    for (int q = threadIdx.x; q < m; q += blockDim.x) s_box[q] = load_box(q);
  __syncthreads();
  for (int i = 0; i < m; ++i) {
    if ((s_supp[i >> 5] >> (i & 31)) & 1u) continue;  // uniform
    const float4 bi = in_smem ? s_box[i] : load_box(i);
    const float ai = __fmul_rn(__fsub_rn(bi.z, bi.x), __fsub_rn(bi.w, bi.y));
    if (i + 1 >= m) break;
    for (int q = i + 1 + threadIdx.x; q < m; q += blockDim.x) {
      if ((s_supp[q >> 5] >> (q & 31)) & 1u) continue;
      const float4 bj = in_smem ? s_box[q] : load_box(q);
      if (box_suppresses(bi, ai, bj, p)) atomicOr(&s_supp[q >> 5], 1u << (q & 31));
    }
    __syncthreads();
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int q0 = 0; q0 < m; q0 += blockDim.x) {
    const int q = q0 + threadIdx.x;
    const bool kept = q < m && !((s_supp[q >> 5] >> (q & 31)) & 1u);
    const int j = q < m ? ord[q] : 0;
    append_survivors(p, img, kept, kept ? k2[j] : 0ull, lo + j, lane);
  }
}

__global__ void __launch_bounds__(1024) nms_output_kernel(const NmsArgs p) {
  pdl_entry();
  extern __shared__ unsigned long long s_dyn[];
  unsigned long long* s_k = s_dyn;                                          // [kOutSortMax]
  uint16_t* s_p = reinterpret_cast<uint16_t*>(s_dyn + kOutSortMax);         // [kOutSortMax] positions < kRankCap = 32768
  __shared__ int s_sel[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_k_, s_n;
  const int img = blockIdx.x;
  const int c = p.count[img];
  if (p.overflow && threadIdx.x == 0) p.overflow[img] = c > p.cap ? c : 0;
  const int S = p.surv_cnt[img];
  const int D = S < p.max_det ? S : p.max_det;
  const unsigned long long* sk = p.surv_key + static_cast<size_t>(img) * kRankCap;
  const int* sp = p.surv_pos + static_cast<size_t>(img) * kRankCap;
  float* out = p.out + static_cast<size_t>(img) * p.max_det * 6;
  const float4* b4 = p.box4 + static_cast<size_t>(img) * kRankCap;
  auto emit = [&](int rank, unsigned long long key, int pos) {
    int row, cls;
    key_to_rowcls(key, p.nc, row, cls);
    const float4 b = b4[pos];
    float* o = out + static_cast<size_t>(rank) * 6;
    o[0] = b.x;
    o[1] = b.y;
    o[2] = b.z;
    o[3] = b.w;
    o[4] = __uint_as_float(static_cast<uint32_t>(key >> 32));
    o[5] = static_cast<float>(cls);
    if (p.out_src) {
      p.out_src[(static_cast<size_t>(img) * p.max_det + rank) * 2 + 0] = row;
      p.out_src[(static_cast<size_t>(img) * p.max_det + rank) * 2 + 1] = cls;
    }
  };
  if (D > 0) {
    unsigned long long thr = 0ull;
    int cnt = S;  // survivors that enter the sort
    const bool select_first = S > kOutSortMax || (S > 1024 && S >= 2 * D);
    if (select_first) {
      // only the top D rows are returned: an exact radix select (8 passes over S keys) followed by a sort of D keys beats
      // sorting everything with an 8192-key shared-memory bitonic network
      thr = block_select_kth(sk, S, D, s_sel, &s_prefix, &s_k_);  // exactly D survivors have key >= thr
      cnt = D;
    }
    if (cnt <= kOutSortMax) {
      int npad = next_pow2(cnt);
      npad = npad < 32 ? 32 : npad;
      if (threadIdx.x == 0) s_n = 0;
      __syncthreads();
      if (select_first) {
        for (int i = threadIdx.x; i < S; i += blockDim.x) {
          const unsigned long long key = sk[i];
          if (key >= thr) {
            const int at = atomicAdd(&s_n, 1);
            s_k[at] = key;
            s_p[at] = static_cast<uint16_t>(sp[i]);
          }
        }
      } else {
        for (int i = threadIdx.x; i < S; i += blockDim.x) {
          s_k[i] = sk[i];
          s_p[i] = static_cast<uint16_t>(sp[i]);
        }
      }
      __syncthreads();
      for (int i = cnt + threadIdx.x; i < npad; i += blockDim.x) {
        s_k[i] = 0ull;
        s_p[i] = 0;
      }
      __syncthreads();
      for (int k = 2; k <= npad; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
          for (int t = threadIdx.x; t < npad / 2; t += blockDim.x) {
            const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
            const bool up = ((i & k) == 0);  // descending overall: "up" halves end with the larger key first
            const unsigned long long a = s_k[i], b = s_k[i | j];
            if (up ? a < b : a > b) {
              s_k[i] = b;
              s_k[i | j] = a;
              const uint16_t t2 = s_p[i];
              s_p[i] = s_p[i | j];
              s_p[i | j] = t2;
            }
          }
          __syncthreads();
        }
      }
      for (int rnk = threadIdx.x; rnk < D; rnk += blockDim.x) emit(rnk, s_k[rnk], s_p[rnk]);
    } else {
      // more than 8192 rows requested AND available: rank by counting straight from global memory (exact, slow, rare)
      for (int i = threadIdx.x; i < S; i += blockDim.x) {
        const unsigned long long key = sk[i];
        if (key < thr) continue;
        int rnk = 0;
        for (int t = 0; t < S; ++t) rnk += (sk[t] > key) ? 1 : 0;
        emit(rnk, key, sp[i]);
      }
    }
  }
  if (threadIdx.x == 0) p.out_count[img] = D;
  for (int i = D * 6 + threadIdx.x; i < p.max_det * 6; i += blockDim.x) out[i] = 0.f;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace
}  // namespace y3

extern "C" int64_t y3_nms_workspace_bytes(int32_t bs, int32_t cap) {
  if (bs <= 0 || cap <= 0) return -1;
  size_t b = 0;
  b += y3::align_up(sizeof(unsigned long long) * size_t(bs) * cap, 256);
  b += y3::align_up(sizeof(int) * size_t(bs) * 2, 256);
  // seg_off, seg_key2, box4, surv_cnt + done_cnt, surv_key, surv_pos, ord
  b += y3::align_up(sizeof(int) * size_t(bs) * 1025, 256);
  b += y3::align_up(sizeof(unsigned long long) * size_t(bs) * y3::kRankCap, 256);
  b += y3::align_up(sizeof(float4) * size_t(bs) * y3::kRankCap, 256);
  b += y3::align_up(sizeof(int) * size_t(bs) * 2, 256);
  b += y3::align_up(sizeof(unsigned long long) * size_t(bs) * y3::kRankCap, 256);
  b += y3::align_up(sizeof(int) * size_t(bs) * y3::kRankCap, 256);
  b += y3::align_up(sizeof(uint16_t) * size_t(bs) * y3::kRankCap, 256);
  b += y3::align_up(sizeof(float4) * size_t(bs) * cap, 256);  // cand_box
  return static_cast<int64_t>(b);
}

extern "C" int32_t y3_nms_default_capacity(int32_t n_rows, int32_t nc, int32_t multi_label) {
  long long want = multi_label ? 4ll * n_rows : n_rows;  // multi-label: room for 4 labels/row before an exact retry
  if (want < y3::kMinCap) want = y3::kMinCap;
  long long cap = y3::kMinCap;
  while (cap < want) cap <<= 1;
  (void)nc;
  return static_cast<int32_t>(cap);
}

extern "C" int y3_nms_batched(const float* pred, const y3_nms_params* q, void* workspace, int64_t workspace_bytes,
                              float* out, int32_t* out_src, int32_t* out_count, int32_t* overflow,
                              y3_stream_t stream_) {
  using namespace y3;
  Y3_REQUIRE(pred && q && workspace && out && out_count, "nms: null pointer");
  Y3_REQUIRE(q->bs > 0 && q->n_rows > 0 && q->nc >= 1 && q->nc <= 1024, "nms: bad shape bs=%d rows=%d nc=%d", q->bs,
             q->n_rows, q->nc);
  Y3_REQUIRE(q->conf_thres >= 0.f && q->conf_thres <= 1.f, "nms: invalid confidence threshold %f", q->conf_thres);
  Y3_REQUIRE(q->iou_thres >= 0.f && q->iou_thres <= 1.f, "nms: invalid IoU threshold %f", q->iou_thres);
  Y3_REQUIRE(q->max_det > 0 && q->max_nms > 0 && q->max_nms <= kRankCap, "nms: max_det/max_nms out of range");
  Y3_REQUIRE(q->cap >= kMinCap && (q->cap & (q->cap - 1)) == 0, "nms: capacity must be a power of two >= %d", kMinCap);
  Y3_REQUIRE(static_cast<long long>(q->n_rows) * q->nc < (1ll << 32), "nms: n_rows*nc overflows the candidate id");
  Y3_REQUIRE(workspace_bytes >= y3_nms_workspace_bytes(q->bs, q->cap), "nms: workspace too small");
  Y3_REQUIRE(q->bs <= 65535, "nms: batch too large");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);

  NmsArgs a{};
  a.pred = pred;
  a.bs = q->bs;
  a.n_rows = q->n_rows;
  a.nc = q->nc;
  a.no = q->nc + 5;
  a.conf_thres = q->conf_thres;
  a.iou_thres = q->iou_thres;
  {
    const float t = q->iou_thres, up = nextafterf(t, INFINITY);
    a.iou_mid = 0.5 * (static_cast<double>(t) + static_cast<double>(up));
    uint32_t bits;
    memcpy(&bits, &t, sizeof(bits));
    a.iou_odd = static_cast<int>(bits & 1u);
  }
  a.max_wh = q->max_wh > 0 ? q->max_wh : 7680.f;
  a.multi_label = (q->multi_label && q->nc > 1) ? 1 : 0;  // general.py:677
  a.agnostic = q->agnostic ? 1 : 0;
  a.max_det = q->max_det;
  a.max_nms = q->max_nms;
  a.cap = q->cap;
  a.use_mask = q->n_classes > 0;
  for (int i = 0; i < q->n_classes; ++i) {
    const int c = q->classes[i];
    if (c >= 0 && c < 1024) a.cls_mask[c >> 5] |= 1u << (c & 31);
  }
  uint8_t* w = static_cast<uint8_t*>(workspace);
  a.keys = reinterpret_cast<unsigned long long*>(w);
  w += align_up(sizeof(unsigned long long) * size_t(a.bs) * a.cap, 256);
  a.count = reinterpret_cast<int*>(w);
  a.flags = a.count + a.bs;
  w += align_up(sizeof(int) * size_t(a.bs) * 2, 256);
  a.seg_off = reinterpret_cast<int*>(w);
  w += align_up(sizeof(int) * size_t(a.bs) * 1025, 256);
  a.seg_key2 = reinterpret_cast<unsigned long long*>(w);
  w += align_up(sizeof(unsigned long long) * size_t(a.bs) * kRankCap, 256);
  a.box4 = reinterpret_cast<float4*>(w);
  w += align_up(sizeof(float4) * size_t(a.bs) * kRankCap, 256);
  a.surv_cnt = reinterpret_cast<int*>(w);
  a.done_cnt = a.surv_cnt + a.bs;
  w += align_up(sizeof(int) * size_t(a.bs) * 2, 256);
  a.surv_key = reinterpret_cast<unsigned long long*>(w);
  w += align_up(sizeof(unsigned long long) * size_t(a.bs) * kRankCap, 256);
  a.surv_pos = reinterpret_cast<int*>(w);
  w += align_up(sizeof(int) * size_t(a.bs) * kRankCap, 256);
  a.ord = reinterpret_cast<uint16_t*>(w);
  w += align_up(sizeof(uint16_t) * size_t(a.bs) * kRankCap, 256);
  a.cand_box = reinterpret_cast<float4*>(w);
  a.out = out;
  a.out_src = out_src;
  a.out_count = out_count;
  a.overflow = overflow;

  Y3_CHECK_CUDA(cudaMemsetAsync(a.count, 0, sizeof(int) * size_t(a.bs) * 2, stream));
  Y3_CHECK_CUDA(::y3::launch_pdl(nms_candidates_kernel, dim3((a.n_rows + 32 * kCandWarps - 1) / (32 * kCandWarps), a.bs), dim3(32 * kCandWarps), 0, stream, a));
  Y3_CHECK_CUDA(::y3::launch_pdl(nms_bucket_kernel, dim3(a.bs), dim3(kBucketThreads), 0, stream, a));
  // the first matrix kernel (one thread per mask word, full test on all 32 pairs) beat a warp-per-segment kernel only at
  // <= 128 members per class and lost at a few hundred.  The two-phase pair test (ballot of intersections, exact test on those) is what made the matrix form win there too.
  if (int rc = launch_seg_mask<kMaskSmall, 128>(a, 0, stream)) return rc;
  if (int rc = launch_seg_mask<kMaskLarge, 256>(a, kMaskSmall, stream)) return rc;
  Y3_CHECK_CUDA(::y3::launch_pdl(nms_seg_block_kernel, dim3(a.nc, a.bs), dim3(256), 0, stream, a));
  {
    constexpr int kOutSmem = kOutSortMax * (sizeof(unsigned long long) + sizeof(uint16_t));
    static bool attr_set = false;
    if (!attr_set) {
      Y3_CHECK_CUDA(cudaFuncSetAttribute(nms_output_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kOutSmem));
      attr_set = true;
    }
    Y3_CHECK_CUDA(::y3::launch_pdl(nms_output_kernel, dim3(a.bs), dim3(1024), kOutSmem, stream, a));
  }
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
