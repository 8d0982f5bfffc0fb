// yolov3_b200 — training-mode pieces of the Conv block (reference models/common.py:71-75 `act(bn(conv(x)))` with
// BatchNorm2d in training mode, eps 1e-3 / momentum 0.03 set by initialize_weights, models/yolo.py:229) and their
// backward.  The convolution itself (forward, and dgrad as a convolution with transposed/flipped weights) runs in
// conv_tc_kernel with an identity epilogue; this file holds the bandwidth-bound parts around it:
//   bn_stats        per-channel sum / sum of squares of the conv output y (padded NHWC bf16; the zero halo adds nothing)
//   bn_finalize     batch mean/var -> (scale, shift), saved (mean, rstd), running-stat update (unbiased var, momentum)
//   bn_act_fwd      a = SiLU(y*scale + shift) (+ residual), optional nearest-2x store / concat-offset store
//   bn_act_bwd_red  dz = da * SiLU'(z);  per-channel sum(dz), sum(dz * yhat)          (dgamma, dbeta)
//   bn_act_bwd      dy = scale * (dz - mean(dz) - yhat * mean(dz*yhat))               (input of dgrad / wgrad)
//   pack_weights    fp32 master weights [co,ci,k,k] -> bf16 forward pack [co_pad, tap*ci+c] and dgrad pack
//                   [ci_pad, tap'*co+o] (taps flipped), every optimizer step
//   zero_stuff      dy of a stride-2 conv scattered onto the even positions of a zero 2x grid (its dgrad is then a
//                   stride-1 conv with flipped weights)
//   wgrad           dW[co, tap, ci] = sum_p dy[p, co] * x[p + shift(tap), ci]  (warp-level bf16 MMA, split over pixels)
//   bias_grad       Detect heads: db[co] = sum_p dy[p, co]
#include <cstdlib>

#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {
namespace {

// geometry of a padded NHWC slice
struct Slice {
  const __nv_bfloat16* p;
  int ld, coff;
};
struct SliceW {
  __nv_bfloat16* p;
  int ld, coff;
};

// ---------------------------------------------------------------------------------------------- row iteration
// Every elementwise / reduction kernel below walks INTERIOR image rows: row r of n*h -> (image, y) with one 32-bit division
// per row, then 16-byte items e = x*c8 + cg inside the row (c8 = channels/8 is a power of two for every BatchNorm of the
// YOLOv3 graphs, so x = e >> log2(c8)).  The first version derived (n, y, x) from a 64-bit flat index with two 64-bit
// divisions per 16 bytes and ran several times above its HBM floor.
struct Rows {
  int n, h, w, c8, c8_shift;  // c8_shift = log2(c8), or -1 when c8 is not a power of two (generic division)
  int upr;                    // work units per image row: a unit = kUnitIters x 256 consecutive 16-byte items of one row
};
// Every thread of a unit issues all of its (kUnitIters x loads-per-item) 16-byte loads before it consumes any: with one whole
// row per block (10 dependent iterations per thread) the small layers ran far below HBM speed on latency alone.
constexpr int kUnitIters = 2;
__device__ __forceinline__ void split_item(const Rows& g, int e, int& x, int& cg) {
  if (g.c8_shift >= 0) {
    x = e >> g.c8_shift;
    cg = e & (g.c8 - 1);
  } else {
    x = e / g.c8;
    cg = e - x * g.c8;
  }
}
__device__ __forceinline__ long long row_base(const Rows& g, int r, int scale = 1) {
  // padded pixel index of interior pixel (y, x=0) of image n; scale = 2: the 2x-upsampled geometry's pixel (2y, 0)
  const int n = r / g.h, y = r - n * g.h;
  const int hp = g.h * scale + 2, wp = g.w * scale + 2;
  return (static_cast<long long>(n) * hp + y * scale + 1) * wp + 1;
}

// block-level reduction of per-thread 8-channel accumulators over the threads that share a channel group, written as ONE
// partial row per block (no atomics: the second stage adds the rows in a fixed order, so results are bit-reproducible)
__device__ __forceinline__ void block_reduce_store(float (&s)[8], float (&q)[8], int c8, float* sh, float* partial_row, int c) {
  const int cg = threadIdx.x % c8, rl = threadIdx.x / c8, nrl = blockDim.x / c8;
  float* ss = sh + threadIdx.x * 8;
  float* qq = sh + 256 * 8 + threadIdx.x * 8;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    ss[i] = s[i];
    qq[i] = q[i];
  }
  __syncthreads();
  if (rl == 0) {
    for (int k = 1; k < nrl; ++k) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i] += sh[(k * c8 + cg) * 8 + i];
        q[i] += sh[256 * 8 + (k * c8 + cg) * 8 + i];
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      partial_row[cg * 8 + i] = s[i];
      partial_row[c + cg * 8 + i] = q[i];
    }
  }
}

// ---------------------------------------------------------------------------------------------- bn_stats
// grid: nblk blocks of 256 threads; block b walks rows b, b+nblk, ...; partial[b] = [sum(c) | sumsq(c)]
__global__ void __launch_bounds__(256, 4) bn_stats_kernel(Slice y, Rows g, float* __restrict__ partial) {
  pdl_entry();
  extern __shared__ float sh[];  // [2][256][8]
  float s[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const int items = g.w * g.c8, units = g.n * g.h * g.upr;
  for (int u = blockIdx.x; u < units; u += gridDim.x) {
    const int r = u / g.upr, e0 = (u - r * g.upr) * (256 * kUnitIters) + threadIdx.x;
    const __nv_bfloat16* base = y.p + row_base(g, r) * y.ld + y.coff;
    uint4 v[kUnitIters];
#pragma unroll
    for (int k = 0; k < kUnitIters; ++k) {
      const int e = e0 + k * 256;
      int x, cg;
      split_item(g, e, x, cg);
      v[k] = e < items ? __ldg(reinterpret_cast<const uint4*>(base + static_cast<long long>(x) * y.ld + cg * 8)) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int k = 0; k < kUnitIters; ++k) {
      float f[8];
      unpack8(v[k], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i] += f[i];
        q[i] = fmaf(f[i], f[i], q[i]);
      }
    }
  }
  block_reduce_store(s, q, g.c8, sh, partial + static_cast<long long>(blockIdx.x) * 2 * g.c8 * 8, g.c8 * 8);
}

// Second stage of every two-stage reduction here: column sums of the nblk partial rows in a FIXED order (bit-reproducible).
// Block = 32 columns x 32 row lanes: lane ty adds rows ty, ty+32, ... (coalesced 128-byte reads across tx), then the 32 lane
// sums are added in index order.  The first version gave each column to one thread that walked all ~300 rows serially.
__device__ __forceinline__ float colsum_32x32(const float* __restrict__ partial, int nblk, long long pitch, int col, bool valid,
                                              float (*sh)[33]) {
  // all of this lane's rows are requested before the first add (kMaxPartialBlocks / 32 <= 14 independent loads in flight): as a
  // load-add loop the 14 L2 round trips serialised
  constexpr int kMaxRowsPerLane = 14;
  float v[kMaxRowsPerLane];
#pragma unroll
  for (int i = 0; i < kMaxRowsPerLane; ++i) {
    const int b = threadIdx.y + 32 * i;
    v[i] = (valid && b < nblk) ? partial[static_cast<long long>(b) * pitch + col] : 0.f;
  }
  float a = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxRowsPerLane; ++i) a += v[i];  // fixed order
  if (valid)
    for (int b = threadIdx.y + 32 * kMaxRowsPerLane; b < nblk; b += 32) a += partial[static_cast<long long>(b) * pitch + col];
  sh[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  float tot = 0.f;
  if (threadIdx.y == 0)
    for (int r = 0; r < 32; ++r) tot += sh[r][threadIdx.x];
  __syncthreads();
  return tot;  // meaningful on threadIdx.y == 0
}

__global__ void __launch_bounds__(1024) colreduce_kernel(const float* __restrict__ partial, int nblk, int width,
                                                         float* __restrict__ out, int accumulate) {
  pdl_entry();
  __shared__ float sh[32][33];
  const int j = blockIdx.x * 32 + threadIdx.x;
  const float a = colsum_32x32(partial, nblk, width, j, j < width, sh);
  if (threadIdx.y == 0 && j < width) out[j] = accumulate ? out[j] + a : a;
}

// ---------------------------------------------------------------------------------------------- bn_finalize
// sums[2][c] given as `nblk` partial rows (nblk = 1: already reduced, e.g. after SyncBatchNorm's all-reduce)
__global__ void __launch_bounds__(1024) bn_finalize_kernel(const float* __restrict__ partial, int nblk, const float* gamma,
                                                           const float* beta, int c, float count, float eps, float momentum,
                                                           float* scale, float* shift, float* mean_out, float* rstd_out,
                                                           float* running_mean, float* running_var) {
  pdl_entry();
  __shared__ float sh[32][33];
  const int i = blockIdx.x * 32 + threadIdx.x;
  const float sum = colsum_32x32(partial, nblk, 2ll * c, i, i < c, sh);
  const float sumsq = colsum_32x32(partial, nblk, 2ll * c, c + i, i < c, sh);  // (its loads do not depend on the first sum)
  if (threadIdx.y != 0 || i >= c) return;
  const float mean = sum / count;
  float var = sumsq / count - mean * mean;
  var = var > 0.f ? var : 0.f;
  const float rstd = rsqrtf(var + eps);
  const float sc = gamma[i] * rstd;
  scale[i] = sc;
  shift[i] = beta[i] - mean * sc;
  mean_out[i] = mean;
  rstd_out[i] = rstd;
  if (running_mean) {
    const float unbiased = count > 1.f ? var * count / (count - 1.f) : var;
    running_mean[i] = (1.f - momentum) * running_mean[i] + momentum * mean;
    running_var[i] = (1.f - momentum) * running_var[i] + momentum * unbiased;
  }
}

// ---------------------------------------------------------------------------------------------- bn_act_fwd
// one thread = one interior pixel x 8 channels per item
struct BnActArgs {
  Slice y;        // conv output (pre-BN)
  Slice res;      // optional residual (p == nullptr: none), geometry of y
  SliceW out;     // activation; padded (h*u+2, w*u+2) when upsample
  const float* scale;
  const float* shift;
  Rows g;
  int upsample;
};
__global__ void __launch_bounds__(256) bn_act_fwd_kernel(const BnActArgs p) {
  pdl_entry();
  const Rows g = p.g;
  const int items = g.w * g.c8, units = g.n * g.h * g.upr;
  const int us = p.upsample ? 2 : 1;
  const long long up_row = static_cast<long long>(2 * g.w + 2) * p.out.ld;
  for (int u = blockIdx.x; u < units; u += gridDim.x) {
    const int r = u / g.upr, e0 = (u - r * g.upr) * (256 * kUnitIters) + threadIdx.x;
    const long long rb = row_base(g, r);
    const long long ob = p.upsample ? row_base(g, r, 2) : rb;
    uint4 vy[kUnitIters], vr[kUnitIters];
#pragma unroll
    for (int k = 0; k < kUnitIters; ++k) {
      const int e = e0 + k * 256;
      int x, cg;
      split_item(g, e, x, cg);
      vy[k] = vr[k] = make_uint4(0, 0, 0, 0);
      if (e < items) {
        vy[k] = __ldg(reinterpret_cast<const uint4*>(p.y.p + (rb + x) * p.y.ld + p.y.coff + cg * 8));
        if (p.res.p) vr[k] = __ldg(reinterpret_cast<const uint4*>(p.res.p + (rb + x) * p.res.ld + p.res.coff + cg * 8));
      }
    }
#pragma unroll
    for (int k = 0; k < kUnitIters; ++k) {
      const int e = e0 + k * 256;
      if (e >= items) continue;
      int x, cg;
      split_item(g, e, x, cg);
      float f[8], rr[8];
      unpack8(vy[k], f);
      const float4 s0 = __ldg(reinterpret_cast<const float4*>(p.scale + cg * 8)), s1 = __ldg(reinterpret_cast<const float4*>(p.scale + cg * 8 + 4));
      const float4 h0 = __ldg(reinterpret_cast<const float4*>(p.shift + cg * 8)), h1 = __ldg(reinterpret_cast<const float4*>(p.shift + cg * 8 + 4));
      const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
      const float sh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
      for (int q = 0; q < 8; ++q) f[q] = silu_fast(fmaf(f[q], sc[q], sh[q]));
      if (p.res.p) {
        unpack8(vr[k], rr);
#pragma unroll
        for (int q = 0; q < 8; ++q) f[q] += rr[q];
      }
      const uint4 o = pack8(f);
      __nv_bfloat16* dst = p.out.p + (ob + static_cast<long long>(x) * us) * p.out.ld + p.out.coff + cg * 8;
      *reinterpret_cast<uint4*>(dst) = o;
      if (p.upsample) {
        *reinterpret_cast<uint4*>(dst + p.out.ld) = o;
        *reinterpret_cast<uint4*>(dst + up_row) = o;
        *reinterpret_cast<uint4*>(dst + up_row + p.out.ld) = o;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- bn_act_bwd
// da: gradient w.r.t. the block output a (geometry of `out` in the forward, i.e. 2x when upsample: the 4 replicas are
// summed).  Pass 1 (reduce) writes per-block partial sums of dz and dz*yhat; a fixed-order second stage turns them into
// (sum_dz, sum_dzy) — and adds them to the beta / gamma gradients; pass 2 (apply) writes dy.
struct BnBwdArgs {
  Slice y;
  Slice da;
  SliceW dy;
  const float* scale;  // gamma * rstd
  const float* shift;  // beta - mean*scale
  const float* mean;
  const float* rstd;
  const float* sum_dz;   // [c]  apply pass
  const float* sum_dzy;  // [c]
  float* partial;        // [nblk][2][c]  reduce pass
  Rows g;
  int upsample;
  float inv_count;
};
__device__ __forceinline__ void load_da(const BnBwdArgs& p, long long rb, long long ub, int x, int cg, float (&d)[8]) {
  if (p.upsample) {
    const long long w2 = 2 * p.g.w + 2;
    const __nv_bfloat16* q = p.da.p + (ub + 2ll * x) * p.da.ld + p.da.coff + cg * 8;
    float t0[8], t1[8], t2[8], t3[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(q)), t0);
    unpack8(__ldg(reinterpret_cast<const uint4*>(q + p.da.ld)), t1);
    unpack8(__ldg(reinterpret_cast<const uint4*>(q + w2 * p.da.ld)), t2);
    unpack8(__ldg(reinterpret_cast<const uint4*>(q + (w2 + 1) * p.da.ld)), t3);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = (t0[k] + t1[k]) + (t2[k] + t3[k]);
  } else {
    unpack8(__ldg(reinterpret_cast<const uint4*>(p.da.p + (rb + x) * p.da.ld + p.da.coff + cg * 8)), d);
  }
}
// dz = da * d/dz[z*sigmoid(z)] = da * s*(1 + z*(1-s)); sigmoid(z) = 0.5*tanh(z/2) + 0.5: ONE MUFU op (tanh.approx, abs error
// ~5e-4 — below the bf16 rounding of dy) instead of ex2 + rcp; these kernels sit close to the MUFU roof (2 ops x 8 elements
// per 16 bytes loaded)
__device__ __forceinline__ float sigmoid_fast(float z) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * z));
  return fmaf(0.5f, t, 0.5f);
}
__device__ __forceinline__ float silu_grad(float z) {
  const float s = sigmoid_fast(z);
  return s * fmaf(z, 1.0f - s, 1.0f);
}

template <bool APPLY, bool UPS>
__global__ void __launch_bounds__(256, UPS ? 2 : 3) bn_act_bwd_kernel(const BnBwdArgs p) {
  pdl_entry();
  // block = 256 threads; thread t keeps channel group t % c8 for the whole kernel (256 % c8 == 0)
  extern __shared__ float sh[];
  const Rows g = p.g;
  const int cg = threadIdx.x % g.c8;
  const int items = g.w * g.c8, units = g.n * g.h * g.upr;
  float a_dz[8] = {0, 0, 0, 0, 0, 0, 0, 0}, a_dzy[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // per-channel constants.  APPLY: dy = sc*(dz - mean(dz) - yhat*mean(dz*yhat)) = sc*dz + k1*y + k0 with yhat = (y - mu)*rs
  float sc[8], shf[8], c2[8], c3[8];  // sums pass: c2 = mu, c3 = rs;  apply pass: c2 = k1, c3 = k0
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    sc[k] = p.scale[cg * 8 + k];
    shf[k] = p.shift[cg * 8 + k];
    const float mu = p.mean[cg * 8 + k], rs = p.rstd[cg * 8 + k];
    if (APPLY) {
      const float m_dz = p.sum_dz[cg * 8 + k] * p.inv_count, m_dzy = p.sum_dzy[cg * 8 + k] * p.inv_count;
      c2[k] = -sc[k] * rs * m_dzy;
      c3[k] = -sc[k] * m_dz - c2[k] * mu;
    } else {
      c2[k] = mu;
      c3[k] = rs;
    }
  }
  for (int u = blockIdx.x; u < units; u += gridDim.x) {
    const int r = u / g.upr, e0 = (u - r * g.upr) * (256 * kUnitIters) + threadIdx.x;
    const long long rb = row_base(g, r);
    const long long ub = p.upsample ? row_base(g, r, 2) : rb;
    // raw 16-byte vectors stay packed until they are consumed (registers: the reduction pass keeps 48 per-channel values);
    // only the 2x-upsample variant (2 layers) sums its four da replicas right away
    uint4 vy[kUnitIters], vd[kUnitIters];
    float du[UPS ? kUnitIters : 1][8];
#pragma unroll
    for (int k = 0; k < kUnitIters; ++k) {
      const int e = e0 + k * 256;
      const int x = g.c8_shift >= 0 ? e >> g.c8_shift : e / g.c8;  // cg is loop-invariant: 256 % c8 == 0
      vy[k] = vd[k] = make_uint4(0, 0, 0, 0);  // dz = 0 beyond the row: adds nothing to the sums
      if (UPS) {
#pragma unroll
        for (int q = 0; q < 8; ++q) du[UPS ? k : 0][q] = 0.f;
      }
      if (e < items) {
        vy[k] = __ldg(reinterpret_cast<const uint4*>(p.y.p + (rb + x) * p.y.ld + p.y.coff + cg * 8));
        if (UPS)
          load_da(p, rb, ub, x, cg, du[UPS ? k : 0]);
        else
          vd[k] = __ldg(reinterpret_cast<const uint4*>(p.da.p + (rb + x) * p.da.ld + p.da.coff + cg * 8));
      }
    }
#pragma unroll
    for (int k = 0; k < kUnitIters; ++k) {
      const int e = e0 + k * 256;
      const int x = g.c8_shift >= 0 ? e >> g.c8_shift : e / g.c8;
      float yv[8], d[8], o[8];
      unpack8(vy[k], yv);
      if (UPS) {
#pragma unroll
        for (int q = 0; q < 8; ++q) d[q] = du[UPS ? k : 0][q];
      } else {
        unpack8(vd[k], d);
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float z = fmaf(yv[q], sc[q], shf[q]);
        const float dz = d[q] * silu_grad(z);
        if (APPLY) {
          o[q] = fmaf(sc[q], dz, fmaf(c2[q], yv[q], c3[q]));
        } else {
          const float yh = (yv[q] - c2[q]) * c3[q];
          a_dz[q] += dz;
          a_dzy[q] = fmaf(dz, yh, a_dzy[q]);
        }
      }
      if (APPLY && e < items) *reinterpret_cast<uint4*>(p.dy.p + (rb + x) * p.dy.ld + p.dy.coff + cg * 8) = pack8(o);
    }
  }
  if (!APPLY)
    block_reduce_store(a_dz, a_dzy, g.c8, sh, p.partial + static_cast<long long>(blockIdx.x) * 2 * g.c8 * 8, g.c8 * 8);
}

// ---------------------------------------------------------------------------------------------- cp.async ring variant
// bn_act_bwd_kernel keeps a unit's 16-byte vectors in registers between issue and use: 4 loads per thread in flight, three
// blocks per SM, a bubble at every unit boundary, long-scoreboard stalls on top; a
// register look-ahead halved the resident blocks and gained nothing.  The variant below stages
// the SAME units through a per-thread shared-memory ring with cp.async: a thread copies its own 16-byte items kRingDepth-1
// units ahead into its own slots and reads them back itself, so there is no barrier and no mbarrier anywhere
// (cp.async.wait_group cannot dead-lock) and 144 KB per SM are in flight without costing registers.  Unit order, item order
// and operations are exactly those of bn_act_bwd_kernel: results are bit-identical (A/B script: tests/diag/ab_shot.py).
// The same ring under bn_stats gained nothing and under bn_act_fwd lost (three 64 KB blocks per SM instead of five or six
// register-only ones): those two were removed again — the passes are bound by resident warps x issue, not by bytes in flight.
// Switch: y3_set_bn_async / Y3_BN_ASYNC (default on).
__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* gptr) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(gptr) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

constexpr int kRingDepth = 4;  // units in the ring: kRingDepth - 1 requested ahead of the one being consumed
// byte offset of (stage, stream, item k) of this thread's slots; NS = streams per unit
template <int NS>
__device__ __forceinline__ uint32_t ring_slot(uint32_t ring, int stage, int s, int k) {
  return ring + ((((stage * NS + s) * kUnitIters + k) * 256 + threadIdx.x) << 4);
}
template <int NS>
constexpr int ring_bytes() {
  return kRingDepth * NS * kUnitIters * 256 * 16;
}
// unit i of this block -> (first item of this thread, padded pixel index of the row's x = 0)
__device__ __forceinline__ void unit_pos(const Rows& g, int i, int& e0, long long& rb) {
  const int u = blockIdx.x + i * gridDim.x;
  const int r = u / g.upr;
  e0 = (u - r * g.upr) * (256 * kUnitIters) + threadIdx.x;
  rb = row_base(g, r);
}
__device__ __forceinline__ int units_of_block(const Rows& g) {
  const int units = g.n * g.h * g.upr;
  return static_cast<int>(blockIdx.x) < units ? (units - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x) : 0;
}
// request unit i of one stream into `stage`
template <int NS>
__device__ __forceinline__ void ring_issue(const Rows& g, const Slice& t, int s, int i, int stage, uint32_t ring) {
  int e0;
  long long rb;
  unit_pos(g, i, e0, rb);
  const int items = g.w * g.c8;
#pragma unroll
  for (int k = 0; k < kUnitIters; ++k) {
    const int e = e0 + k * 256;
    int x, cg;
    split_item(g, e, x, cg);
    if (e < items) cp_async16(ring_slot<NS>(ring, stage, s, k), t.p + (rb + x) * t.ld + t.coff + cg * 8);
  }
}

// the non-upsample reduce / apply passes (the two 2x-upsample layers stay on bn_act_bwd_kernel<*, true>)
template <bool APPLY>
__global__ void __launch_bounds__(256, 3) bn_act_bwd_async_kernel(const BnBwdArgs p) {
  pdl_entry();
  extern __shared__ __align__(16) float ring_mem[];  // ring (64 KB); the reduce pass reuses it as [2][256][8]
  float* sh = ring_mem;
  const uint32_t ring = smem_u32(ring_mem);
  const Rows g = p.g;
  const int cg = threadIdx.x % g.c8;  // fixed per thread: 256 % c8 == 0
  const int items = g.w * g.c8, nb = units_of_block(g);
  float a_dz[8] = {0, 0, 0, 0, 0, 0, 0, 0}, a_dzy[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  float sc[8], shf[8], c2[8], c3[8];  // as in bn_act_bwd_kernel
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    sc[k] = p.scale[cg * 8 + k];
    shf[k] = p.shift[cg * 8 + k];
    const float mu = p.mean[cg * 8 + k], rs = p.rstd[cg * 8 + k];
    if (APPLY) {
      const float m_dz = p.sum_dz[cg * 8 + k] * p.inv_count, m_dzy = p.sum_dzy[cg * 8 + k] * p.inv_count;
      c2[k] = -sc[k] * rs * m_dzy;
      c3[k] = -sc[k] * m_dz - c2[k] * mu;
    } else {
      c2[k] = mu;
      c3[k] = rs;
    }
  }
#pragma unroll
  for (int i = 0; i < kRingDepth - 1; ++i) {
    if (i < nb) {
      ring_issue<2>(g, p.y, 0, i, i, ring);
      ring_issue<2>(g, p.da, 1, i, i, ring);
    }
    cp_async_commit();
  }
  int st_c = 0, st_i = kRingDepth - 1;
  for (int i = 0; i < nb; ++i) {
    if (i + kRingDepth - 1 < nb) {
      ring_issue<2>(g, p.y, 0, i + kRingDepth - 1, st_i, ring);
      ring_issue<2>(g, p.da, 1, i + kRingDepth - 1, st_i, ring);
    }
    cp_async_commit();
    cp_async_wait<kRingDepth - 1>();
    int e0;
    long long rb;
    unit_pos(g, i, e0, rb);
#pragma unroll
    for (int k = 0; k < kUnitIters; ++k) {
      const int e = e0 + k * 256;
      const int x = g.c8_shift >= 0 ? e >> g.c8_shift : e / g.c8;
      uint4 vy = make_uint4(0, 0, 0, 0), vd = make_uint4(0, 0, 0, 0);  // dz = 0 beyond the row: adds nothing to the sums
      if (e < items) {
        vy = lds128(ring_slot<2>(ring, st_c, 0, k));
        vd = lds128(ring_slot<2>(ring, st_c, 1, k));
      }
      float yv[8], d[8], o[8];
      unpack8(vy, yv);
      unpack8(vd, d);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float z = fmaf(yv[q], sc[q], shf[q]);
        const float dz = d[q] * silu_grad(z);
        if (APPLY) {
          o[q] = fmaf(sc[q], dz, fmaf(c2[q], yv[q], c3[q]));
        } else {
          const float yh = (yv[q] - c2[q]) * c3[q];
          a_dz[q] += dz;
          a_dzy[q] = fmaf(dz, yh, a_dzy[q]);
        }
      }
      if (APPLY && e < items) *reinterpret_cast<uint4*>(p.dy.p + (rb + x) * p.dy.ld + p.dy.coff + cg * 8) = pack8(o);
    }
    st_c = st_c + 1 == kRingDepth ? 0 : st_c + 1;
    st_i = st_i + 1 == kRingDepth ? 0 : st_i + 1;
  }
  cp_async_wait<0>();
  if (!APPLY) {
    __syncthreads();
    block_reduce_store(a_dz, a_dzy, g.c8, sh, p.partial + static_cast<long long>(blockIdx.x) * 2 * g.c8 * 8, g.c8 * 8);
  }
}

// ---------------------------------------------------------------------------------------------- pack_weights
// w: fp32 [co, ci, k, k] (PyTorch layout).  fwd: bf16 [co_pad, (kh*k+kw)*ci + c];  dgrad: bf16 [ci_pad, (kh'*k+kw')*co + o]
// with (kh', kw') = (k-1-kh, k-1-kw).  Rows beyond co / ci stay zero (buffers are zero-initialised once).
__global__ void __launch_bounds__(256) pack_weights_kernel(const float* __restrict__ w, int co, int ci, int k,
                                                           __nv_bfloat16* __restrict__ fwd, __nv_bfloat16* __restrict__ dgr) {
  pdl_entry();
  const long long total = static_cast<long long>(co) * ci * k * k;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int kw = static_cast<int>(i % k);
    long long t = i / k;
    const int kh = static_cast<int>(t % k);
    t /= k;
    const int c = static_cast<int>(t % ci);
    const int o = static_cast<int>(t / ci);
    const __nv_bfloat16 v = __float2bfloat16(w[i]);
    if (fwd) fwd[static_cast<long long>(o) * k * k * ci + (kh * k + kw) * ci + c] = v;
    if (dgr) dgr[static_cast<long long>(c) * k * k * co + ((k - 1 - kh) * k + (k - 1 - kw)) * co + o] = v;
  }
}

// ---------------------------------------------------------------------------------------------- zero_stuff
// src: dy of a stride-2 conv, padded NHWC [n, ho+2, wo+2, ld]; dst: zero-initialised padded [n, 2ho+2, 2wo+2, c]:
// dst(2*oy, 2*ox) = src(oy, ox)  (unpadded coordinates).  Only the even positions are ever written.
__global__ void __launch_bounds__(256) zero_stuff_kernel(Slice src, SliceW dst, int n, int ho, int wo, int c8) {
  pdl_entry();
  const long long total = static_cast<long long>(n) * ho * wo * c8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % c8);
    long long t = i / c8;
    const int x = static_cast<int>(t % wo);
    t /= wo;
    const int y = static_cast<int>(t % ho);
    const int b = static_cast<int>(t / ho);
    const long long rs = (static_cast<long long>(b) * (ho + 2) + y + 1) * (wo + 2) + x + 1;
    const long long rd = (static_cast<long long>(b) * (2 * ho + 2) + 2 * y + 1) * (2 * wo + 2) + 2 * x + 1;
    *reinterpret_cast<uint4*>(dst.p + rd * dst.ld + dst.coff + cg * 8) =
        __ldg(reinterpret_cast<const uint4*>(src.p + rs * src.ld + src.coff + cg * 8));
  }
}

// ---------------------------------------------------------------------------------------------- wgrad
// dW[co, tap, ci] += sum over a chunk of padded pixels p of dy[p, co] * x[p + shift(tap), ci]   (stride-1 geometry;
// for a stride-2 conv the caller passes the zero-stuffed dy so that the same relation holds on the input grid).
// CTA tile: 64 (co) x 64 (ci) for one tap; K = pixels, consumed 32 at a time.  Both operands are "K-rows" in memory
// (pixel-major, channels contiguous), i.e. exactly the col-major A / row... fragments of mma.m16n8k16 after a transposed
// shared-memory read (ldmatrix.trans).  fp32 partial sums are reduced with atomics into the fp32 gradient.
constexpr int kWgPix = 32;    // pixels per smem stage
constexpr int kWgTile = 64;   // channels per tile side

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

struct WgradArgs {
  Slice dy;   // [rows, ld] padded pixel list, channels [coff, coff+co)
  Slice x;    // input activation, same padded geometry
  float* dw;  // fp32 [co, ci, taps] == PyTorch's [co, ci, k, k], or (ohwi) [co, taps, ci]
  int ohwi;
  int co, ci, taps, wp;
  long long rows;
  int rows_per_cta;
};

// grid: (pixel chunks, co/64 * ci/64, taps); block 128 threads (4 warps: 2x2 over the 64x64 tile, 32x32 each)
__global__ void __launch_bounds__(128) wgrad_kernel(const WgradArgs p) {
  pdl_entry();
  __shared__ __align__(16) __nv_bfloat16 s_a[kWgPix][kWgTile + 8];  // dy chunk  [pixel][co]   (+8: conflict-free ldmatrix)
  __shared__ __align__(16) __nv_bfloat16 s_b[kWgPix][kWgTile + 8];  // x chunk   [pixel][ci]
  const int tiles_ci = (p.ci + kWgTile - 1) / kWgTile;
  const int co0 = (blockIdx.y / tiles_ci) * kWgTile, ci0 = (blockIdx.y % tiles_ci) * kWgTile;
  const int tap = blockIdx.z;
  const int shift = p.taps == 9 ? (tap / 3 - 1) * p.wp + (tap % 3 - 1) : 0;
  const long long r0 = static_cast<long long>(blockIdx.x) * p.rows_per_cta;
  const long long r1 = r0 + p.rows_per_cta < p.rows ? r0 + p.rows_per_cta : p.rows;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;  // warp's 32x32 sub-tile (co, ci)
  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;

  for (long long r = r0; r < r1; r += kWgPix) {
    // stage 32 pixels x 64 channels of dy and of (shifted) x: 128 threads x 2 x 16 B each
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int idx = threadIdx.x + it * 128;  // 0..255 = 32 pixels x 8 chunks
      const int px = idx >> 3, ch = (idx & 7) * 8;
      const long long ra = r + px, rb = r + px + shift;
      uint4 va = make_uint4(0, 0, 0, 0), vb = make_uint4(0, 0, 0, 0);
      if (ra < r1 && co0 + ch < p.co) va = __ldg(reinterpret_cast<const uint4*>(p.dy.p + ra * p.dy.ld + p.dy.coff + co0 + ch));
      if (ra < r1 && rb >= 0 && rb < p.rows && ci0 + ch < p.ci)
        vb = __ldg(reinterpret_cast<const uint4*>(p.x.p + rb * p.x.ld + p.x.coff + ci0 + ch));
      *reinterpret_cast<uint4*>(&s_a[px][ch]) = va;
      *reinterpret_cast<uint4*>(&s_b[px][ch]) = vb;
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < kWgPix / 16; ++ks) {
      // A fragments (16 co x 16 pixels, row-major A[m][k] = dy[pixel k][co m]): transposed 8x8 loads from [pixel][co]
      uint32_t af[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        // matrices: (m0-7,k0-7) (m8-15,k0-7) (m0-7,k8-15) (m8-15,k8-15); smem rows are pixels (k), 8 consecutive co per row
        const int mat = lane >> 3, rr = lane & 7;
        const int kk = ks * 16 + (mat >> 1) * 8 + rr;
        const int mm = wm + mi * 16 + (mat & 1) * 8;
        ldmatrix_x4_trans(af[mi], smem_u32(&s_a[kk][mm]));
      }
      // B fragments (16 pixels x 8 ci, "col" operand B[k][n] = x[pixel k][ci n]): b0 = (k 2t..2t+1, n g), b1 = k+8
      uint32_t bf[4][2];
#pragma unroll
      for (int nj = 0; nj < 2; ++nj) {
        // one x4.trans covers two n8 tiles: matrices (k0-7,n0-7) (k8-15,n0-7) (k0-7,n8-15) (k8-15,n8-15)
        uint32_t t4[4];
        const int mat = lane >> 3, rr = lane & 7;
        const int kk = ks * 16 + (mat & 1) * 8 + rr;
        const int nn = wn + nj * 16 + (mat >> 1) * 8;
        ldmatrix_x4_trans(t4, smem_u32(&s_b[kk][nn]));
        bf[nj * 2 + 0][0] = t4[0];
        bf[nj * 2 + 0][1] = t4[1];
        bf[nj * 2 + 1][0] = t4[2];
        bf[nj * 2 + 1][1] = t4[3];
      }
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int nj = 0; nj < 4; ++nj) mma16816(acc[mi][nj], af[mi], bf[nj][0], bf[nj][1]);
    }
    __syncthreads();
  }
  // C fragment: c0,c1 = (row g, cols 2t,2t+1), c2,c3 = (row g+8, same cols)
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int nj = 0; nj < 4; ++nj) {
      const int co = co0 + wm + mi * 16 + g, ci = ci0 + wn + nj * 8 + t * 2;
      if (ci >= p.ci) continue;  // ci is a multiple of 8, so ci+1 is in range with ci
      const long long step = p.ohwi ? 1 : p.taps;  // distance between ci and ci + 1
      if (co < p.co) {
        float* d0 = p.ohwi ? p.dw + (static_cast<long long>(co) * p.taps + tap) * p.ci + ci
                           : p.dw + (static_cast<long long>(co) * p.ci + ci) * p.taps + tap;
        atomicAdd(d0, acc[mi][nj][0]);
        atomicAdd(d0 + step, acc[mi][nj][1]);
      }
      if (co + 8 < p.co) {
        float* d1 = p.ohwi ? p.dw + (static_cast<long long>(co + 8) * p.taps + tap) * p.ci + ci
                           : p.dw + (static_cast<long long>(co + 8) * p.ci + ci) * p.taps + tap;
        atomicAdd(d1, acc[mi][nj][2]);
        atomicAdd(d1 + step, acc[mi][nj][3]);
      }
    }
}

// ---------------------------------------------------------------------------------------------- bias_grad (fp32 head grads)
// g: fp32 pixel-major [rows, ld]; db[c] += sum_rows g[row, c]
__global__ void __launch_bounds__(256) colsum_f32_kernel(const float* __restrict__ g, int ld, int c, long long rows,
                                                         int rows_per_block, float* __restrict__ db) {
  pdl_entry();
  const int col = threadIdx.x % c, rl = threadIdx.x / c, nrl = blockDim.x / c;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
  const long long r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
  float s = 0.f;
  if (rl < nrl)
    for (long long r = r0 + rl; r < r1; r += nrl) s += g[r * ld + col];
  if (rl < nrl) atomicAdd(db + col, s);
}

// ---------------------------------------------------------------------------------------------- add / copy
// dst (+)= src over the interior pixels of two padded NHWC slices with the same [n,h,w,c] (gradient fan-in:
// Bottleneck shortcut, tensors with several consumers)
__global__ void __launch_bounds__(256) add_nhwc_kernel(Slice src, SliceW dst, int n, int h, int w, int c8, int accumulate) {
  pdl_entry();
  const long long total = static_cast<long long>(n) * h * w * c8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % c8);
    long long t = i / c8;
    const int x = static_cast<int>(t % w);
    t /= w;
    const int y = static_cast<int>(t % h);
    const int b = static_cast<int>(t / h);
    const long long row = (static_cast<long long>(b) * (h + 2) + y + 1) * (w + 2) + x + 1;
    uint4 v = __ldg(reinterpret_cast<const uint4*>(src.p + row * src.ld + src.coff + cg * 8));
    uint4* d = reinterpret_cast<uint4*>(dst.p + row * dst.ld + dst.coff + cg * 8);
    if (accumulate) {
      float a[8], bq[8];
      unpack8(v, a);
      unpack8(*d, bq);
#pragma unroll
      for (int k = 0; k < 8; ++k) a[k] += bq[k];
      v = pack8(a);
    }
    *d = v;
  }
}

// ---------------------------------------------------------------------------------------------- im2col of the image
// Training treats layer 0 (3x3, c_in = 3) as a 1x1 convolution over this buffer so that forward, dgrad-free backward
// and wgrad reuse the generic kernels: out[pixel][(c*3+kh)*3+kw] = image[c][y+kh-1][x+kw-1] (zero outside), 27 -> 32.
template <typename TIN>
__global__ void __launch_bounds__(256) im2col_first_kernel(const TIN* __restrict__ in, float div, int n, int h, int w,
                                                           SliceW out) {
  pdl_entry();
  const long long total = static_cast<long long>(n) * h * w;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % w);
    const long long t = i / w;
    const int y = static_cast<int>(t % h);
    const int b = static_cast<int>(t / h);
    float v[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) v[k] = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int yy = y + kh - 1, xx = x + kw - 1;
          if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
            const float px = static_cast<float>(in[((static_cast<long long>(b) * 3 + c) * h + yy) * w + xx]);
            v[(c * 3 + kh) * 3 + kw] = div > 0.f ? px / div : px;
          }
        }
    const long long row = (static_cast<long long>(b) * (h + 2) + y + 1) * (w + 2) + x + 1;
    uint4* d = reinterpret_cast<uint4*>(out.p + row * out.ld + out.coff);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float f[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] = v[q * 8 + k];
      d[q] = pack8(f);
    }
  }
}

// ---------------------------------------------------------------------------------------------- batched weight packs
// The fp32 master weights live in ONE flat buffer, every conv weight stored [co][kh][kw][ci] (PyTorch channels_last
// strides of the [co,ci,k,k] parameter) — which IS the forward pack's order.  Per optimizer step the whole buffer is
// converted to bf16 by one elementwise kernel (the forward packs are views of that copy) and ONE launch of the kernel
// below transposes every layer into its dgrad pack [ci_pad][(k-1-kh)*k + (k-1-kw)][co].  71 per-layer launches with
// scattered 2-byte stores become two bandwidth-bound ones.
__global__ void __launch_bounds__(256) f32_to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n8) {
  pdl_entry();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(src) + 2 * i), b = __ldg(reinterpret_cast<const float4*>(src) + 2 * i + 1);
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    reinterpret_cast<uint4*>(dst)[i] = pack8(f);
  }
}

// one 32(co) x 32(ci) transpose tile per block iteration; tiles of all layers are numbered consecutively (tile_begin)
__global__ void __launch_bounds__(256) pack_dgrad_batched_kernel(const y3_pack_item* __restrict__ items, int n_items,
                                                                 const __nv_bfloat16* __restrict__ wbf, int total_tiles) {
  pdl_entry();
  __shared__ __nv_bfloat16 tile[32][34];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    int lo = 0, hi = n_items - 1;  // the layer this tile belongs to
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (items[mid].tile_begin <= t) lo = mid; else hi = mid - 1;
    }
    const y3_pack_item it = items[lo];
    const int taps = it.k * it.k;
    const int tiles_ci = (it.ci + 31) / 32, tiles_co = (it.co_rows + 31) / 32;
    int local = t - it.tile_begin;
    const int tap = local / (tiles_ci * tiles_co);
    local -= tap * tiles_ci * tiles_co;
    const int co0 = (local / tiles_ci) * 32, ci0 = (local % tiles_ci) * 32;
    const __nv_bfloat16* src = wbf + it.src_off;  // [co_rows][taps][ci]
    __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(it.dst);  // [ci_pad][taps][dst_co]
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int co = co0 + ty + j * 8, ci = ci0 + tx;
      tile[ty + j * 8][tx] = (co < it.co_rows && ci < it.ci) ? src[(static_cast<long long>(co) * taps + tap) * it.ci + ci]
                                                             : __float2bfloat16(0.f);
    }
    __syncthreads();
    const int ftap = taps - 1 - tap;  // (k-1-kh)*k + (k-1-kw)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ci = ci0 + ty + j * 8, co = co0 + tx;
      if (ci < it.ci && co < it.dst_co) dst[(static_cast<long long>(ci) * taps + ftap) * it.dst_co + co] = tile[tx][ty + j * 8];
    }
  }
}

// ---------------------------------------------------------------------------------------------- Detect-head gradient
// g: dL/draw fp32 [n, na, ny, nx, no] (the loss kernel's output) -> dy bf16 padded NHWC [n, ny+2, nx+2, ld], channel a*no+o
// (the head conv's output order), plus per-block partial column sums (bias gradient; second stage = colreduce_kernel).
// Thread t owns channel t: consecutive threads read consecutive o of one anchor (coalesced) and write consecutive channels.
__global__ void __launch_bounds__(256) head_grad_pack_kernel(const float* __restrict__ g, int n, int na, int ny, int nx, int no,
                                                             SliceW dy, float* __restrict__ partial) {
  pdl_entry();
  const int ch = threadIdx.x, co = na * no;
  const int a = ch / no, o = ch - a * no;
  float acc = 0.f;
  const int rows = n * ny;
  for (int r = blockIdx.x; r < rows; r += gridDim.x) {
    const int b = r / ny, y = r - b * ny;
    const long long drow = (static_cast<long long>(b) * (ny + 2) + y + 1) * (nx + 2) + 1;
    const float* src = g + ((static_cast<long long>(b) * na + a) * ny + y) * nx * no + o;
    for (int x = 0; x < nx; ++x) {
      float v = 0.f;
      if (ch < co) v = __ldg(src + static_cast<long long>(x) * no);
      acc += v;
      if (ch < dy.ld - dy.coff) dy.p[(drow + x) * dy.ld + dy.coff + ch] = __float2bfloat16(v);
    }
  }
  partial[static_cast<long long>(blockIdx.x) * 256 + ch] = acc;
}

int grid_for(long long total, int per_block = 256, int cap_mult = 32) {
  long long b = (total + per_block - 1) / per_block;
  const long long cap = static_cast<long long>(num_sms()) * cap_mult;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<int>(b);
}

}  // namespace
}  // namespace y3

// =============================================================================================== C ABI
using y3::Slice;
using y3::SliceW;

namespace y3 {
namespace {
int log2_or_neg(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return (1 << l) == v ? l : -1;
}
Rows make_rows(int n, int h, int w, int c) {
  Rows g;
  g.n = n;
  g.h = h;
  g.w = w;
  g.c8 = c / 8;
  g.c8_shift = log2_or_neg(g.c8);
  g.upr = (w * g.c8 + 256 * kUnitIters - 1) / (256 * kUnitIters);
  return g;
}
int g_bn_async = -1;
int bn_async_enabled() {
  if (g_bn_async < 0) {
    const char* e = getenv("Y3_BN_ASYNC");
    g_bn_async = e ? (e[0] != '0') : Y3_BN_ASYNC_DEFAULT;
  }
  return g_bn_async;
}
// ring kernels: opt in to > 48 KB of dynamic shared memory and ask for the largest shared-memory carve-out, so that three
// 64 KB blocks are resident per SM (both attributes are idempotent; the carve-out is a hint)
template <auto Kern>
cudaError_t allow_smem(int bytes) {
  static bool done = false;  // per kernel; benign race: idempotent attributes.  Set on the first (eager, warm-up) launch
  if (done) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributePreferredSharedMemoryCarveout, static_cast<int>(cudaSharedmemCarveoutMaxShared));
  if (e == cudaSuccess && bytes > 48 * 1024) e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  done = e == cudaSuccess;
  return e;
}
constexpr int kMaxPartialBlocks = 396;  // = 3 resident 256-thread blocks per SM x 132 SMs (H100): exactly one wave of the reduction
                                        // kernels (a partial second wave doubles the small layers' time); fixed: sizes stay device-independent

__global__ void __launch_bounds__(1024) bn_bwd_finalize_kernel(const float* __restrict__ partial, int nblk, int c,
                                                               float* __restrict__ sums, float* __restrict__ dbeta_acc,
                                                               float* __restrict__ dgamma_acc) {
  pdl_entry();
  __shared__ float sh[32][33];
  const int j = blockIdx.x * 32 + threadIdx.x;
  const float a = colsum_32x32(partial, nblk, 2ll * c, j, j < 2 * c, sh);
  if (threadIdx.y != 0 || j >= 2 * c) return;
  sums[j] = a;
  if (j < c) {
    if (dbeta_acc) dbeta_acc[j] += a;
  } else if (dgamma_acc) {
    dgamma_acc[j - c] += a;
  }
}
}  // namespace
}  // namespace y3

extern "C" int y3_set_bn_async(int32_t on) {
  const int prev = y3::bn_async_enabled();
  y3::g_bn_async = on ? 1 : 0;
  return prev;
}

extern "C" int32_t y3_bn_partial_blocks(int32_t n, int32_t h, int32_t w, int32_t c) {
  // work units of the streaming kernels (c == 0: one unit per image row, the Detect-head gradient pack), capped
  long long units = static_cast<long long>(n) * h;
  if (c > 0) units *= (static_cast<long long>(w) * (c / 8) + 256 * y3::kUnitIters - 1) / (256 * y3::kUnitIters);
  return static_cast<int32_t>(units < y3::kMaxPartialBlocks ? (units > 0 ? units : 1) : y3::kMaxPartialBlocks);
}

extern "C" int y3_bn_stats(const void* y, int32_t ld, int32_t coff, int32_t c, int32_t n, int32_t h, int32_t w, float* partial,
                           y3_stream_t stream) {
  Y3_REQUIRE(y && partial && c > 0 && c % 8 == 0 && 256 % (c / 8) == 0 && n > 0 && h > 0 && w > 0 && ld % 8 == 0 && coff % 8 == 0,
             "bn_stats: bad arguments (c must be a power of two in [8, 2048])");
  const int nblk = y3_bn_partial_blocks(n, h, w, c);
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_stats_kernel, dim3(nblk), dim3(256), 2 * 256 * 8 * sizeof(float), static_cast<cudaStream_t>(stream), Slice{static_cast<const __nv_bfloat16*>(y), ld, coff}, y3::make_rows(n, h, w, c), partial));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_colreduce_f32(const float* partial, int32_t nblk, int32_t width, float* out, int32_t accumulate,
                                y3_stream_t stream) {
  Y3_REQUIRE(partial && out && nblk > 0 && width > 0, "colreduce: bad arguments");
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::colreduce_kernel, dim3((width + 31) / 32), dim3(32, 32), 0, static_cast<cudaStream_t>(stream), partial, nblk, width, out, accumulate));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_bn_finalize(const float* partial, int32_t nblk, const float* gamma, const float* beta, int32_t c, float count,
                              float eps, float momentum, float* scale, float* shift, float* mean, float* rstd,
                              float* running_mean, float* running_var, y3_stream_t stream) {
  Y3_REQUIRE(partial && nblk > 0 && gamma && beta && scale && shift && mean && rstd && c > 0 && count > 0, "bn_finalize: bad arguments");
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_finalize_kernel, dim3((c + 31) / 32), dim3(32, 32), 0, static_cast<cudaStream_t>(stream), partial, nblk, gamma, beta, c, count, eps, momentum, scale, shift, mean, rstd, running_mean, running_var));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_bn_act_fwd(const y3_bn_act_desc* d, y3_stream_t stream) {
  Y3_REQUIRE(d && d->y && d->out && d->scale && d->shift && d->c % 8 == 0 && d->n > 0 && d->h > 0 && d->w > 0,
             "bn_act_fwd: bad arguments");
  y3::BnActArgs a;
  a.y = Slice{static_cast<const __nv_bfloat16*>(d->y), d->y_ld, d->y_coff};
  a.res = Slice{static_cast<const __nv_bfloat16*>(d->res), d->res_ld, d->res_coff};
  a.out = SliceW{static_cast<__nv_bfloat16*>(d->out), d->out_ld, d->out_coff};
  a.scale = d->scale;
  a.shift = d->shift;
  a.g = y3::make_rows(d->n, d->h, d->w, d->c);
  a.upsample = d->upsample;
  const long long units = static_cast<long long>(d->n) * d->h * a.g.upr;
  const long long cap = 8ll * y3::num_sms();
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_act_fwd_kernel, dim3(static_cast<unsigned>(units < cap ? units : cap)), dim3(256), 0, static_cast<cudaStream_t>(stream), a));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_bn_act_bwd(const y3_bn_bwd_desc* d, y3_stream_t stream_) {
  Y3_REQUIRE(d && d->y && d->da && d->dy && d->scale && d->shift && d->mean && d->rstd && d->sums, "bn_act_bwd: null pointer");
  Y3_REQUIRE(d->c % 8 == 0 && 256 % (d->c / 8) == 0 && d->n > 0 && d->h > 0 && d->w > 0,
             "bn_act_bwd: bad shape (c must be a power of two in [8, 2048])");
  Y3_REQUIRE(d->phase >= 0 && d->phase <= 2 && d->count >= 0.f, "bn_act_bwd: bad phase/count");
  Y3_REQUIRE(d->phase == 2 || d->partial, "bn_act_bwd: the reduction phase needs the partial-sum workspace");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  y3::BnBwdArgs a;
  a.y = Slice{static_cast<const __nv_bfloat16*>(d->y), d->y_ld, d->y_coff};
  a.da = Slice{static_cast<const __nv_bfloat16*>(d->da), d->da_ld, d->da_coff};
  a.dy = SliceW{static_cast<__nv_bfloat16*>(d->dy), d->dy_ld, d->dy_coff};
  a.scale = d->scale;
  a.shift = d->shift;
  a.mean = d->mean;
  a.rstd = d->rstd;
  a.sum_dz = d->sums;
  a.sum_dzy = d->sums + d->c;
  a.partial = d->partial;
  a.g = y3::make_rows(d->n, d->h, d->w, d->c);
  a.upsample = d->upsample;
  const long long pixels = static_cast<long long>(d->n) * d->h * d->w;
  a.inv_count = 1.0f / (d->count > 0.f ? d->count : static_cast<float>(pixels));
  const int nblk = y3_bn_partial_blocks(d->n, d->h, d->w, d->c);
  const bool async = y3::bn_async_enabled() != 0;
  if (d->phase != 2) {
    if (d->upsample)
      Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_act_bwd_kernel<false, true>, dim3(nblk), dim3(256), 2 * 256 * 8 * sizeof(float), stream, a));
    else if (async) {
      Y3_CHECK_CUDA(y3::allow_smem<y3::bn_act_bwd_async_kernel<false>>(y3::ring_bytes<2>()));
      Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_act_bwd_async_kernel<false>, dim3(nblk), dim3(256), y3::ring_bytes<2>(), stream, a));
    } else
      Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_act_bwd_kernel<false, false>, dim3(nblk), dim3(256), 2 * 256 * 8 * sizeof(float), stream, a));
    Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_bwd_finalize_kernel, dim3((2 * d->c + 31) / 32), dim3(32, 32), 0, stream, d->partial, nblk, d->c, d->sums, d->dbeta_acc,
                                                                                  d->dgamma_acc));
  }
  if (d->phase != 1) {
    const long long units = static_cast<long long>(d->n) * d->h * a.g.upr;
    const long long cap = 3ll * y3::num_sms();  // one wave at the kernel's 3 resident blocks per SM
    if (d->upsample)
      Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_act_bwd_kernel<true, true>, dim3(static_cast<unsigned>(units < cap ? units : cap)), dim3(256), 0, stream, a));
    else if (async) {
      Y3_CHECK_CUDA(y3::allow_smem<y3::bn_act_bwd_async_kernel<true>>(y3::ring_bytes<2>()));
      Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_act_bwd_async_kernel<true>, dim3(static_cast<unsigned>(units < cap ? units : cap)), dim3(256), y3::ring_bytes<2>(), stream, a));
    } else
      Y3_CHECK_CUDA(::y3::launch_pdl(y3::bn_act_bwd_kernel<true, false>, dim3(static_cast<unsigned>(units < cap ? units : cap)), dim3(256), 0, stream, a));
  }
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_f32_to_bf16(const float* src, void* dst, int64_t n, y3_stream_t stream) {
  Y3_REQUIRE(src && dst && n > 0 && n % 8 == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(dst) & 15) == 0, "f32_to_bf16: n must be a multiple of 8, pointers 16-byte aligned");
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::f32_to_bf16_kernel, dim3(y3::grid_for(n / 8, 256, 16)), dim3(256), 0, static_cast<cudaStream_t>(stream), src, static_cast<__nv_bfloat16*>(dst), n / 8));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_pack_dgrad_batched(const y3_pack_item* items_dev, int32_t n_items, const void* wbf, int32_t total_tiles,
                                     y3_stream_t stream) {
  Y3_REQUIRE(items_dev && wbf && n_items > 0 && total_tiles > 0, "pack_dgrad_batched: bad arguments");
  const int cap = 16 * y3::num_sms();
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::pack_dgrad_batched_kernel, dim3(total_tiles < cap ? total_tiles : cap), dim3(256), 0, static_cast<cudaStream_t>(stream), items_dev, n_items, static_cast<const __nv_bfloat16*>(wbf), total_tiles));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_head_grad_pack(const float* g, int32_t n, int32_t na, int32_t ny, int32_t nx, int32_t no, void* dy,
                                 int32_t dy_ld, int32_t dy_coff, float* partial, y3_stream_t stream) {
  Y3_REQUIRE(g && dy && partial && n > 0 && na > 0 && ny > 0 && nx > 0 && no > 0 && na * no <= 256 && dy_ld - dy_coff <= 256,
             "head_grad_pack: bad arguments (na*no <= 256)");
  const int nblk = y3_bn_partial_blocks(n, ny, 0, 0);
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::head_grad_pack_kernel, dim3(nblk), dim3(256), 0, static_cast<cudaStream_t>(stream), g, n, na, ny, nx, no, SliceW{static_cast<__nv_bfloat16*>(dy), dy_ld, dy_coff}, partial));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_pack_weights(const float* w, int32_t co, int32_t ci, int32_t k, void* fwd, void* dgrad,
                               y3_stream_t stream) {
  Y3_REQUIRE(w && (fwd || dgrad) && co > 0 && ci > 0 && (k == 1 || k == 3), "pack_weights: bad arguments");
  const long long total = static_cast<long long>(co) * ci * k * k;
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::pack_weights_kernel, dim3(y3::grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), w, co, ci, k, static_cast<__nv_bfloat16*>(fwd), static_cast<__nv_bfloat16*>(dgrad)));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_zero_stuff(const void* src, int32_t src_ld, int32_t src_coff, void* dst, int32_t dst_ld, int32_t dst_coff,
                             int32_t n, int32_t ho, int32_t wo, int32_t c, y3_stream_t stream) {
  Y3_REQUIRE(src && dst && c % 8 == 0 && n > 0 && ho > 0 && wo > 0, "zero_stuff: bad arguments");
  const long long total = static_cast<long long>(n) * ho * wo * (c / 8);
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::zero_stuff_kernel, dim3(y3::grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), Slice{static_cast<const __nv_bfloat16*>(src), src_ld, src_coff}, SliceW{static_cast<__nv_bfloat16*>(dst), dst_ld, dst_coff}, n,
      ho, wo, c / 8));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_conv_wgrad(const y3_wgrad_desc* d, y3_stream_t stream) {
  Y3_REQUIRE(d && d->dy && d->x && d->dw, "wgrad: null pointer");
  Y3_REQUIRE(d->co % 8 == 0 && d->ci % 8 == 0 && (d->ksize == 1 || d->ksize == 3) && d->n > 0 && d->h > 0 && d->w > 0,
             "wgrad: c_out/c_in must be multiples of 8 (got %d/%d), ksize 1|3", d->co, d->ci);
  Y3_REQUIRE(d->dy_ld % 8 == 0 && d->dy_coff % 8 == 0 && d->x_ld % 8 == 0 && d->x_coff % 8 == 0, "wgrad: bad slices");
  Y3_REQUIRE(d->stride == 0 || d->stride == 1 || (d->stride == 2 && y3::wgrad_tc_enabled() && d->ci % 32 == 0),
             "wgrad: stride must be 1, or 2 with the tensor-core kernel (c_in % 32 == 0)");
  // wgmma kernel (csrc/y3_wgrad_tc.cu) whenever its tiling fits; the warp-level MMA kernel below otherwise
  if (y3::wgrad_tc_enabled() && d->ci % 32 == 0 && (reinterpret_cast<uintptr_t>(d->dy) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(d->x) & 15) == 0)
    return y3::wgrad_tc(*d, static_cast<cudaStream_t>(stream));
  Y3_REQUIRE(d->dw_layout == Y3_DW_OIHW || d->dw_layout == Y3_DW_OHWI,
             "wgrad: the tap-major accumulation layout needs the tensor-core kernel (c_in % 32 == 0)");
  Y3_REQUIRE(d->stride != 2, "wgrad: the direct stride-2 form needs the tensor-core kernel (c_in % 32 == 0)");
  y3::WgradArgs a;
  a.ohwi = d->dw_layout == Y3_DW_OHWI ? 1 : 0;
  a.dy = Slice{static_cast<const __nv_bfloat16*>(d->dy), d->dy_ld, d->dy_coff};
  a.x = Slice{static_cast<const __nv_bfloat16*>(d->x), d->x_ld, d->x_coff};
  a.dw = d->dw;
  a.co = d->co;
  a.ci = d->ci;
  a.taps = d->ksize * d->ksize;
  a.wp = d->w + 2;
  a.rows = static_cast<long long>(d->n) * (d->h + 2) * (d->w + 2);
  // split the pixel dimension so that the grid fills the machine ~4x
  const int t_co = (d->co + 63) / 64, t_ci = (d->ci + 63) / 64;
  const long long tiles = static_cast<long long>(t_co) * t_ci * a.taps;
  long long chunks = (4ll * y3::num_sms() + tiles - 1) / tiles;
  const long long max_chunks = (a.rows + 1023) / 1024;
  if (chunks > max_chunks) chunks = max_chunks;
  if (chunks < 1) chunks = 1;
  long long rpc = (a.rows + chunks - 1) / chunks;
  rpc = (rpc + y3::kWgPix - 1) / y3::kWgPix * y3::kWgPix;
  chunks = (a.rows + rpc - 1) / rpc;
  a.rows_per_cta = static_cast<int>(rpc);
  const dim3 grid(static_cast<unsigned>(chunks), static_cast<unsigned>(t_co * t_ci), a.taps);
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::wgrad_kernel, dim3(grid), dim3(128), 0, static_cast<cudaStream_t>(stream), a));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_conv_wgrad_s2_supported(int32_t h, int32_t w) { return y3::wgrad_tc_enabled() ? y3::wgrad_tc_s2_supported(h, w) : 0; }

extern "C" int y3_conv_wgrad_tap_major(int32_t c_in) { return (y3::wgrad_tc_enabled() && c_in % 32 == 0) ? 1 : 0; }

extern "C" int y3_colsum_f32(const float* g, int32_t ld, int32_t c, int64_t rows, float* out, y3_stream_t stream) {
  Y3_REQUIRE(g && out && c > 0 && c <= 256 && rows > 0, "colsum: bad arguments");
  const int rows_per_block = 1024;
  const long long blocks = (rows + rows_per_block - 1) / rows_per_block;
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::colsum_f32_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, static_cast<cudaStream_t>(stream), g, ld, c, rows, rows_per_block, out));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_add_nhwc(const void* src, int32_t src_ld, int32_t src_coff, void* dst, int32_t dst_ld, int32_t dst_coff,
                           int32_t n, int32_t h, int32_t w, int32_t c, int32_t accumulate, y3_stream_t stream) {
  Y3_REQUIRE(src && dst && c % 8 == 0 && n > 0 && h > 0 && w > 0, "add_nhwc: bad arguments");
  const long long total = static_cast<long long>(n) * h * w * (c / 8);
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::add_nhwc_kernel, dim3(y3::grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), Slice{static_cast<const __nv_bfloat16*>(src), src_ld, src_coff}, SliceW{static_cast<__nv_bfloat16*>(dst), dst_ld, dst_coff}, n, h,
      w, c / 8, accumulate));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_im2col_first(const void* in, int32_t in_dtype, float in_div, int32_t n, int32_t h, int32_t w, void* out,
                               int32_t out_ld, int32_t out_coff, y3_stream_t stream) {
  Y3_REQUIRE(in && out && n > 0 && h > 0 && w > 0 && out_ld % 8 == 0 && out_coff % 8 == 0 && out_coff + 32 <= out_ld,
             "im2col_first: bad arguments");
  const long long total = static_cast<long long>(n) * h * w;
  const SliceW o{static_cast<__nv_bfloat16*>(out), out_ld, out_coff};
  if (in_dtype == Y3_IN_U8)
    Y3_CHECK_CUDA(::y3::launch_pdl(y3::im2col_first_kernel<uint8_t>, dim3(y3::grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), static_cast<const uint8_t*>(in), in_div, n, h, w, o));
  else
    Y3_CHECK_CUDA(::y3::launch_pdl(y3::im2col_first_kernel<float>, dim3(y3::grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), static_cast<const float*>(in), in_div, n, h, w, o));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
