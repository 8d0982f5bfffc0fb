// yolov3_b200 — max-pool on padded NHWC bf16 (8 channels / 16 bytes per thread, coalesced along channels).
// Covers the three pooling uses of the shipped YAMLs:
//   * nn.MaxPool2d(2, 2, 0)                         (yolov3-tiny.yaml backbone)        k=2 stride=2 off=0
//   * nn.ZeroPad2d([0,1,0,1]) + nn.MaxPool2d(2,1,0) (yolov3-tiny.yaml layers 11-12)    k=2 stride=1 off=0 oob_zero=1
//   * SPP's MaxPool2d(k, 1, k//2), -inf padding     (reference models/common.py:279)   k=5 stride=1 off=-2 oob_zero=0
//     (9x9 and 13x13 are produced by cascading the 5x5 pool, which is exact for max with -inf padding)
#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {
namespace {

struct PoolArgs {
  const __nv_bfloat16* in;
  __nv_bfloat16* out;
  int in_ld, in_coff, out_ld, out_coff;
  int n, h, w, c8;  // input size (unpadded), channel groups of 8
  int ho, wo;
  int k, stride, off, oob_zero;
};

__device__ __forceinline__ uint32_t bf16x2_max(uint32_t a, uint32_t b) {
  __nv_bfloat162 x = *reinterpret_cast<__nv_bfloat162*>(&a), y = *reinterpret_cast<__nv_bfloat162*>(&b);
  __nv_bfloat162 m = __hmax2(x, y);
  return *reinterpret_cast<uint32_t*>(&m);
}

__global__ void __launch_bounds__(256) maxpool_kernel(const PoolArgs p) {
  pdl_entry();
  const long long total = static_cast<long long>(p.n) * p.ho * p.wo * p.c8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % p.c8);
    long long t = i / p.c8;
    const int x = static_cast<int>(t % p.wo);
    t /= p.wo;
    const int y = static_cast<int>(t % p.ho);
    const int n = static_cast<int>(t / p.ho);
    const uint32_t ninf = 0xFF80FF80u;  // two bf16 -inf
    uint4 m = make_uint4(ninf, ninf, ninf, ninf);
    bool saw_oob = false;
    for (int dy = 0; dy < p.k; ++dy) {
      const int yy = y * p.stride + p.off + dy;
      for (int dx = 0; dx < p.k; ++dx) {
        const int xx = x * p.stride + p.off + dx;
        if (yy < 0 || yy >= p.h || xx < 0 || xx >= p.w) {
          saw_oob = true;
          continue;
        }
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(
            p.in + ((static_cast<long long>(n) * (p.h + 2) + yy + 1) * (p.w + 2) + xx + 1) * p.in_ld + p.in_coff + cg * 8));
        m.x = bf16x2_max(m.x, v.x);
        m.y = bf16x2_max(m.y, v.y);
        m.z = bf16x2_max(m.z, v.z);
        m.w = bf16x2_max(m.w, v.w);
      }
    }
    if (saw_oob && p.oob_zero) {
      m.x = bf16x2_max(m.x, 0u);
      m.y = bf16x2_max(m.y, 0u);
      m.z = bf16x2_max(m.z, 0u);
      m.w = bf16x2_max(m.w, 0u);
    }
    *reinterpret_cast<uint4*>(p.out + ((static_cast<long long>(n) * (p.ho + 2) + y + 1) * (p.wo + 2) + x + 1) * p.out_ld +
                              p.out_coff + cg * 8) = m;
  }
}

// e4m3 (FP8 inference): 16 channels per thread; codes are decoded exactly to f16, maxed and re-encoded exactly, so the
// output keeps the input's scale.  -inf stands for "no element yet"; every window holds at least one in-image element.
__device__ __forceinline__ uint4 e4m3x16_max(uint4 m, uint4 v, bool first) {
  uint32_t mw[4] = {m.x, m.y, m.z, m.w}, vw[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (first) {
      mw[i] = vw[i];
      continue;
    }
    uint32_t r = 0;
#pragma unroll
    for (int hlf = 0; hlf < 2; ++hlf) {
      const float2 a = unpack_e4m3x2(static_cast<uint16_t>(mw[i] >> (16 * hlf)));
      const float2 b = unpack_e4m3x2(static_cast<uint16_t>(vw[i] >> (16 * hlf)));
      r |= static_cast<uint32_t>(pack_e4m3x2(fmaxf(a.x, b.x), fmaxf(a.y, b.y))) << (16 * hlf);
    }
    mw[i] = r;
  }
  return make_uint4(mw[0], mw[1], mw[2], mw[3]);
}

__global__ void __launch_bounds__(256) maxpool_e4m3_kernel(const PoolArgs p) {
  pdl_entry();
  const uint8_t* in = reinterpret_cast<const uint8_t*>(p.in);
  uint8_t* out = reinterpret_cast<uint8_t*>(p.out);
  const int c16 = p.c8 / 2;
  const long long total = static_cast<long long>(p.n) * p.ho * p.wo * c16;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % c16);
    long long t = i / c16;
    const int x = static_cast<int>(t % p.wo);
    t /= p.wo;
    const int y = static_cast<int>(t % p.ho);
    const int n = static_cast<int>(t / p.ho);
    uint4 m = make_uint4(0u, 0u, 0u, 0u);
    bool any = false, saw_oob = false;
    for (int dy = 0; dy < p.k; ++dy) {
      const int yy = y * p.stride + p.off + dy;
      for (int dx = 0; dx < p.k; ++dx) {
        const int xx = x * p.stride + p.off + dx;
        if (yy < 0 || yy >= p.h || xx < 0 || xx >= p.w) {
          saw_oob = true;
          continue;
        }
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(
            in + ((static_cast<long long>(n) * (p.h + 2) + yy + 1) * (p.w + 2) + xx + 1) * p.in_ld + p.in_coff + cg * 16));
        m = e4m3x16_max(m, v, !any);
        any = true;
      }
    }
    if (saw_oob && p.oob_zero) m = e4m3x16_max(m, make_uint4(0u, 0u, 0u, 0u), !any);
    *reinterpret_cast<uint4*>(out + ((static_cast<long long>(n) * (p.ho + 2) + y + 1) * (p.wo + 2) + x + 1) * p.out_ld +
                              p.out_coff + cg * 16) = m;
  }
}

// amax = max(amax, max |x|) over the interior pixels of a padded NHWC slice (FP8 calibration).  |x| >= 0, so the float
// order is the order of the bit patterns as integers: one atomicMax per block on the bits, independent of the order.
template <int FMT>
__global__ void __launch_bounds__(256) amax_kernel(const y3_amax_desc d) {
  pdl_entry();
  constexpr int kPer = FMT == Y3_FMT_E4M3 ? 16 : 8;  // channels per 16-byte vector
  const int es = FMT == Y3_FMT_E4M3 ? 1 : 2;
  const int cv = d.c / kPer;
  const long long total = static_cast<long long>(d.n) * d.h * d.w * cv;
  const uint8_t* base = reinterpret_cast<const uint8_t*>(d.x);
  float m = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % cv);
    long long t = i / cv;
    const int x = static_cast<int>(t % d.w);
    t /= d.w;
    const int y = static_cast<int>(t % d.h);
    const int n = static_cast<int>(t / d.h);
    const long long e = ((static_cast<long long>(n) * (d.h + 2) + y + 1) * (d.w + 2) + x + 1) * d.ld + d.coff + g * kPer;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(base + e * es));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (FMT == Y3_FMT_E4M3) {
        const float2 a = unpack_e4m3x2(static_cast<uint16_t>(w[k])), b = unpack_e4m3x2(static_cast<uint16_t>(w[k] >> 16));
        m = fmaxf(m, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(b.x), fabsf(b.y))));
      } else {
        const float2 a = unpack_bf16x2(w[k]);
        m = fmaxf(m, fmaxf(fabsf(a.x), fabsf(a.y)));
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(~0u, m, o));
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) m = fmaxf(m, red[k]);
    atomicMax(reinterpret_cast<unsigned int*>(d.amax), __float_as_uint(m));
  }
}

// ---------------------------------------------------------------------------------------------- training mode
// Forward with argmax: idx[n, ho, wo, c] (uint8) = dy*k + dx of the FIRST maximum in row-major window order, which is the
// element torch.nn.MaxPool2d routes the gradient to (ATen max_pool2d_with_indices: `val > maxval || isnan(val)`).
__global__ void __launch_bounds__(256) maxpool_idx_kernel(const PoolArgs p, uint8_t* __restrict__ idx) {
  pdl_entry();
  const long long total = static_cast<long long>(p.n) * p.ho * p.wo * p.c8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % p.c8);
    long long t = i / p.c8;
    const int x = static_cast<int>(t % p.wo);
    t /= p.wo;
    const int y = static_cast<int>(t % p.ho);
    const int n = static_cast<int>(t / p.ho);
    float m[8];
    uint32_t am[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      m[e] = -INFINITY;
      am[e] = 255u;  // no in-image element seen (cannot happen for pad <= k/2)
    }
    for (int dy = 0; dy < p.k; ++dy) {
      const int yy = y * p.stride + p.off + dy;
      const bool oob_y = yy < 0 || yy >= p.h;
      if (oob_y && !p.oob_zero) continue;
      for (int dx = 0; dx < p.k; ++dx) {
        const int xx = x * p.stride + p.off + dx;
        const bool oob = oob_y || xx < 0 || xx >= p.w;
        if (oob && !p.oob_zero) continue;
        // oob_zero: the window reaches into an nn.ZeroPad2d border (yolov3-tiny.yaml:29-30): the pad value 0 competes like any
        // element; if it wins, the gradient goes to the pad, i.e. nowhere (the backward gathers over real pixels only)
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (!oob)
          v = __ldg(reinterpret_cast<const uint4*>(
              p.in + ((static_cast<long long>(n) * (p.h + 2) + yy + 1) * (p.w + 2) + xx + 1) * p.in_ld + p.in_coff + cg * 8));
        float f[8];
        unpack8(v, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (f[e] > m[e] || f[e] != f[e] || am[e] == 255u) {  // ATen: (val > maxval) || isnan(val); first element seeds
            m[e] = f[e];
            am[e] = static_cast<uint32_t>(dy * p.k + dx);
          }
        }
      }
    }
    uint4 o;
    o.x = pack_bf16x2(m[0], m[1]);
    o.y = pack_bf16x2(m[2], m[3]);
    o.z = pack_bf16x2(m[4], m[5]);
    o.w = pack_bf16x2(m[6], m[7]);
    *reinterpret_cast<uint4*>(p.out + ((static_cast<long long>(n) * (p.ho + 2) + y + 1) * (p.wo + 2) + x + 1) * p.out_ld +
                              p.out_coff + cg * 8) = o;
    uint2 ii;
    ii.x = am[0] | (am[1] << 8) | (am[2] << 16) | (am[3] << 24);
    ii.y = am[4] | (am[5] << 8) | (am[6] << 16) | (am[7] << 24);
    *reinterpret_cast<uint2*>(idx + ((static_cast<long long>(n) * p.ho + y) * p.wo + x) * (p.c8 * 8) + cg * 8) = ii;
  }
}

// Backward as a gather (no atomics, deterministic): input pixel (yy, xx) collects dy of every window whose recorded argmax
// is this pixel.  `in`/`out` of PoolArgs are reused as dOut (read) / dIn (written or accumulated).
__global__ void __launch_bounds__(256) maxpool_bwd_kernel(const PoolArgs p, const uint8_t* __restrict__ idx, int accumulate) {
  pdl_entry();
  const long long total = static_cast<long long>(p.n) * p.h * p.w * p.c8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % p.c8);
    long long t = i / p.c8;
    const int xx = static_cast<int>(t % p.w);
    t /= p.w;
    const int yy = static_cast<int>(t % p.h);
    const int n = static_cast<int>(t / p.h);
    float g[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    // windows (y, x) with y*stride + off <= yy < y*stride + off + k
    for (int dy = 0; dy < p.k; ++dy) {
      const int ys = yy - p.off - dy;
      if (ys < 0 || ys % p.stride) continue;
      const int y = ys / p.stride;
      if (y >= p.ho) continue;
      for (int dx = 0; dx < p.k; ++dx) {
        const int xs = xx - p.off - dx;
        if (xs < 0 || xs % p.stride) continue;
        const int x = xs / p.stride;
        if (x >= p.wo) continue;
        const uint2 ii = __ldg(reinterpret_cast<const uint2*>(idx + ((static_cast<long long>(n) * p.ho + y) * p.wo + x) * (p.c8 * 8) + cg * 8));
        const uint32_t want = static_cast<uint32_t>(dy * p.k + dx);
        const uint32_t w4 = want * 0x01010101u;
        if (__vcmpeq4(ii.x, w4) | __vcmpeq4(ii.y, w4)) {
          const uint4 v = __ldg(reinterpret_cast<const uint4*>(
              p.in + ((static_cast<long long>(n) * (p.ho + 2) + y + 1) * (p.wo + 2) + x + 1) * p.in_ld + p.in_coff + cg * 8));
          float f[8];
          unpack8(v, f);
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const uint32_t a = ((e < 4 ? ii.x : ii.y) >> (8 * (e & 3))) & 255u;
            if (a == want) g[e] += f[e];
          }
        }
      }
    }
    __nv_bfloat16* dst = p.out + ((static_cast<long long>(n) * (p.h + 2) + yy + 1) * (p.w + 2) + xx + 1) * p.out_ld + p.out_coff + cg * 8;
    if (accumulate) {
      float f[8];
      unpack8(*reinterpret_cast<const uint4*>(dst), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) g[e] += f[e];
    }
    uint4 o;
    o.x = pack_bf16x2(g[0], g[1]);
    o.y = pack_bf16x2(g[2], g[3]);
    o.z = pack_bf16x2(g[4], g[5]);
    o.w = pack_bf16x2(g[6], g[7]);
    *reinterpret_cast<uint4*>(dst) = o;
  }
}

}  // namespace

static int pool_args(const y3_pool_desc& d, PoolArgs* a) {
  Y3_REQUIRE(d.in && d.out && d.n > 0 && d.h > 0 && d.w > 0 && d.c > 0 && d.c % 8 == 0, "pool: bad shape");
  Y3_REQUIRE(d.in_ld % 8 == 0 && d.in_coff % 8 == 0 && d.out_ld % 8 == 0 && d.out_coff % 8 == 0 &&
                 d.in_coff + d.c <= d.in_ld && d.out_coff + d.c <= d.out_ld,
             "pool: bad channel slice");
  Y3_REQUIRE(d.k >= 1 && d.k <= 13 && d.stride >= 1 && d.ho > 0 && d.wo > 0, "pool: bad window");
  Y3_REQUIRE(d.fmt == Y3_FMT_BF16, "pool (train): bf16 only (fmt %d)", d.fmt);
  a->in = static_cast<const __nv_bfloat16*>(d.in);
  a->out = static_cast<__nv_bfloat16*>(d.out);
  a->in_ld = d.in_ld;
  a->in_coff = d.in_coff;
  a->out_ld = d.out_ld;
  a->out_coff = d.out_coff;
  a->n = d.n;
  a->h = d.h;
  a->w = d.w;
  a->c8 = d.c / 8;
  a->ho = d.ho;
  a->wo = d.wo;
  a->k = d.k;
  a->stride = d.stride;
  a->off = d.off;
  a->oob_zero = d.oob_zero;
  return Y3_OK;
}

static unsigned pool_grid(long long total) {
  long long blocks = (total + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 32;
  return static_cast<unsigned>(blocks > cap ? cap : blocks);
}

int pool_train_fwd(const y3_pool_desc& d, uint8_t* idx, cudaStream_t stream) {
  PoolArgs a;
  if (int rc = pool_args(d, &a)) return rc;
  Y3_REQUIRE(idx, "pool (train): idx is required");
  Y3_CHECK_CUDA(::y3::launch_pdl(maxpool_idx_kernel, dim3(pool_grid(static_cast<long long>(a.n) * a.ho * a.wo * a.c8)), dim3(256), 0, stream, a, idx));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

int pool_bwd(const y3_pool_desc& d, const uint8_t* idx, int accumulate, cudaStream_t stream) {
  PoolArgs a;
  if (int rc = pool_args(d, &a)) return rc;
  Y3_REQUIRE(idx, "pool_bwd: null idx");
  Y3_CHECK_CUDA(::y3::launch_pdl(maxpool_bwd_kernel, dim3(pool_grid(static_cast<long long>(a.n) * a.h * a.w * a.c8)), dim3(256), 0, stream, a, idx, accumulate));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

int pool_launch(const y3_pool_desc& d, cudaStream_t stream) {
  Y3_REQUIRE(d.in && d.out && d.n > 0 && d.h > 0 && d.w > 0 && d.c > 0 && d.c % 8 == 0, "pool: bad shape");
  Y3_REQUIRE(d.in_ld % 8 == 0 && d.in_coff % 8 == 0 && d.out_ld % 8 == 0 && d.out_coff % 8 == 0 &&
                 d.in_coff + d.c <= d.in_ld && d.out_coff + d.c <= d.out_ld,
             "pool: bad channel slice");
  Y3_REQUIRE(d.k >= 1 && d.k <= 13 && d.stride >= 1 && d.ho > 0 && d.wo > 0, "pool: bad window");
  Y3_REQUIRE(d.fmt == Y3_FMT_BF16 || d.fmt == Y3_FMT_E4M3, "pool: unknown format %d", d.fmt);
  if (d.fmt == Y3_FMT_E4M3)
    Y3_REQUIRE(d.c % 16 == 0 && d.in_ld % 16 == 0 && d.in_coff % 16 == 0 && d.out_ld % 16 == 0 && d.out_coff % 16 == 0,
               "pool: e4m3 needs channels, ld and coff multiples of 16");
  PoolArgs a;
  a.in = static_cast<const __nv_bfloat16*>(d.in);
  a.out = static_cast<__nv_bfloat16*>(d.out);
  a.in_ld = d.in_ld;
  a.in_coff = d.in_coff;
  a.out_ld = d.out_ld;
  a.out_coff = d.out_coff;
  a.n = d.n;
  a.h = d.h;
  a.w = d.w;
  a.c8 = d.c / 8;
  a.ho = d.ho;
  a.wo = d.wo;
  a.k = d.k;
  a.stride = d.stride;
  a.off = d.off;
  a.oob_zero = d.oob_zero;
  const long long total = static_cast<long long>(a.n) * a.ho * a.wo * a.c8 / (d.fmt == Y3_FMT_E4M3 ? 2 : 1);
  long long blocks = (total + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 32;
  if (blocks > cap) blocks = cap;
  Y3_CHECK_CUDA(::y3::launch_pdl(d.fmt == Y3_FMT_E4M3 ? maxpool_e4m3_kernel : maxpool_kernel,
                                 dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, a));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

}  // namespace y3

extern "C" int y3_maxpool_train_fwd(const y3_pool_desc* d, uint8_t* idx, y3_stream_t stream) {
  if (!d) return y3::set_error(Y3_ERR_BAD_ARG, "pool: null descriptor");
  return y3::pool_train_fwd(*d, idx, static_cast<cudaStream_t>(stream));
}

extern "C" int y3_maxpool_bwd(const y3_pool_desc* d, const uint8_t* idx, int32_t accumulate, y3_stream_t stream) {
  if (!d) return y3::set_error(Y3_ERR_BAD_ARG, "pool: null descriptor");
  return y3::pool_bwd(*d, idx, accumulate, static_cast<cudaStream_t>(stream));
}

namespace y3 {
int amax_launch(const y3_amax_desc& d, cudaStream_t stream) {
  Y3_REQUIRE(d.x && d.amax && d.n > 0 && d.h > 0 && d.w > 0 && d.c > 0, "amax: bad arguments");
  Y3_REQUIRE(d.fmt == Y3_FMT_BF16 || d.fmt == Y3_FMT_E4M3, "amax: unknown format %d", d.fmt);
  const int per = d.fmt == Y3_FMT_E4M3 ? 16 : 8;
  Y3_REQUIRE(d.c % per == 0 && d.ld % per == 0 && d.coff % per == 0 && d.coff + d.c <= d.ld,
             "amax: channels, ld and coff must be multiples of %d", per);
  Y3_REQUIRE((reinterpret_cast<uintptr_t>(d.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.amax) & 3) == 0,
             "amax: misaligned pointer");
  const long long total = static_cast<long long>(d.n) * d.h * d.w * (d.c / per);
  long long blocks = (total + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  Y3_CHECK_CUDA(::y3::launch_pdl(d.fmt == Y3_FMT_E4M3 ? amax_kernel<Y3_FMT_E4M3> : amax_kernel<Y3_FMT_BF16>,
                                 dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, d));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
}  // namespace y3

extern "C" int y3_amax_nhwc(const void* x, int32_t fmt, int32_t ld, int32_t coff, int32_t n, int32_t h, int32_t w, int32_t c,
                            float* amax, y3_stream_t stream) {
  const y3_amax_desc d{x, fmt, ld, coff, n, h, w, c, amax};
  return y3::amax_launch(d, static_cast<cudaStream_t>(stream));
}

extern "C" int y3_maxpool_fwd(const y3_pool_desc* d, y3_stream_t stream) {
  if (!d) return y3::set_error(Y3_ERR_BAD_ARG, "pool: null descriptor");
  return y3::pool_launch(*d, static_cast<cudaStream_t>(stream));
}
