// yolov3_b200 — layer-0 convolution (c_in = 3): 3x3 stride-1 pad-1 on the NCHW image (fp32, or uint8 with the /255 of
// detect.py:190 fused) with folded BN + SiLU, fused with the NCHW -> padded-NHWC-bf16 conversion.  Bandwidth-bound
// (24.7 FLOP/B, SURVEY App. A).  v1 was one thread per pixel with fp32 FMAs (LDS/FMA-bound); this version feeds warp-level bf16 MMAs from a shared-memory patch.
// Also the test-only layout converters.
// Replaces Conv.forward_fuse for model.0 (reference models/common.py:77-81, models/yolov3.yaml:18).
#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {
namespace {

template <typename TIN>
__device__ __forceinline__ float load_px(const TIN* p, float div);
template <>
__device__ __forceinline__ float load_px<float>(const float* p, float div) {
  const float v = __ldg(p);
  return div > 0.f ? __fdiv_rn(v, div) : v;
}
template <>
__device__ __forceinline__ float load_px<uint8_t>(const uint8_t* p, float div) {
  const float v = static_cast<float>(__ldg(p));
  return div > 0.f ? __fdiv_rn(v, div) : v;
}

// four consecutive pixels of one row (16-byte / 4-byte vector load)
template <typename TIN>
__device__ __forceinline__ float4 load_px4(const TIN* p, float div);
template <>
__device__ __forceinline__ float4 load_px4<float>(const float* p, float div) {
  float4 v = __ldg(reinterpret_cast<const float4*>(p));
  if (div > 0.f) v = make_float4(__fdiv_rn(v.x, div), __fdiv_rn(v.y, div), __fdiv_rn(v.z, div), __fdiv_rn(v.w, div));
  return v;
}
template <>
__device__ __forceinline__ float4 load_px4<uint8_t>(const uint8_t* p, float div) {
  const uchar4 u = __ldg(reinterpret_cast<const uchar4*>(p));
  float4 v = make_float4(u.x, u.y, u.z, u.w);
  if (div > 0.f) v = make_float4(__fdiv_rn(v.x, div), __fdiv_rn(v.y, div), __fdiv_rn(v.z, div), __fdiv_rn(v.w, div));
  return v;
}

// Tensor-core version (legacy warp-level mma.sync m16n8k16: K = 27 padded to 32 is far too thin for a wgmma tile and
// the layer is bandwidth-bound anyway).  One block = 128 consecutive pixels of one image row; the 3x3x(128+2) input
// patch is staged in shared memory with coalesced loads, each warp then builds the im2col A fragments for its 32 pixels
// straight from smem, multiplies by the [32 x COUT] bf16 weight fragments held in registers, and stores bf16 NHWC.
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

constexpr int kFirstRows = 8;   // output rows per block (weight fragments and the input patch are reused across them)
constexpr int kFirstTW = 128;   // output columns per block

// VEC: W % 4 == 0 and the image base is 16-byte (fp32) / 4-byte (uint8) aligned: the patch rows are staged with one
// vector load per lane, all 8 rows a warp owns in flight at once.  The scalar staging loop kept ~5 dependent 4-byte loads
// per thread in flight and most of the kernel's stall samples sat on its STS.
template <int COUT, typename TIN, bool VEC>
__global__ void __launch_bounds__(128) conv_first_kernel(const TIN* __restrict__ in, float in_div, int H, int W,
                                                         const float* __restrict__ wgt, const float* __restrict__ bias,
                                                         __nv_bfloat16* __restrict__ out, int out_ld, int out_coff) {
  pdl_entry();
  // patch column of image column ww is (ww - w0) + 4: the 128 interior columns start 16-byte aligned, halos at 3 and 132
  constexpr int TW = kFirstTW, R = kFirstRows, NT = COUT / 8, PITCH = TW + 8, C0 = 3;
  __shared__ __align__(16) float s_in[3][R + 2][PITCH];
  const int w0 = blockIdx.x * TW, h0 = blockIdx.y * R, n = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  // ---- stage the (R+2) x (TW+2) x 3 input patch (zero outside the image = the conv's padding)
  if (VEC) {
    constexpr int ROWS = 3 * (R + 2), PER_WARP = (ROWS + 3) / 4;
    float4 v[PER_WARP];
    float hv[PER_WARP];
#pragma unroll
    for (int i = 0; i < PER_WARP; ++i) {
      const int rc = warp + i * 4;  // patch row = (channel, rr)
      const int c = rc / (R + 2), rr = rc - c * (R + 2);
      const int hh = h0 + rr - 1, ww = w0 + lane * 4;
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      hv[i] = 0.f;
      if (rc < ROWS && hh >= 0 && hh < H) {
        const TIN* row = in + ((static_cast<size_t>(n) * 3 + c) * H + hh) * W;
        if (ww < W) v[i] = load_px4<TIN>(row + ww, in_div);
        const int hw = lane == 0 ? w0 - 1 : w0 + TW;  // lanes 0 / 1: left / right halo column
        if (lane < 2 && hw >= 0 && hw < W) hv[i] = load_px<TIN>(row + hw, in_div);
      }
    }
#pragma unroll
    for (int i = 0; i < PER_WARP; ++i) {
      const int rc = warp + i * 4;
      if (rc < ROWS) {
        float* dst = &s_in[0][0][0] + rc * PITCH;
        *reinterpret_cast<float4*>(dst + 4 + lane * 4) = v[i];
        if (lane < 2) dst[lane == 0 ? C0 : C0 + TW + 1] = hv[i];
      }
    }
  } else {
    for (int i = threadIdx.x; i < 3 * (R + 2) * (TW + 2); i += blockDim.x) {
      const int col = i % (TW + 2), rc = i / (TW + 2);
      const int c = rc / (R + 2), rr = rc - c * (R + 2);
      const int hh = h0 + rr - 1, ww = w0 + col - 1;
      float v = 0.f;
      if (hh >= 0 && hh < H && ww >= 0 && ww < W)
        v = load_px<TIN>(in + ((static_cast<size_t>(n) * 3 + c) * H + hh) * W + ww, in_div);
      (&s_in[0][0][0])[rc * PITCH + C0 + col] = v;
    }
  }
  // ---- weight fragments: B[k][n], k = (c*3+kh)*3+kw (27 real rows, zero padded to 32)
  uint32_t bfrag[2][NT][2];
  int a_off[2][4];  // smem offset of the 4 k-values this lane contributes per k-step (-1 = zero padding)
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = ks * 16 + t * 2 + (j & 1) + (j >> 1) * 8;
      a_off[ks][j] = k < 27 ? ((k / 9) * (R + 2) + (k % 9) / 3) * PITCH + k % 3 + C0 : -1;
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
      for (int hlf = 0; hlf < 2; ++hlf) {
        const int k = ks * 16 + t * 2 + hlf * 8, co = nt * 8 + g;
        const float lo = k < 27 ? __ldg(wgt + k * COUT + co) : 0.f;
        const float hi = k + 1 < 27 ? __ldg(wgt + (k + 1) * COUT + co) : 0.f;
        bfrag[ks][nt][hlf] = pack_bf16x2(lo, hi);
      }
    }
  }
  float bia[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    bia[nt][0] = __ldg(bias + nt * 8 + t * 2);
    bia[nt][1] = __ldg(bias + nt * 8 + t * 2 + 1);
  }
  __syncthreads();
  const float* sbase = &s_in[0][0][0];
#pragma unroll 1
  for (int rr = 0; rr < R; ++rr) {
    const int h = h0 + rr;
    if (h >= H) break;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int px = warp * 32 + mt * 16;  // first pixel (tile-relative) of this 16-row MMA tile
      float acc[NT][4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        // A fragment: a0 = (row g, k 2t..2t+1), a1 = (row g+8, same), a2 = (row g, k+8..), a3 = (row g+8, k+8..)
        float v[2][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int o = a_off[ks][j] + rr * PITCH + px + g;
          v[0][j] = a_off[ks][j] >= 0 ? sbase[o] : 0.f;
          v[1][j] = a_off[ks][j] >= 0 ? sbase[o + 8] : 0.f;
        }
        const uint32_t a[4] = {pack_bf16x2(v[0][0], v[0][1]), pack_bf16x2(v[1][0], v[1][1]), pack_bf16x2(v[0][2], v[0][3]),
                               pack_bf16x2(v[1][2], v[1][3])};
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_bf16_16816(acc[nt], a, bfrag[ks][nt]);
      }
      // C fragment: c0,c1 = (row g, cols 2t,2t+1), c2,c3 = (row g+8, same cols)
#pragma unroll
      for (int hlf = 0; hlf < 2; ++hlf) {
        uint32_t wv[NT];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
          wv[nt] = pack_bf16x2(silu_fast(acc[nt][hlf * 2 + 0] + bia[nt][0]), silu_fast(acc[nt][hlf * 2 + 1] + bia[nt][1]));
        const int w = w0 + px + g + hlf * 8;
        const size_t row = (static_cast<size_t>(n) * (H + 2) + h + 1) * (W + 2) + w + 1;
        if (NT == 4) {
          // 4x4 transpose inside each lane quad: afterwards lane t owns the 16 contiguous bytes of n-tile t
#pragma unroll
          for (int sft = 1; sft <= 2; sft <<= 1) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              if (i & sft) continue;
              const bool up = (t & sft) != 0;
              const uint32_t send = up ? wv[i] : wv[i | sft];
              const uint32_t recv = __shfl_xor_sync(0xffffffffu, send, sft);
              if (up) wv[i] = recv; else wv[i | sft] = recv;
            }
          }
          if (w < W)
            *reinterpret_cast<uint4*>(out + row * out_ld + out_coff + t * 8) = make_uint4(wv[0], wv[1], wv[2], wv[3]);
        } else if (w < W) {
          uint32_t* dst = reinterpret_cast<uint32_t*>(out + row * out_ld + out_coff);
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) dst[nt * 4 + t] = wv[nt];
        }
      }
    }
  }
}

__global__ void nchw_to_padded_kernel(const float* __restrict__ src, int C, int H, int W, __nv_bfloat16* __restrict__ dst,
                                      int ld, int coff, size_t total) {
  pdl_entry();
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int w = i % W;
  const int h = (i / W) % H;
  const int c = (i / (static_cast<size_t>(W) * H)) % C;
  const int n = i / (static_cast<size_t>(W) * H * C);
  dst[((static_cast<size_t>(n) * (H + 2) + h + 1) * (W + 2) + w + 1) * ld + coff + c] = __float2bfloat16(src[i]);
}

__global__ void padded_to_nchw_kernel(const __nv_bfloat16* __restrict__ src, int ld, int coff, int C, int H, int W,
                                      float* __restrict__ dst, size_t total) {
  pdl_entry();
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int w = i % W;
  const int h = (i / W) % H;
  const int c = (i / (static_cast<size_t>(W) * H)) % C;
  const int n = i / (static_cast<size_t>(W) * H * C);
  dst[i] = __bfloat162float(src[((static_cast<size_t>(n) * (H + 2) + h + 1) * (W + 2) + w + 1) * ld + coff + c]);
}

}  // namespace
}  // namespace y3

extern "C" int y3_conv_first_fwd(const y3_first_desc* d, y3_stream_t stream) {
  Y3_REQUIRE(d && d->in && d->weight && d->bias && d->out, "conv_first: null pointer");
  Y3_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0 && d->n <= 65535 && d->h <= 65535, "conv_first: bad shape");
  Y3_REQUIRE(d->out_ld % 8 == 0 && d->out_coff % 8 == 0 && d->out_coff + d->c_out <= d->out_ld &&
                 (reinterpret_cast<uintptr_t>(d->out) & 15) == 0,
             "conv_first: bad output slice");
  Y3_REQUIRE(d->c_out == 16 || d->c_out == 32, "conv_first: c_out=%d unsupported (16 or 32)", d->c_out);
  Y3_REQUIRE(d->in_dtype == Y3_IN_F32 || d->in_dtype == Y3_IN_U8, "conv_first: bad input dtype %d", d->in_dtype);
  const dim3 grid((d->w + y3::kFirstTW - 1) / y3::kFirstTW, (d->h + y3::kFirstRows - 1) / y3::kFirstRows, d->n), block(128);
  auto* o = static_cast<__nv_bfloat16*>(d->out);
  auto s = static_cast<cudaStream_t>(stream);
  const bool vec = d->w % 4 == 0 && (reinterpret_cast<uintptr_t>(d->in) & (d->in_dtype == Y3_IN_F32 ? 15 : 3)) == 0;
#define Y3_FIRST(CO, T)                                                                                                 \
  do {                                                                                                                  \
    if (vec)                                                                                                            \
      Y3_CHECK_CUDA(::y3::launch_pdl(y3::conv_first_kernel<CO, T, true>, dim3(grid), dim3(block), 0, s, static_cast<const T*>(d->in), d->in_div, d->h, d->w,    \
                                                                d->weight, d->bias, o, d->out_ld, d->out_coff));         \
    else                                                                                                                \
      Y3_CHECK_CUDA(::y3::launch_pdl(y3::conv_first_kernel<CO, T, false>, dim3(grid), dim3(block), 0, s, static_cast<const T*>(d->in), d->in_div, d->h, d->w,   \
                                                                 d->weight, d->bias, o, d->out_ld, d->out_coff));        \
  } while (0)
  if (d->c_out == 32) {
    if (d->in_dtype == Y3_IN_F32) Y3_FIRST(32, float); else Y3_FIRST(32, uint8_t);
  } else {
    if (d->in_dtype == Y3_IN_F32) Y3_FIRST(16, float); else Y3_FIRST(16, uint8_t);
  }
#undef Y3_FIRST
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_nchw_to_padded_nhwc(const float* src, int32_t n, int32_t c, int32_t h, int32_t w, void* dst,
                                      int32_t dst_ld, int32_t dst_coff, y3_stream_t stream) {
  Y3_REQUIRE(src && dst && n > 0 && c > 0 && h > 0 && w > 0 && dst_coff + c <= dst_ld, "nchw_to_padded: bad args");
  const size_t total = static_cast<size_t>(n) * c * h * w;
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::nchw_to_padded_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), src, c, h, w, static_cast<__nv_bfloat16*>(dst), dst_ld, dst_coff, total));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_padded_nhwc_to_nchw(const void* src, int32_t src_ld, int32_t src_coff, int32_t n, int32_t c, int32_t h,
                                      int32_t w, float* dst, y3_stream_t stream) {
  Y3_REQUIRE(src && dst && n > 0 && c > 0 && h > 0 && w > 0 && src_coff + c <= src_ld, "padded_to_nchw: bad args");
  const size_t total = static_cast<size_t>(n) * c * h * w;
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::padded_to_nchw_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(src), src_ld, src_coff, c, h, w, dst, total));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
