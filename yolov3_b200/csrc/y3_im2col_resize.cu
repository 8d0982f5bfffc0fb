// yolov3_b200 — the multi-scale rescale of the reference's training loop (train.py:394-399: imgs.float() / 255, then
// F.interpolate(imgs, size=ns, mode="bilinear", align_corners=False)) fused into layer 0's im2col.
//
// The arithmetic restates torch's CUDA upsample_bilinear2d (no scale factors given) operation for operation.  build.py
// compiles this file like torch compiles its own kernels: no fast math, FMA contraction on, so that the same expressions
// contract the same way and the result stays within one bf16 step of im2col_first(F.interpolate(...)).
//
// Each 256-thread block owns a 32 x 8 tile of output pixels of one image.  It first computes the rescaled tile plus a
// one-pixel border for the three channels into shared memory (zero outside the image: the 3x3 conv's padding), then each
// thread builds its pixel's 27 taps from there and stores them, with 5 zero columns, as four 16-byte vectors.  Per output
// pixel the kernel writes the 64-byte im2col row and reads a few bytes of the source; the unfused path also writes and
// reads two fp32 copies of the batch.
#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {
namespace {

constexpr int kTileW = 32, kTileH = 8;
constexpr int kSmemW = kTileW + 2, kSmemH = kTileH + 2;

// area_pixel_compute_source_index (aten/src/ATen/native/cuda/UpSample.cuh), align_corners = false, not cubic
__device__ __forceinline__ float source_index(float scale, int dst) {
  const float src = scale * (dst + 0.5f) - 0.5f;
  return src < 0.f ? 0.f : src;
}

// imgs.float() / 255: torch multiplies by the reciprocal of a CPU scalar (inv = 1 leaves an fp32 source exact)
template <typename TIN>
__device__ __forceinline__ float load_px(const TIN* p, float inv) {
  return static_cast<float>(__ldg(p)) * inv;
}

template <typename TIN>
__global__ void __launch_bounds__(kTileW * kTileH) im2col_first_resize_kernel(const TIN* __restrict__ in, float inv, int src_h,
                                                                              int src_w, int h, int w, float rh, float rw,
                                                                              __nv_bfloat16* __restrict__ out, int out_ld,
                                                                              int out_coff) {
  pdl_entry();
  __shared__ float tile[3][kSmemH][kSmemW];
  const int b = blockIdx.z, x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
  for (int e = threadIdx.x; e < 3 * kSmemH * kSmemW; e += blockDim.x) {
    const int c = e / (kSmemH * kSmemW), r = (e / kSmemW) % kSmemH, col = e % kSmemW;
    const int oy = y0 + r - 1, ox = x0 + col - 1;
    float v = 0.f;
    if (oy >= 0 && oy < h && ox >= 0 && ox < w) {
      // upsample_bilinear2d_out_frame (aten/src/ATen/native/cuda/UpSampleBilinear2d.cu)
      const float h1r = source_index(rh, oy);
      const int h1 = static_cast<int>(h1r);
      const int h1p = (h1 < src_h - 1) ? 1 : 0;
      const float h1lambda = h1r - h1;
      const float h0lambda = 1.f - h1lambda;
      const float w1r = source_index(rw, ox);
      const int w1 = static_cast<int>(w1r);
      const int w1p = (w1 < src_w - 1) ? 1 : 0;
      const float w1lambda = w1r - w1;
      const float w0lambda = 1.f - w1lambda;
      const TIN* p = in + ((static_cast<long long>(b) * 3 + c) * src_h + h1) * src_w + w1;
      const float a = load_px(p, inv), bb = load_px(p + w1p, inv);
      const float cc = load_px(p + static_cast<long long>(h1p) * src_w, inv);
      const float d = load_px(p + static_cast<long long>(h1p) * src_w + w1p, inv);
      v = h0lambda * (w0lambda * a + w1lambda * bb) + h1lambda * (w0lambda * cc + w1lambda * d);
    }
    tile[c][r][col] = v;
  }
  __syncthreads();
  const int tx = threadIdx.x % kTileW, ty = threadIdx.x / kTileW;
  const int x = x0 + tx, y = y0 + ty;
  if (x >= w || y >= h) return;
  float v[32];
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) v[(c * 3 + kh) * 3 + kw] = tile[c][ty + kh][tx + kw];
#pragma unroll
  for (int k = 27; k < 32; ++k) v[k] = 0.f;
  const long long row = (static_cast<long long>(b) * (h + 2) + y + 1) * (w + 2) + x + 1;
  uint4* dst = reinterpret_cast<uint4*>(out + row * out_ld + out_coff);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = v[q * 8 + k];
    dst[q] = pack8(f);
  }
}

}  // namespace
}  // namespace y3

extern "C" int y3_im2col_first_resize(const void* in, int32_t in_dtype, float in_div, int32_t n, int32_t src_h, int32_t src_w,
                                      int32_t h, int32_t w, void* out, int32_t out_ld, int32_t out_coff, y3_stream_t stream) {
  Y3_REQUIRE(in && out && n > 0 && n <= 65535 && src_h > 0 && src_w > 0 && h > 0 && w > 0 && out_ld % 8 == 0 &&
                 out_coff % 8 == 0 && out_coff + 32 <= out_ld && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "im2col_first_resize: bad arguments");
  Y3_REQUIRE(in_dtype == Y3_IN_U8 || in_dtype == Y3_IN_F32, "im2col_first_resize: bad input dtype %d", in_dtype);
  // area_pixel_compute_scale: float(input_size) / output_size, on the host like torch
  const float rh = static_cast<float>(src_h) / h, rw = static_cast<float>(src_w) / w;
  const float inv = in_div > 0.f ? 1.0f / in_div : 1.0f;
  const dim3 grid((w + y3::kTileW - 1) / y3::kTileW, (h + y3::kTileH - 1) / y3::kTileH, n);
  const dim3 block(y3::kTileW * y3::kTileH);
  auto* o = static_cast<__nv_bfloat16*>(out);
  if (in_dtype == Y3_IN_U8)
    Y3_CHECK_CUDA(::y3::launch_pdl(y3::im2col_first_resize_kernel<uint8_t>, grid, block, 0, static_cast<cudaStream_t>(stream),
                                   static_cast<const uint8_t*>(in), inv, src_h, src_w, h, w, rh, rw, o, out_ld, out_coff));
  else
    Y3_CHECK_CUDA(::y3::launch_pdl(y3::im2col_first_resize_kernel<float>, grid, block, 0, static_cast<cudaStream_t>(stream),
                                   static_cast<const float*>(in), inv, src_h, src_w, h, w, rh, rw, o, out_ld, out_coff));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
