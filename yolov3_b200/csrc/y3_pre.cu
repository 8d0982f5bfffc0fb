// yolov3_b200 — device-side image pre-processing (SURVEY §8(f) row f1).  Replaces, for the detect.py / val.py input path,
//   letterbox(im0, img_size, stride, auto)           utils/augmentations.py:104-134  (cv2.resize INTER_LINEAR + copyMakeBorder 114)
//   im.transpose((2, 0, 1))[::-1]; ascontiguousarray  utils/dataloaders.py:308-310   (HWC -> CHW, BGR -> RGB)
// with ONE kernel that reads the decoded uint8 HWC BGR frame and writes the letterboxed uint8 image either HWC/BGR (the
// drop-in result of letterbox) or CHW/RGB — i.e. straight into the uint8 input buffer of the engine, whose first conv applies
// the im/255 of detect.py:187-191.  The resize is OpenCV's 8-bit INTER_LINEAR restated bit for bit (y3_resize.cuh).
// Compiled without fast-math / FMA contraction (build.py EXACT_SOURCES): every float step is the one OpenCV rounds.
#include "y3_common.cuh"
#include "y3_internal.h"
#include "y3_resize.cuh"

namespace y3 {
namespace {

struct LbArgs {
  ResizeGeom rs;        // source and resize
  int top, left;        // border offsets of the resized image inside the output
  int out_h, out_w;
  uint8_t pad[3];       // border colour in SOURCE channel order
  uint8_t* dst;
  int chw, swap_rb;     // output layout / channel order
};

__global__ void __launch_bounds__(256) letterbox_kernel(const LbArgs p) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= p.out_w) return;
  int v[3] = {p.pad[0], p.pad[1], p.pad[2]};
  const int dx = x - p.left, dy = y - p.top;
  if (dx >= 0 && dx < p.rs.new_w && dy >= 0 && dy < p.rs.new_h) resize_pixel(p.rs, dx, dy, v);
  if (p.chw) {
    const size_t plane = static_cast<size_t>(p.out_h) * p.out_w, at = static_cast<size_t>(y) * p.out_w + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) p.dst[(p.swap_rb ? 2 - c : c) * plane + at] = static_cast<uint8_t>(v[c]);
  } else {
    uint8_t* o = p.dst + (static_cast<size_t>(y) * p.out_w + x) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[p.swap_rb ? 2 - c : c] = static_cast<uint8_t>(v[c]);
  }
}

}  // namespace
}  // namespace y3

extern "C" int y3_letterbox_u8(const y3_letterbox_desc* d, y3_stream_t stream) {
  Y3_REQUIRE(d && d->src && d->dst, "letterbox: null pointer");
  Y3_REQUIRE(d->src_h > 0 && d->src_w > 0 && d->src_pitch >= 3 * d->src_w && d->new_h > 0 && d->new_w > 0, "letterbox: bad source / resize shape");
  Y3_REQUIRE(d->top >= 0 && d->left >= 0 && d->out_h >= d->top + d->new_h && d->out_w >= d->left + d->new_w, "letterbox: the resized image must fit the output");
  y3::LbArgs a;
  a.rs.src = static_cast<const uint8_t*>(d->src);
  a.rs.src_h = d->src_h;
  a.rs.src_w = d->src_w;
  a.rs.src_pitch = d->src_pitch;
  a.rs.new_h = d->new_h;
  a.rs.new_w = d->new_w;
  y3::resize_setup(a.rs);
  a.top = d->top;
  a.left = d->left;
  a.out_h = d->out_h;
  a.out_w = d->out_w;
  for (int c = 0; c < 3; ++c) a.pad[c] = d->pad[c];
  a.dst = static_cast<uint8_t*>(d->dst);
  a.chw = d->out_chw ? 1 : 0;
  a.swap_rb = d->swap_rb ? 1 : 0;
  y3::letterbox_kernel<<<dim3((d->out_w + 255) / 256, d->out_h), 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
