// yolov3_b200 — the training augmentation of LoadImagesAndLabels on the device (SURVEY §8(f)).  Replaces the image arithmetic of
//   load_image's cv2.resize                   utils/dataloaders.py:737-756   -> y3_resize_u8_batched (every source of a batch)
//   load_mosaic's img4 / letterbox's border   utils/dataloaders.py:764-822, utils/augmentations.py:104-134
//   random_perspective's cv2.warpAffine       utils/augmentations.py:137-216
//   mixup                                     utils/augmentations.py:270-275
//   augment_hsv                               utils/augmentations.py:57-73
//   flipud / fliplr, HWC->CHW, BGR->RGB       utils/dataloaders.py:711-733   -> y3_augment_u8 (one launch per batch)
//   collate_fn4's 2x2 tiles / 2x upsample     utils/dataloaders.py:833-858   -> y3_augment_u8 writing each item into its
//                                                                              quadrant, y3_upsample2x_u8 (train.py --quad)
// The mosaic canvas is virtual: every warp tap looks its pixel up in the item's placement table (114 where no source is placed),
// so the 2s x 2s img4 is never written.  The random draws, the geometry and the labels stay on the host (yolov3_b200/augment.py).
// The validation loader (augment=False) uses y3_resize_area_u8_batched (load_image's INTER_AREA shrink) and
// y3_letterbox_u8_batched (letterbox without a warp, straight into the CHW RGB batch).  y3_letterbox_u8 is the same letterbox
// for one image (preprocess.py: detect.py's letterbox(im0) and transpose((2, 0, 1))[::-1], HWC BGR or CHW RGB out).
//
// OpenCV's 8-bit rules restated bit for bit (opencv-python 4.13; pinned against cv2 by tests/test_augment_cpu.py):
//  * warpAffine INTER_LINEAR: coordinates (A11 x) 1024 per column and (A12 y + b1) 1024 per row, each rounded half-even in
//    double, + 16, >> 5; source pixel = >> 5, fraction index (Y & 31) 32 + (X & 31); 16-bit weights (units of 2^15) from float
//    products of the k/32 fractions, which are exact, so the four always sum to 2^15; (sum + 2^14) >> 15.
//  * BGR2HSV: max / min, the 12-bit division tables sdiv = rint((255 << 12) / i), hdiv = rint((180 << 12) / (6 i)).
//  * HSV2BGR: float32, q = v fma(-s, f, 1), t = v fma(-s, 1 - f, 1), truncation of x * 255.
// Compiled without fast-math / FMA contraction (build.py EXACT_SOURCES); the two fused multiply-adds OpenCV's compiler makes are
// written as __fmaf_rn.
#include "y3_common.cuh"
#include "y3_internal.h"
#include "y3_resize.cuh"

namespace y3 {
namespace {

constexpr int kAugThreads = 256;
constexpr int kAugRows = 4;  // output rows per block: the shared weight table and descriptor are set up once per 1024 pixels

__global__ void __launch_bounds__(256) resize_batched_kernel(const y3_resize_item* __restrict__ items) {
  pdl_entry();
  const y3_resize_item it = items[blockIdx.z];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= it.dst_w || y >= it.dst_h) return;
  ResizeGeom g = resize_geom(it.src, it.src_h, it.src_w, it.src_pitch, it.dst_h, it.dst_w);
  resize_setup(g);
  int v[3];
  resize_pixel(g, x, y, v);
  uint8_t* o = static_cast<uint8_t*>(it.dst) + static_cast<size_t>(y) * it.dst_pitch + x * 3;
  o[0] = static_cast<uint8_t>(v[0]);
  o[1] = static_cast<uint8_t>(v[1]);
  o[2] = static_cast<uint8_t>(v[2]);
}

// load_image's cv2.resize(..., INTER_AREA) of the validation loader: one thread per output pixel, which recomputes the two
// short area tables of its row and column (y3_resize.cuh area_pixel)
__global__ void __launch_bounds__(256) resize_area_batched_kernel(const y3_resize_item* __restrict__ items) {
  pdl_entry();
  const y3_resize_item it = items[blockIdx.z];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= it.dst_w || y >= it.dst_h) return;
  ResizeGeom g = resize_geom(it.src, it.src_h, it.src_w, it.src_pitch, it.dst_h, it.dst_w);
  area_setup(g);
  int v[3];
  area_pixel(g, x, y, v);
  uint8_t* o = static_cast<uint8_t*>(it.dst) + static_cast<size_t>(y) * it.dst_pitch + x * 3;
  o[0] = static_cast<uint8_t>(v[0]);
  o[1] = static_cast<uint8_t>(v[1]);
  o[2] = static_cast<uint8_t>(v[2]);
}

// letterbox without a warp: letterbox's INTER_LINEAR resize, the border and the store, for one image (y3_letterbox_u8) ...
__global__ void __launch_bounds__(256) letterbox_kernel(const y3_letterbox_desc d) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x < d.out_w) letterbox_pixel(d, x, blockIdx.y);
}

// ... and for a whole batch (the validation loader: the 114 border and the CHW RGB store of __getitem__ with augment=False)
__global__ void __launch_bounds__(256) letterbox_batched_kernel(const y3_letterbox_desc* __restrict__ descs) {
  pdl_entry();
  const y3_letterbox_desc d = descs[blockIdx.z];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x < d.out_w && y < d.out_h) letterbox_pixel(d, x, y);
}

// one canvas pixel: a placed source pixel, else the 114 of img4 / the letterbox border / warpAffine's borderValue
__device__ __forceinline__ void canvas_px(const y3_aug_canvas& cv, int X, int Y, int (&t)[3]) {
  for (int k = 0; k < cv.n_place; ++k) {
    const y3_aug_place& p = cv.place[k];
    if (X >= p.x0 && X < p.x1 && Y >= p.y0 && Y < p.y1) {
      const uint8_t* q = static_cast<const uint8_t*>(p.src) + static_cast<size_t>(Y - p.off_y) * p.pitch + (X - p.off_x) * 3;
      t[0] = q[0];
      t[1] = q[1];
      t[2] = q[2];
      return;
    }
  }
  t[0] = t[1] = t[2] = 114;
}

// cv2.warpAffine(canvas, M, INTER_LINEAR, BORDER_CONSTANT 114) at output pixel (x, y)
__device__ __forceinline__ void warp_px(const y3_aug_canvas& cv, const ushort4* wtab, int x, int y, int (&v)[3]) {
  const double* m = cv.inv;
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], static_cast<double>(y)), m[2]), 1024.0)) + 16;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], static_cast<double>(y)), m[5]), 1024.0)) + 16;
  const int X = (X0 + __double2int_rn(__dmul_rn(__dmul_rn(m[0], static_cast<double>(x)), 1024.0))) >> 5;
  const int Y = (Y0 + __double2int_rn(__dmul_rn(__dmul_rn(m[3], static_cast<double>(x)), 1024.0))) >> 5;
  const int sx = X >> 5, sy = Y >> 5;
  const ushort4 w = wtab[(Y & 31) * 32 + (X & 31)];
  int t00[3], t01[3], t10[3], t11[3];
  canvas_px(cv, sx, sy, t00);
  canvas_px(cv, sx + 1, sy, t01);
  canvas_px(cv, sx, sy + 1, t10);
  canvas_px(cv, sx + 1, sy + 1, t11);
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = (t00[c] * w.x + t01[c] * w.y + t10[c] * w.z + t11[c] * w.w + (1 << 14)) >> 15;
}

__device__ __forceinline__ int div_table(int num, int i) {  // rint(num / i), 0 at i == 0 (OpenCV's sdiv_table / hdiv_table)
  return i == 0 ? 0 : __double2int_rn(__ddiv_rn(static_cast<double>(num), static_cast<double>(i)));
}

__host__ __device__ constexpr unsigned long long sector_code(int b, int g, int r) {
  return static_cast<unsigned long long>(b | g << 2 | r << 4);
}

// cv2.COLOR_BGR2HSV (8U, hrange 180), the LUTs of augment_hsv, cv2.COLOR_HSV2BGR (8U) — in place on a BGR pixel
__device__ __forceinline__ void hsv_px(const uint8_t (*lut)[256], const int* sdiv, const int* hdiv, int (&v)[3]) {
  const int b = v[0], g = v[1], r = v[2];
  const int vmax = max(max(b, g), r), diff = vmax - min(min(b, g), r);
  const int s = (diff * sdiv[vmax] + 2048) >> 12;
  int h = vmax == r ? g - b : (vmax == g ? b - r + 2 * diff : r - g + 4 * diff);
  h = (h * hdiv[diff] + 2048) >> 12;
  h += h < 0 ? 180 : 0;
  const int H = lut[0][h], S = lut[1][s], V = lut[2][vmax];
  const float vf = __fmul_rn(static_cast<float>(V), 1.f / 255.f);
  float ob = vf, og = vf, orr = vf;
  if (S != 0) {
    const float sf = __fmul_rn(static_cast<float>(S), 1.f / 255.f);
    const float hh = __fmul_rn(static_cast<float>(H), 6.f / 180.f);
    const float sector = floorf(hh);
    const float f = __fsub_rn(hh, sector);
    const float p = __fmul_rn(vf, __fsub_rn(1.f, sf));
    const float q = __fmul_rn(vf, __fmaf_rn(-sf, f, 1.f));
    const float t = __fmul_rn(vf, __fmaf_rn(-sf, __fsub_rn(1.f, f), 1.f));
    const auto tab = [&](unsigned i) { return i == 0 ? vf : (i == 1 ? p : (i == 2 ? q : t)); };  // (v, p, q, t)
    // sector table {1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0}: indices into tab for b, g, r
    constexpr unsigned long long kSec = sector_code(1, 3, 0) | sector_code(1, 0, 2) << 6 | sector_code(3, 0, 1) << 12 |
                                        sector_code(0, 2, 1) << 18 | sector_code(0, 1, 3) << 24 | sector_code(2, 1, 0) << 30;
    const unsigned code = static_cast<unsigned>(kSec >> (6 * static_cast<int>(sector))) & 63u;
    ob = tab(code & 3);
    og = tab((code >> 2) & 3);
    orr = tab((code >> 4) & 3);
  }
  v[0] = static_cast<int>(__fmul_rn(ob, 255.f));
  v[1] = static_cast<int>(__fmul_rn(og, 255.f));
  v[2] = static_cast<int>(__fmul_rn(orr, 255.f));
}

__global__ void __launch_bounds__(kAugThreads) augment_kernel(const y3_augment_desc* __restrict__ descs, int out_h, int out_w,
                                                              uint8_t* __restrict__ out) {
  __shared__ y3_augment_desc sd;
  __shared__ ushort4 wtab[1024];  // unsigned: the weight of a zero fraction is 32768
  __shared__ int sdiv[256], hdiv[256];
  pdl_entry();
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(descs + blockIdx.z);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sd);
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(y3_augment_desc) / 4); i += kAugThreads) dst[i] = src[i];
  }
  for (int i = threadIdx.x; i < 1024; i += kAugThreads) {  // OpenCV's initInterTab2D for INTER_LINEAR, float products
    const float fy = __fmul_rn(1.f / 32.f, static_cast<float>(i >> 5)), fx = __fmul_rn(1.f / 32.f, static_cast<float>(i & 31));
    const float cy0 = __fsub_rn(1.f, fy), cx0 = __fsub_rn(1.f, fx);
    wtab[i] = make_ushort4(static_cast<unsigned short>(__float2int_rn(__fmul_rn(__fmul_rn(cy0, cx0), 32768.f))),
                           static_cast<unsigned short>(__float2int_rn(__fmul_rn(__fmul_rn(cy0, fx), 32768.f))),
                           static_cast<unsigned short>(__float2int_rn(__fmul_rn(__fmul_rn(fy, cx0), 32768.f))),
                           static_cast<unsigned short>(__float2int_rn(__fmul_rn(__fmul_rn(fy, fx), 32768.f))));
  }
  for (int i = threadIdx.x; i < 256; i += kAugThreads) {
    sdiv[i] = div_table(255 << 12, i);
    hdiv[i] = div_table(180 << 12, 6 * i);
  }
  __syncthreads();
  const int ox = blockIdx.x * kAugThreads + threadIdx.x;
  if (ox >= out_w) return;
  size_t plane = static_cast<size_t>(out_h) * out_w, pitch = out_w;
  uint8_t* img = out + static_cast<size_t>(blockIdx.z) * 3 * plane;
  if (sd.dst) {  // a quadrant of a 2x2 tile or a scratch image (collate_fn4)
    img = static_cast<uint8_t*>(sd.dst);
    plane = static_cast<size_t>(sd.dst_plane);
    pitch = static_cast<size_t>(sd.dst_pitch);
  }
  const int x = sd.fliplr ? out_w - 1 - ox : ox;
  for (int oy = blockIdx.y * kAugRows; oy < min(out_h, (blockIdx.y + 1) * kAugRows); ++oy) {
    const int y = sd.flipud ? out_h - 1 - oy : oy;
    int v[3];
    warp_px(sd.canvas[0], wtab, x, y, v);
    if (sd.mixup) {  // (im * r + im2 * (1 - r)).astype(np.uint8), float64
      int v2[3];
      warp_px(sd.canvas[1], wtab, x, y, v2);
      const double r = sd.mix_r, r1 = __dsub_rn(1.0, r);
#pragma unroll
      for (int c = 0; c < 3; ++c)
        v[c] = static_cast<int>(__dadd_rn(__dmul_rn(static_cast<double>(v[c]), r), __dmul_rn(static_cast<double>(v2[c]), r1)));
    }
    if (sd.hsv) hsv_px(sd.lut, sdiv, hdiv, v);
    const size_t at = static_cast<size_t>(oy) * pitch + ox;
    img[at] = static_cast<uint8_t>(v[2]);  // RGB planes
    img[plane + at] = static_cast<uint8_t>(v[1]);
    img[2 * plane + at] = static_cast<uint8_t>(v[0]);
  }
}

// collate_fn4's 2x bilinear upsample (align_corners=False) in integer form: one thread per source pixel of one plane writes
// the 2x2 output block it is the nearest source of.  Every tap weight is a quarter per axis, so F.interpolate's float sum is
// exact and its truncation to uint8 is (sum of 16ths) >> 4.
__global__ void __launch_bounds__(256) upsample2x_kernel(const uint8_t* __restrict__ src, const int32_t* __restrict__ dst_index,
                                                         int h, int w, uint8_t* __restrict__ out) {
  pdl_entry();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const int k = blockIdx.z / 3, c = blockIdx.z % 3;
  const size_t plane = static_cast<size_t>(h) * w;
  const uint8_t* s = src + (static_cast<size_t>(k) * 3 + c) * plane;
  const int xm = max(x - 1, 0), xp = min(x + 1, w - 1);
  int l[3], r[3];  // rows y-1, y, y+1 (clamped): 4x the horizontal interpolation at output columns 2x and 2x+1
  for (int j = 0; j < 3; ++j) {
    const uint8_t* p = s + static_cast<size_t>(min(max(y - 1 + j, 0), h - 1)) * w;
    const int m = p[x];
    l[j] = p[xm] + 3 * m;
    r[j] = 3 * m + p[xp];
  }
  uint8_t* o = out + (static_cast<size_t>(dst_index[k]) * 3 + c) * 4 * plane + static_cast<size_t>(2 * y) * (2 * w) + 2 * x;
  *reinterpret_cast<uchar2*>(o) = make_uchar2(static_cast<uint8_t>((l[0] + 3 * l[1]) >> 4),
                                              static_cast<uint8_t>((r[0] + 3 * r[1]) >> 4));
  *reinterpret_cast<uchar2*>(o + 2 * w) = make_uchar2(static_cast<uint8_t>((3 * l[1] + l[2]) >> 4),
                                                      static_cast<uint8_t>((3 * r[1] + r[2]) >> 4));
}

}  // namespace
}  // namespace y3

namespace y3 {
namespace {

// what every resize entry point requires of an item
int check_resize_item(const y3_resize_item& it, const char* who, int i) {
  Y3_REQUIRE(it.src && it.dst && it.src_h > 0 && it.src_w > 0 && it.dst_h > 0 && it.dst_w > 0 &&
                 it.src_pitch >= 3 * it.src_w && it.dst_pitch >= 3 * it.dst_w,
             "%s: item %d: bad shape or pointer", who, i);
  return Y3_OK;
}

// what every letterbox entry point requires of a descriptor
int check_letterbox_desc(const y3_letterbox_desc& d, const char* who, int i) {
  Y3_REQUIRE(d.src && d.dst && d.src_h > 0 && d.src_w > 0 && d.src_pitch >= 3 * d.src_w && d.new_h > 0 && d.new_w > 0,
             "%s: item %d: bad source / resize shape or null pointer", who, i);
  Y3_REQUIRE(d.top >= 0 && d.left >= 0 && d.out_h >= d.top + d.new_h && d.out_w >= d.left + d.new_w,
             "%s: item %d: the resized image must fit the output", who, i);
  return Y3_OK;
}

// one launch of a batched resize kernel over `items` (device), validated and sized from `host_items`; `shrink_only` refuses
// an item that scales up (INTER_AREA is built for scales >= 1 only)
int launch_resize(void (*kern)(const y3_resize_item*), const char* who, bool shrink_only, const y3_resize_item* items,
                  const y3_resize_item* host_items, int32_t n_items, y3_stream_t stream) {
  Y3_REQUIRE(items && host_items && n_items > 0 && n_items <= 65535, "%s: bad arguments (n_items %d)", who, n_items);
  int max_h = 0, max_w = 0;
  for (int i = 0; i < n_items; ++i) {
    const y3_resize_item& it = host_items[i];
    if (const int rc = check_resize_item(it, who, i)) return rc;
    Y3_REQUIRE(!shrink_only || (it.dst_h <= it.src_h && it.dst_w <= it.src_w),
               "%s: item %d: %dx%d -> %dx%d scales up; INTER_AREA is built for scales >= 1 only", who, i, it.src_h,
               it.src_w, it.dst_h, it.dst_w);
    max_h = max(max_h, it.dst_h);
    max_w = max(max_w, it.dst_w);
  }
  Y3_REQUIRE(max_h <= 65535, "%s: output too tall (%d rows)", who, max_h);
  Y3_CHECK_CUDA(launch_pdl(kern, dim3((max_w + 255) / 256, max_h, n_items), dim3(256), 0, static_cast<cudaStream_t>(stream),
                           items));
  return Y3_OK;
}

}  // namespace
}  // namespace y3

extern "C" int y3_resize_u8_batched(const y3_resize_item* items, const y3_resize_item* host_items, int32_t n_items,
                                    y3_stream_t stream) {
  return y3::launch_resize(y3::resize_batched_kernel, "resize", false, items, host_items, n_items, stream);
}

extern "C" int y3_resize_area_u8_batched(const y3_resize_item* items, const y3_resize_item* host_items, int32_t n_items,
                                         y3_stream_t stream) {
  return y3::launch_resize(y3::resize_area_batched_kernel, "resize_area", true, items, host_items, n_items, stream);
}

extern "C" int y3_letterbox_u8(const y3_letterbox_desc* d, y3_stream_t stream) {
  Y3_REQUIRE(d, "letterbox: null descriptor");
  if (const int rc = y3::check_letterbox_desc(*d, "letterbox", 0)) return rc;
  y3::letterbox_kernel<<<dim3((d->out_w + 255) / 256, d->out_h), 256, 0, static_cast<cudaStream_t>(stream)>>>(*d);
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_letterbox_u8_batched(const y3_letterbox_desc* descs, const y3_letterbox_desc* host_descs, int32_t n,
                                       y3_stream_t stream) {
  Y3_REQUIRE(descs && host_descs && n > 0 && n <= 65535, "letterbox_batched: bad arguments (n %d)", n);
  int max_h = 0, max_w = 0;
  for (int i = 0; i < n; ++i) {
    if (const int rc = y3::check_letterbox_desc(host_descs[i], "letterbox_batched", i)) return rc;
    max_h = max(max_h, host_descs[i].out_h);
    max_w = max(max_w, host_descs[i].out_w);
  }
  Y3_REQUIRE(max_h <= 65535, "letterbox_batched: output too tall (%d rows)", max_h);
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::letterbox_batched_kernel, dim3((max_w + 255) / 256, max_h, n), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), descs));
  return Y3_OK;
}

extern "C" int y3_augment_u8(const y3_augment_desc* descs, int32_t n, int32_t out_h, int32_t out_w, void* out,
                             y3_stream_t stream) {
  Y3_REQUIRE(descs && out && n > 0 && n <= 65535 && out_h > 0 && out_w > 0, "augment: bad arguments (n %d, %dx%d)", n, out_h,
             out_w);
  Y3_REQUIRE((reinterpret_cast<uintptr_t>(descs) & 7) == 0, "augment: descriptors must be 8-byte aligned");
  const int gy = (out_h + y3::kAugRows - 1) / y3::kAugRows;
  Y3_REQUIRE(gy <= 65535, "augment: output too tall (%d rows)", out_h);
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::augment_kernel, dim3((out_w + y3::kAugThreads - 1) / y3::kAugThreads, gy, n),
                                 dim3(y3::kAugThreads), 0, static_cast<cudaStream_t>(stream), descs, out_h, out_w,
                                 static_cast<uint8_t*>(out)));
  return Y3_OK;
}

extern "C" int y3_upsample2x_u8(const void* src, const int32_t* dst_index, int32_t n, int32_t h, int32_t w, void* out,
                                y3_stream_t stream) {
  Y3_REQUIRE(src && dst_index && out && n > 0 && 3 * n <= 65535 && h > 0 && w > 0 && h <= 65535,
             "upsample2x: bad arguments (n %d, %dx%d)", n, h, w);
  Y3_REQUIRE((reinterpret_cast<uintptr_t>(out) & 1) == 0, "upsample2x: out must be 2-byte aligned");
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::upsample2x_kernel, dim3((w + 255) / 256, h, 3 * n), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), static_cast<const uint8_t*>(src), dst_index, h, w,
                                 static_cast<uint8_t*>(out)));
  return Y3_OK;
}
