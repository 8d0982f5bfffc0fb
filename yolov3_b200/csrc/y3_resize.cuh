// yolov3_b200 — OpenCV's 8-bit INTER_LINEAR resize (third-party, opencv-python 4.13; resize.cpp) restated bit for bit, shared
// by the letterbox kernels and the batched resize of the loaders (y3_augment.cu): 11-bit fixed-point coefficients from float
// fractions, horizontal pass to int, vertical pass ((b0*(S0>>4))>>16 + (b1*(S1>>4))>>16 + 2) >> 2; an exact 2x shrink takes
// INTER_AREA's 2x2 average like cv::resize does, and an equal size is a plain copy.  The letterbox pixel (border, resize,
// HWC / CHW store) and INTER_AREA for scales >= 1 (the validation loader's load_image shrink) follow.
// Include only from sources compiled without fast-math / FMA contraction (build.py EXACT_SOURCES).
#pragma once

#include <math.h>
#include <stdint.h>

#include "../../include/yolov3_b200.h"

namespace y3 {

struct ResizeGeom {
  const uint8_t* src;  // [src_h, src_w, 3] bytes, row pitch src_pitch
  int src_h, src_w, src_pitch;
  int new_h, new_w;          // size after the resize
  double scale_x, scale_y;   // src / dst, as cv::resize computes them (1 / (dsize / ssize))
  int mode;                  // 0: copy (no resize), 1: bilinear, 2: 2x2 area average, 3: kx x ky block mean, 4: area
  int kx, ky;                // the integer factors of mode 3
};

// the source and the output size of a resize; resize_setup / area_setup derive the rest
__device__ __forceinline__ ResizeGeom resize_geom(const void* src, int src_h, int src_w, int src_pitch, int new_h, int new_w) {
  ResizeGeom g;
  g.src = static_cast<const uint8_t*>(src);
  g.src_h = src_h;
  g.src_w = src_w;
  g.src_pitch = src_pitch;
  g.new_h = new_h;
  g.new_w = new_w;
  return g;
}

// scale and mode of a resize from the sizes (the scalar part of cv::resize)
__host__ __device__ inline void resize_setup(ResizeGeom& g) {
  g.scale_x = 1.0 / (static_cast<double>(g.new_w) / g.src_w);
  g.scale_y = 1.0 / (static_cast<double>(g.new_h) / g.src_h);
  g.mode = 1;
  if (g.new_h == g.src_h && g.new_w == g.src_w) {
    g.mode = 0;
  } else {
    const long long isx = llrint(g.scale_x), isy = llrint(g.scale_y);
    const double eps = 2.220446049250313e-16;
    if (isx == 2 && isy == 2 && fabs(g.scale_x - isx) < eps && fabs(g.scale_y - isy) < eps) g.mode = 2;
  }
}

__device__ __forceinline__ void resize_coef(int d, double scale, int sn, bool clamp_frac, int& s0, int& a0, int& a1) {
  float f = static_cast<float>((d + 0.5) * scale - 0.5);
  int s = static_cast<int>(floorf(f));
  f = __fsub_rn(f, static_cast<float>(s));
  if (clamp_frac) {  // horizontal: cv::resize zeroes the fraction when it clamps the column; rows are clamped at fetch time only
    if (s < 0) {
      f = 0.f;
      s = 0;
    }
    if (s >= sn - 1) {
      f = 0.f;
      s = sn - 1;
    }
  }
  s0 = s;
  a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, f), 2048.0f));
  a1 = __float2int_rn(__fmul_rn(f, 2048.0f));
}

// pixel (dx, dy) of the resized image, in source channel order
__device__ __forceinline__ void resize_pixel(const ResizeGeom& p, int dx, int dy, int (&v)[3]) {
  if (p.mode == 0) {
    const uint8_t* q = p.src + static_cast<size_t>(dy) * p.src_pitch + dx * 3;
    v[0] = q[0];
    v[1] = q[1];
    v[2] = q[2];
  } else if (p.mode == 2) {
    const uint8_t* q0 = p.src + static_cast<size_t>(2 * dy) * p.src_pitch + 2 * dx * 3;
    const uint8_t* q1 = q0 + p.src_pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = (q0[c] + q0[3 + c] + q1[c] + q1[3 + c] + 2) >> 2;
  } else {
    int sx, ax0, ax1, sy, b0, b1;
    resize_coef(dx, p.scale_x, p.src_w, true, sx, ax0, ax1);
    resize_coef(dy, p.scale_y, p.src_h, false, sy, b0, b1);
    const int sx1 = min(sx + 1, p.src_w - 1);
    const int r0 = min(max(sy, 0), p.src_h - 1), r1 = min(max(sy + 1, 0), p.src_h - 1);
    const uint8_t* q0 = p.src + static_cast<size_t>(r0) * p.src_pitch;
    const uint8_t* q1 = p.src + static_cast<size_t>(r1) * p.src_pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int s0 = q0[sx * 3 + c] * ax0 + q0[sx1 * 3 + c] * ax1;
      const int s1 = q1[sx * 3 + c] * ax0 + q1[sx1 * 3 + c] * ax1;
      v[c] = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
    }
  }
}

// output pixel (x, y) of the letterbox d: pad[] outside the resized image, its INTER_LINEAR pixel inside; stored HWC or CHW,
// the channels reversed when swap_rb
__device__ __forceinline__ void letterbox_pixel(const y3_letterbox_desc& d, int x, int y) {
  int v[3] = {d.pad[0], d.pad[1], d.pad[2]};
  const int dx = x - d.left, dy = y - d.top;
  if (dx >= 0 && dx < d.new_w && dy >= 0 && dy < d.new_h) {
    ResizeGeom g = resize_geom(d.src, d.src_h, d.src_w, d.src_pitch, d.new_h, d.new_w);
    resize_setup(g);
    resize_pixel(g, dx, dy, v);
  }
  uint8_t* dst = static_cast<uint8_t*>(d.dst);
  const size_t at = static_cast<size_t>(y) * d.out_w + x;
  if (d.out_chw) {
    const size_t plane = static_cast<size_t>(d.out_h) * d.out_w;
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[(d.swap_rb ? 2 - c : c) * plane + at] = static_cast<uint8_t>(v[c]);
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[at * 3 + (d.swap_rb ? 2 - c : c)] = static_cast<uint8_t>(v[c]);
  }
}

// ------------------------------------------------------------------------------------------------------------ INTER_AREA
// cv::resize(..., INTER_AREA) for 8-bit, 3-channel images and scales >= 1 in both axes (resizeAreaFast_ / resizeArea_):
//  * an integer factor (kx, ky) in both axes: (2, 2) is the (a+b+c+d+2)>>2 of mode 2; any other is the integer block sum
//    times the float 1 / (kx ky), rounded half-even (mode 3);
//  * any other scale (mode 4): per axis the spans of computeResizeAreaTab, built in double with float alphas; per source
//    row of the y-span, buf = sum of S alpha over the x-span (float, in table order), then sum = beta buf, sum += beta buf;
//    the output is sum rounded half-even, saturated.
__host__ __device__ inline void area_setup(ResizeGeom& g) {
  g.scale_x = 1.0 / (static_cast<double>(g.new_w) / g.src_w);
  g.scale_y = 1.0 / (static_cast<double>(g.new_h) / g.src_h);
  g.kx = g.ky = 0;
  if (g.new_h == g.src_h && g.new_w == g.src_w) {
    g.mode = 0;
    return;
  }
  const long long isx = llrint(g.scale_x), isy = llrint(g.scale_y);
  const double eps = 2.220446049250313e-16;
  if (fabs(g.scale_x - isx) < eps && fabs(g.scale_y - isy) < eps) {
    g.mode = isx == 2 && isy == 2 ? 2 : 3;
    g.kx = static_cast<int>(isx);
    g.ky = static_cast<int>(isy);
  } else {
    g.mode = 4;
  }
}

// the entries of computeResizeAreaTab for one destination index: an optional leading partial source index (s1 - 1), the
// full indices [s1, s2) and an optional trailing partial index s2
struct AreaSpan {
  int s1, s2;
  bool lead, trail;
  float a_lead, a_full, a_trail;
};

__device__ __forceinline__ AreaSpan area_span(int d, double scale, int ssize) {
  AreaSpan sp;
  const double fs1 = d * scale, fs2 = fs1 + scale;
  const double rest = ssize - fs1;
  const double cell = rest < scale ? rest : scale;  // std::min(scale, ssize - fsx1)
  int s1 = static_cast<int>(ceil(fs1));
  int s2 = static_cast<int>(floor(fs2));
  s2 = min(s2, ssize - 1);
  s1 = min(s1, s2);
  sp.s1 = s1;
  sp.s2 = s2;
  sp.lead = s1 - fs1 > 1e-3;
  sp.a_lead = static_cast<float>((s1 - fs1) / cell);
  sp.a_full = static_cast<float>(1.0 / cell);
  sp.trail = fs2 - s2 > 1e-3;
  const double t = fs2 - s2 < 1.0 ? fs2 - s2 : 1.0;
  sp.a_trail = static_cast<float>((cell < t ? cell : t) / cell);
  return sp;
}

__device__ __forceinline__ void area_row(const uint8_t* row, const AreaSpan& x, float (&buf)[3]) {
  buf[0] = buf[1] = buf[2] = 0.f;
  const auto tap = [&](int sx, float a) {
#pragma unroll
    for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn(static_cast<float>(row[sx * 3 + c]), a));
  };
  if (x.lead) tap(x.s1 - 1, x.a_lead);
  for (int sx = x.s1; sx < x.s2; ++sx) tap(sx, x.a_full);
  if (x.trail) tap(x.s2, x.a_trail);
}

// pixel (dx, dy) of the INTER_AREA-resized image (area_setup), in source channel order
__device__ __forceinline__ void area_pixel(const ResizeGeom& p, int dx, int dy, int (&v)[3]) {
  if (p.mode == 3) {
    const uint8_t* q = p.src + static_cast<size_t>(dy) * p.ky * p.src_pitch + static_cast<size_t>(dx) * p.kx * 3;
    int s[3] = {0, 0, 0};
    for (int r = 0; r < p.ky; ++r, q += p.src_pitch)
      for (int k = 0; k < p.kx; ++k) {
#pragma unroll
        for (int c = 0; c < 3; ++c) s[c] += q[k * 3 + c];
      }
    const float inv = __fdiv_rn(1.f, static_cast<float>(p.kx * p.ky));
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = min(max(__float2int_rn(__fmul_rn(static_cast<float>(s[c]), inv)), 0), 255);
    return;
  }
  if (p.mode != 4) {
    resize_pixel(p, dx, dy, v);  // copy, 2x2
    return;
  }
  const AreaSpan x = area_span(dx, p.scale_x, p.src_w), y = area_span(dy, p.scale_y, p.src_h);
  float sum[3] = {0.f, 0.f, 0.f}, buf[3];
  const auto row = [&](int sy, float beta) {
    area_row(p.src + static_cast<size_t>(sy) * p.src_pitch, x, buf);
#pragma unroll
    for (int c = 0; c < 3; ++c) sum[c] = __fadd_rn(sum[c], __fmul_rn(beta, buf[c]));
  };
  if (y.lead) row(y.s1 - 1, y.a_lead);
  for (int sy = y.s1; sy < y.s2; ++sy) row(sy, y.a_full);
  if (y.trail) row(y.s2, y.a_trail);
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = min(max(__float2int_rn(sum[c]), 0), 255);
}

}  // namespace y3
