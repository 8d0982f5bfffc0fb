// yolov3_b200 — OpenCV's 8-bit INTER_LINEAR resize (third-party, opencv-python 4.13; resize.cpp) restated bit for bit, shared
// by the letterbox kernel (y3_pre.cu) and the batched resize of the training loader (y3_augment.cu): 11-bit fixed-point
// coefficients from float fractions, horizontal pass to int, vertical pass ((b0*(S0>>4))>>16 + (b1*(S1>>4))>>16 + 2) >> 2; an
// exact 2x shrink takes INTER_AREA's 2x2 average like cv::resize does, and an equal size is a plain copy.
// Include only from sources compiled without fast-math / FMA contraction (build.py EXACT_SOURCES).
#pragma once

#include <math.h>
#include <stdint.h>

namespace y3 {

struct ResizeGeom {
  const uint8_t* src;  // [src_h, src_w, 3] bytes, row pitch src_pitch
  int src_h, src_w, src_pitch;
  int new_h, new_w;          // size after the resize
  double scale_x, scale_y;   // src / dst, as cv::resize computes them (1 / (dsize / ssize))
  int mode;                  // 0: copy (no resize), 1: bilinear, 2: 2x2 area average
};

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

}  // namespace y3
