// yolov3_b200 — Detect-head decode: sigmoid + anchor-grid transform of all pyramid levels in ONE coalesced pass.
// Replaces Detect.forward's eval branch and _make_grid (reference models/yolo.py:100-123): no grid / anchor_grid
// tensors, no split/cat; grid offsets come from the element index.  raw level l is fp32 [bs, na, ny, nx, no]
// (= the reference's x[i]); z is fp32 [bs, sum_l na*ny*nx, no] with row = off_l + (a*ny + y)*nx + x, i.e. exactly
// torch.cat(z, 1) of models/yolo.py:110.  Compiled without fast-math/FMA contraction: (2*s + g) * stride is evaluated
// with the reference's operation order and rounding.
#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {
namespace {

struct DecodeArgs {
  const float* raw[Y3_MAX_LEVELS];
  int ny[Y3_MAX_LEVELS], nx[Y3_MAX_LEVELS];
  int row_off[Y3_MAX_LEVELS + 1];  // first z row of each level; [nl] = total rows
  float stride[Y3_MAX_LEVELS];
  float anchor_w[Y3_MAX_LEVELS][Y3_MAX_ANCHORS], anchor_h[Y3_MAX_LEVELS][Y3_MAX_ANCHORS];  // pixels
  int nl, bs, na, no;
  float* z;
};

__global__ void __launch_bounds__(256) decode_kernel(const DecodeArgs p) {
  pdl_entry();
  const long long per_img = static_cast<long long>(p.row_off[p.nl]) * p.no;
  const long long total = per_img * p.bs;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / per_img);
    const long long e = i - b * per_img;
    const int row = static_cast<int>(e / p.no);
    const int k = static_cast<int>(e - static_cast<long long>(row) * p.no);
    int l = 0;
    while (l + 1 < p.nl && row >= p.row_off[l + 1]) ++l;
    const int r = row - p.row_off[l];
    const int plane = p.ny[l] * p.nx[l];
    const float v = p.raw[l][(static_cast<long long>(b) * p.na * plane + r) * p.no + k];
    const float s = 1.0f / (1.0f + expf(-v));
    float o = s;
    if (k < 4) {
      const int a = r / plane, cell = r - a * plane;
      const int y = cell / p.nx[l], x = cell - y * p.nx[l];
      if (k == 0)
        o = (s * 2.0f + (static_cast<float>(x) - 0.5f)) * p.stride[l];
      else if (k == 1)
        o = (s * 2.0f + (static_cast<float>(y) - 0.5f)) * p.stride[l];
      else {
        const float t = s * 2.0f;
        o = (t * t) * (k == 2 ? p.anchor_w[l][a] : p.anchor_h[l][a]);
      }
    }
    p.z[i] = o;
  }
}

// ---- fused variant used by the graph executor: reads the head convs' fp32 pixel-major output [bs*ny*nx, ld]
// (column a*no + k), writes z AND (optionally) the reference-layout logits raw_l[bs, na, ny, nx, no].
// One warp per (image, cell, anchor): 340-byte contiguous reads and writes.
struct HeadDecodeArgs {
  const float* head[Y3_MAX_LEVELS];
  float* raw[Y3_MAX_LEVELS];
  int head_ld[Y3_MAX_LEVELS];
  int ny[Y3_MAX_LEVELS], nx[Y3_MAX_LEVELS];
  int row_off[Y3_MAX_LEVELS + 1];
  float stride[Y3_MAX_LEVELS];
  float anchor_w[Y3_MAX_LEVELS][Y3_MAX_ANCHORS], anchor_h[Y3_MAX_LEVELS][Y3_MAX_ANCHORS];
  int nl, bs, na, no;
  float* z;
};

constexpr int kDecodeRows = 4;  // consecutive z rows per warp iteration (they are contiguous in z and in the logits)

// sigmoid through the fast exp/divide units: relative error ~1e-6, far inside the 1e-5 decode tolerance (the bit-exact
// requirement applies to NMS on a given z, not to z itself); the IEEE expf/division sequence cost ~1/3 of this kernel.
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

// NITER = ceil(kDecodeRows * no / 128) unrolled iterations of 4 x 32 elements per warp and group of 4 z rows.
// Fast path (the 4 rows share image, level and anchor — always, when ny*nx is a multiple of 4): the rows are consecutive
// cells, so the source of group-local element e = q*no + k is base + q*head_ld + k and its destination is z_base + e:
// both offsets are per-lane constants computed once before the loop; per element the kernel then does one load, one
// sigmoid, one store, and only the 4 box fields of each row take the grid/anchor branch.  The first version recomputed the
// (q, k) split and moved seven shuffle words per element: 96 warp instructions per 32 outputs, issue-bound.
template <int NITER>
__global__ void __launch_bounds__(256, NITER <= 3 ? 3 : 1) head_decode_kernel(const HeadDecodeArgs p) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int rows_per_img = p.row_off[p.nl];
  const int total = rows_per_img * p.bs;  // < 2^31 (checked by the launcher)
  const int groups = (total + kDecodeRows - 1) / kDecodeRows;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int no = p.no;
  const int full_el = kDecodeRows * no;
  uint32_t qk[NITER * 4];  // (q << 16) | k of this lane's elements
  int rel[NITER * 4];      // q * head_ld + k (all levels share head_ld on the fast path)
#pragma unroll
  for (int t = 0; t < NITER * 4; ++t) {
    const int e = (t >> 2) * 128 + (t & 3) * 32 + lane;
    const int q = e / no;
    qk[t] = (static_cast<uint32_t>(q) << 16) | static_cast<uint32_t>(e - q * no);
    rel[t] = q * p.head_ld[0] + (e - q * no);
  }
  bool same_ld = true;
  for (int l = 1; l < p.nl; ++l) same_ld = same_ld && p.head_ld[l] == p.head_ld[0];
  for (int gidx = warp0; gidx < groups; gidx += nwarps) {
    // descriptor of the group's first row (warp-uniform integer work, no shuffles)
    const int w0 = gidx * kDecodeRows;
    const int b0 = w0 / rows_per_img;
    const int row0 = w0 - b0 * rows_per_img;
    int l0 = 0;
    while (l0 + 1 < p.nl && row0 >= p.row_off[l0 + 1]) ++l0;
    const int r0 = row0 - p.row_off[l0];
    const int nx0 = p.nx[l0], plane0 = p.ny[l0] * nx0;
    const int a0 = r0 / plane0, cell0 = r0 - a0 * plane0;
    const long long z_base = static_cast<long long>(gidx) * full_el;  // rows of a group are contiguous in z
    if (same_ld && w0 + kDecodeRows <= total && cell0 + kDecodeRows <= plane0 && row0 + kDecodeRows <= rows_per_img &&
        !p.raw[l0] && p.z) {
      const float* src = p.head[l0] + (static_cast<long long>(b0) * plane0 + cell0) * p.head_ld[l0] + a0 * no;
      float* dst = p.z + z_base;
      const float stride = p.stride[l0], aw = p.anchor_w[l0][a0], ah = p.anchor_h[l0][a0];
      const int y0 = cell0 / nx0, x0 = cell0 - y0 * nx0;
      float v[NITER * 4];
#pragma unroll
      for (int t = 0; t < NITER * 4; ++t) {
        const int e = (t >> 2) * 128 + (t & 3) * 32 + lane;
        v[t] = (e < full_el) ? __ldg(src + rel[t]) : 0.f;
      }
#pragma unroll
      for (int t = 0; t < NITER * 4; ++t) {
        const int e = (t >> 2) * 128 + (t & 3) * 32 + lane;
        if (e >= full_el) continue;
        const int k = qk[t] & 0xFFFF;
        const float s = sigmoid_fast(v[t]);
        float o = s;
        if (k < 4) {
          const float t2 = s * 2.0f;
          if (k < 2) {
            int x = x0 + static_cast<int>(qk[t] >> 16), y = y0;
            if (x >= nx0) {  // the four cells wrap onto the next grid row
              x -= nx0;
              ++y;
            }
            o = (t2 + (static_cast<float>(k == 0 ? x : y) - 0.5f)) * stride;
          } else {
            o = (t2 * t2) * (k == 2 ? aw : ah);
          }
        }
        dst[e] = o;
      }
      continue;
    }
    // ---- general path: rows of different levels / anchors / images in one group, the tail group, raw_out requested
    const int w = w0 + (lane & 3);
    uint32_t d_off = 0, d_pos = 0;
    if (lane < kDecodeRows && w < total) {
      const int b = w / rows_per_img;
      const int row = w - b * rows_per_img;
      int l = 0;
      while (l + 1 < p.nl && row >= p.row_off[l + 1]) ++l;
      const int r = row - p.row_off[l];
      const int plane = p.ny[l] * p.nx[l];
      const int a = r / plane, cell = r - a * plane;
      const int y = cell / p.nx[l], x = cell - y * p.nx[l];
      d_off = static_cast<uint32_t>((b * plane + cell) * p.head_ld[l] + a * no);
      d_pos = static_cast<uint32_t>(x) | (static_cast<uint32_t>(y) << 13) | (static_cast<uint32_t>(a) << 26) |
              (static_cast<uint32_t>(l) << 29);
    }
    const int n_el = min(kDecodeRows, total - w0) * no;
#pragma unroll 1
    for (int t = 0; t < NITER * 4; ++t) {
      const int e = (t >> 2) * 128 + (t & 3) * 32 + lane;
      const int q = e / no, k = e - q * no;
      const uint32_t so = __shfl_sync(0xffffffffu, d_off, q & 3);
      const uint32_t pos = __shfl_sync(0xffffffffu, d_pos, q & 3);
      if (e >= n_el) continue;
      const int l = pos >> 29, a = (pos >> 26) & 7;
      const float x = __ldg(p.head[l] + so + k);
      if (p.raw[l]) {
        // reference-layout logits [bs, na, ny, nx, no]: row (b*na + a)*plane + cell
        const int b = (w0 + q) / rows_per_img;
        const int plane = p.ny[l] * p.nx[l];
        const int cell = ((pos >> 13) & 0x1FFF) * p.nx[l] + (pos & 0x1FFF);
        p.raw[l][((static_cast<long long>(b) * p.na + a) * plane + cell) * no + k] = x;
      }
      if (p.z) {
        const float s = sigmoid_fast(x);
        float o = s;
        if (k < 4) {
          const float t2 = s * 2.0f;
          if (k < 2)
            o = (t2 + (static_cast<float>(k == 0 ? (pos & 0x1FFF) : ((pos >> 13) & 0x1FFF)) - 0.5f)) * p.stride[l];
          else
            o = (t2 * t2) * (k == 2 ? p.anchor_w[l][a] : p.anchor_h[l][a]);
        }
        p.z[z_base + e] = o;
      }
    }
  }
}

}  // namespace
}  // namespace y3

extern "C" int y3_detect_head_decode_fwd(const y3_decode_desc* d, y3_stream_t stream) {
  Y3_REQUIRE(d && d->nl >= 1 && d->nl <= Y3_MAX_LEVELS && d->na >= 1 && d->na <= Y3_MAX_ANCHORS && d->bs > 0 && d->no >= 5,
             "head_decode: bad arguments");
  y3::HeadDecodeArgs a{};
  a.nl = d->nl;
  a.bs = d->bs;
  a.na = d->na;
  a.no = d->no;
  a.z = d->z;
  int off = 0;
  for (int l = 0; l < d->nl; ++l) {
    const y3_detect_level& lv = d->levels[l];
    Y3_REQUIRE(lv.head && lv.ny > 0 && lv.nx > 0 && lv.head_ld >= d->na * d->no, "head_decode: bad level %d", l);
    a.head[l] = lv.head;
    a.head_ld[l] = lv.head_ld;
    a.raw[l] = lv.raw_out;
    a.ny[l] = lv.ny;
    a.nx[l] = lv.nx;
    a.stride[l] = lv.stride;
    a.row_off[l] = off;
    off += d->na * lv.ny * lv.nx;
    for (int j = 0; j < d->na; ++j) {
      a.anchor_w[l][j] = lv.anchor_w[j];
      a.anchor_h[l][j] = lv.anchor_h[j];
    }
  }
  a.row_off[d->nl] = off;
  Y3_REQUIRE(static_cast<long long>(off) * d->bs < (1ll << 31), "head_decode: too many rows");
  const long long warps = (static_cast<long long>(off) * d->bs + y3::kDecodeRows - 1) / y3::kDecodeRows;
  long long blocks = (warps + 7) / 8;
  const long long cap = static_cast<long long>(y3::num_sms()) * 32;
  if (blocks > cap) blocks = cap;
  for (int l = 0; l < d->nl; ++l) {
    Y3_REQUIRE(static_cast<long long>(d->bs) * d->levels[l].ny * d->levels[l].nx * d->levels[l].head_ld < (1ll << 31) &&
                   d->levels[l].ny < 8192 && d->levels[l].nx < 8192,
               "head_decode: level %d too large", l);
  }
  Y3_REQUIRE(d->na <= 8 && d->nl <= 8, "head_decode: na/nl > 8");
  const int niter = (y3::kDecodeRows * d->no + 127) / 128;
  Y3_REQUIRE(niter <= 8, "head_decode: no=%d > 256 is not supported", d->no);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned g = static_cast<unsigned>(blocks);
  switch (niter) {
    case 1: Y3_CHECK_CUDA(::y3::launch_pdl(y3::head_decode_kernel<1>, dim3(g), dim3(256), 0, st, a)); break;
    case 2: Y3_CHECK_CUDA(::y3::launch_pdl(y3::head_decode_kernel<2>, dim3(g), dim3(256), 0, st, a)); break;
    case 3: Y3_CHECK_CUDA(::y3::launch_pdl(y3::head_decode_kernel<3>, dim3(g), dim3(256), 0, st, a)); break;
    case 4: Y3_CHECK_CUDA(::y3::launch_pdl(y3::head_decode_kernel<4>, dim3(g), dim3(256), 0, st, a)); break;
    default: Y3_CHECK_CUDA(::y3::launch_pdl(y3::head_decode_kernel<8>, dim3(g), dim3(256), 0, st, a)); break;
  }
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_detect_decode_fwd(const y3_detect_level* levels, int32_t nl, int32_t bs, int32_t na, int32_t no,
                                    float* z, y3_stream_t stream) {
  Y3_REQUIRE(levels && z && nl >= 1 && nl <= Y3_MAX_LEVELS && na >= 1 && na <= Y3_MAX_ANCHORS && bs > 0 && no >= 5,
             "decode: bad arguments (nl=%d na=%d bs=%d no=%d)", nl, na, bs, no);
  y3::DecodeArgs a{};
  a.nl = nl;
  a.bs = bs;
  a.na = na;
  a.no = no;
  a.z = z;
  int off = 0;
  for (int l = 0; l < nl; ++l) {
    Y3_REQUIRE(levels[l].raw && levels[l].ny > 0 && levels[l].nx > 0, "decode: bad level %d", l);
    a.raw[l] = levels[l].raw;
    a.ny[l] = levels[l].ny;
    a.nx[l] = levels[l].nx;
    a.stride[l] = levels[l].stride;
    a.row_off[l] = off;
    off += na * levels[l].ny * levels[l].nx;
    for (int j = 0; j < na; ++j) {
      a.anchor_w[l][j] = levels[l].anchor_w[j];
      a.anchor_h[l][j] = levels[l].anchor_h[j];
    }
  }
  a.row_off[nl] = off;
  const long long total = static_cast<long long>(off) * no * bs;
  long long blocks = (total + 255) / 256;
  const long long cap = static_cast<long long>(y3::num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::decode_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, static_cast<cudaStream_t>(stream), a));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
