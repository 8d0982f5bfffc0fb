// yolov3_b200 — host-side internals shared by the translation units behind the C ABI.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/yolov3_b200.h"

namespace y3 {

// ---- error plumbing (thread-local last-error string)
int set_error(int code, const char* fmt, ...);
#define Y3_CHECK_CUDA(expr)                                                                            \
  do {                                                                                                 \
    cudaError_t _e = (expr);                                                                           \
    if (_e != cudaSuccess)                                                                             \
      return ::y3::set_error(Y3_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)
#define Y3_REQUIRE(cond, ...)                                       \
  do {                                                              \
    if (!(cond)) return ::y3::set_error(Y3_ERR_BAD_ARG, __VA_ARGS__); \
  } while (0)

// ---- TMA descriptor encoding through the driver entry point (no link-time libcuda dependency)
// dims/strides innermost first; strides in BYTES for dims 1..rank-1; swizzle_bytes in {32,64,128}.
int encode_tensor_map_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                           const uint32_t* box, int swizzle_bytes);

int num_sms();
int pdl_enabled();   // programmatic dependent launch on (default; Y3_PDL=0 or y3_set_pdl(0) turns it off)
void pdl_set(int on);
// Kernel-variant switch (A/B-able at run time; results are bit-identical either way, see y3_set_bn_async in the public header)
#ifndef Y3_BN_ASYNC_DEFAULT
#define Y3_BN_ASYNC_DEFAULT 1
#endif

// ---- tensor-core conv: kernel arguments (device view) and a prepared launch
struct ConvTcArgs {
  int mode;  // 0: "flat" stride-1 (1x1 / 3x3) on the padded pixel list; 1: "patch" stride-2 3x3
  int taps, kblocks, cin;
  int a_coff, a_ld;
  uint32_t a_tx_bytes;   // bytes one A box delivers
  int xpair;             // patch mode with x-paired weights: 6 taps of 2*c_in channels
  int stages;            // depth of the shared-memory ring (set by the launcher from the tile configuration)
  int bres;              // 1: the whole weight tile stays resident in shared memory (loaded once per CTA)
  int m_tiles, n_tiles;
  // flat geometry (input and conv-output share it)
  int hp, wp, rows_total;
  uint32_t plane_mul, plane_shr, wp_mul, wp_shr;  // exact division by hp*wp and wp (fast_div)
  // patch geometry
  int tw, th, tiles_w, tiles_h, ho, wo;
  // epilogue
  const float* bias;
  int cout, act;
  __nv_bfloat16* out;
  int out_ld, out_coff, upsample;
  const __nv_bfloat16* res;
  int res_ld, res_coff;
  float* out_f32;   // fp32 pixel-major output [n*ho*wo, out_f32_ld] (Detect heads) instead of `out`
  int out_f32_ld;
  int* err;
  // custom tap list (flat mode, no halo reuse): tap t reads the pixel list shifted by tap_shift[t] rows and the weight
  // columns [tap_wcol[t] * cin, +cin).  phase = 1: output pixel (oy, ox) is stored at (2 oy + ph_a, 2 ox + ph_b) of a padded
  // [n, 2 oh + 2, 2 ow + 2] grid (one parity class of a transposed stride-2 convolution; residual read from the same place)
  int custom_taps;
  int tap_shift[4], tap_wcol[4];
  int phase, ph_a, ph_b;
};

struct ConvTcExtra {  // host side of the above (conv_tc_prepare)
  int ntaps;
  int dr[4], ds[4];   // tap offsets in input-pixel units (rows, columns), >= 0 or negative
  int wcol[4];        // weight tap index of each
  int phase, ph_a, ph_b;
};

struct ConvTcPlan {
  CUtensorMap map_a, map_b;
  int halo;    // 1: stride-1 3x3 with one A box per filter row (halo reuse)
  int bres;    // 1: weights resident in shared memory (single N tile, small K)
  ConvTcArgs args;
  int block_n, block_k;
  int grid;
};
int conv_tc_prepare(const y3_conv_desc& d, ConvTcPlan* plan, bool select_only = false, const ConvTcExtra* extra = nullptr);
int conv_tc_launch(const ConvTcPlan& plan, cudaStream_t stream);
int pool_launch(const y3_pool_desc& d, cudaStream_t stream);
int wgrad_tc_enabled();
int wgrad_tc(const y3_wgrad_desc& d, cudaStream_t stream);
int wgrad_tc_s2_supported(int h, int w);
int pool_train_fwd(const y3_pool_desc& d, uint8_t* idx, cudaStream_t stream);
int pool_bwd(const y3_pool_desc& d, const uint8_t* idx, int accumulate, cudaStream_t stream);

}  // namespace y3
