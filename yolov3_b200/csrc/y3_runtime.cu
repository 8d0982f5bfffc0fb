// yolov3_b200 — host runtime glue behind the C ABI: error strings, device probe, TMA descriptor encoding.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "y3_internal.h"

namespace y3 {

namespace {
thread_local char g_err[512] = {0};

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
std::mutex g_mu;
EncodeTiledFn g_encode = nullptr;

EncodeTiledFn get_encode() {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  return g_encode;
}
}  // namespace

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int num_sms() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
      sms = 132;
  }
  return sms;
}

namespace {
int g_pdl = -1;
}
int pdl_enabled() {
  if (g_pdl < 0) {
    const char* e = getenv("Y3_PDL");
    g_pdl = (e && e[0] == '0') ? 0 : 1;
  }
  return g_pdl;
}
void pdl_set(int on) { g_pdl = on ? 1 : 0; }

int encode_tensor_map(CUtensorMap* out, int fmt, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                      const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error(Y3_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstr[i - 1] = strides[i];
  }
  const CUtensorMapSwizzle sw = swizzle_bytes == 128  ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                      : CU_TENSOR_MAP_SWIZZLE_NONE;
  // e4m3 moves as raw bytes: TMA only copies, the wgmma reads the format
  const CUtensorMapDataType dt = fmt == Y3_FMT_E4M3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  const CUresult r = enc(out, dt, static_cast<cuuint32_t>(rank), const_cast<void*>(base),
                         gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char shape[160] = {0};
    int off = 0;
    for (int i = 0; i < rank; ++i)
      off += snprintf(shape + off, sizeof(shape) - off, "[%llu/%u/%llu]", (unsigned long long)dims[i], box[i],
                      (unsigned long long)(i ? strides[i] : 0));
    return set_error(Y3_ERR_CUDA, "cuTensorMapEncodeTiled failed (CUresult %d) rank %d dims/box/stride %s", int(r), rank,
                     shape);
  }
  return Y3_OK;
}

}  // namespace y3

extern "C" int y3_version(void) { return 101; }

extern "C" int y3_last_error(char* buf, size_t n) {
  const size_t len = strlen(y3::g_err);
  if (buf && n) {
    const size_t c = len < n - 1 ? len : n - 1;
    memcpy(buf, y3::g_err, c);
    buf[c] = 0;
  }
  return static_cast<int>(len);
}

extern "C" int y3_device_check(void) {
  int dev = 0, major = 0, minor = 0;
  Y3_CHECK_CUDA(cudaGetDevice(&dev));
  Y3_CHECK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  Y3_CHECK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0)
    return y3::set_error(Y3_ERR_UNSUPPORTED, "device compute capability %d.%d is not sm_90", major, minor);
  return Y3_OK;
}

extern "C" int y3_set_pdl(int32_t on) {
  const int prev = y3::pdl_enabled();
  y3::pdl_set(on);
  return prev;
}

extern "C" int64_t y3_abi_sizeof(int32_t which) {
  switch (which) {
    case 0: return sizeof(y3_conv_desc);
    case 1: return sizeof(y3_first_desc);
    case 2: return sizeof(y3_pool_desc);
    case 3: return sizeof(y3_detect_level);
    case 4: return sizeof(y3_decode_desc);
    case 5: return sizeof(y3_op);
    case 6: return sizeof(y3_nms_params);
    case 7: return sizeof(y3_loss_desc);
    case 8: return sizeof(y3_bn_act_desc);
    case 9: return sizeof(y3_bn_bwd_desc);
    case 10: return sizeof(y3_wgrad_desc);
    case 11: return sizeof(y3_pack_item);
    case 12: return sizeof(y3_letterbox_desc);
    case 13: return sizeof(y3_amax_desc);
    case 14: return sizeof(y3_resize_item);
    case 15: return sizeof(y3_augment_desc);
    case 16: return sizeof(y3_jpeg_geom);
    case 17: return sizeof(y3_jpeg_info);
    case 18: return sizeof(y3_jpeg_desc);
    case 19: return sizeof(y3_halo_item);
  }
  return -1;
}
