// yolov3_b200 — baseline JPEG decode on the device, bit for bit cv2.imread (libjpeg-turbo defaults; see y3_jpeg.cuh for the
// arithmetic and the host parse).  Four launches per batch, one desc per image:
//   unstuff_kernel   one block per image: drops stuffed zeros and RSTn markers (block-wide scan of kept bytes)
//   huffman_kernel   one block per image: self-synchronising subsequence decode (Weissenberger & Schmidt, ICPP 2018) —
//                    one thread per kSubBits-bit subsequence of a restart segment; rounds pass each exit state on as the
//                    next entry until nothing changes (segment starts are exact, so the fixed point is the sequential
//                    decode); a scan of block counts places each subsequence; a second decode writes the coefficients;
//                    then the per-component DC prefix sums, reset at each restart
//   idct_kernel      8 threads per DCT block (columns, then rows), into padded component planes
//   color_kernel     one thread per output pixel: fancy upsampling, YCbCr -> BGR, EXIF orientation, HWC store
// Integer arithmetic only; compiled without fast-math all the same (build.py EXACT_SOURCES).
#include "y3_common.cuh"
#include "y3_internal.h"
#include "y3_jpeg.cuh"

namespace y3 {
namespace {

using namespace jpeg;

constexpr int kThreads = 256;
constexpr int kUnstuffPerThread = 16;

// exclusive block scan of one int per thread; *total gets the sum.  sh: >= 32 ints of shared memory.
__device__ __forceinline__ int block_excl_scan(int v, int* sh, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) sh[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int s = lane < (kThreads >> 5) ? sh[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    sh[lane] = s;
  }
  __syncthreads();
  const int base = warp ? sh[warp - 1] : 0;
  *total = sh[(kThreads >> 5) - 1];
  return base + x - v;
}

__global__ void __launch_bounds__(kThreads) unstuff_kernel(const y3_jpeg_desc* __restrict__ descs) {
  __shared__ int sh[32];
  pdl_entry();
  const y3_jpeg_desc& d = descs[blockIdx.x];
  const Layout L = layout(d.geom);
  const uint8_t* in = static_cast<const uint8_t*>(d.data);
  uint8_t* out = static_cast<uint8_t*>(d.ws) + L.unst;
  const int n = d.geom.data_len;
  int base = 0;
  for (int t0 = 0; t0 < n; t0 += kThreads * kUnstuffPerThread) {
    const int i0 = t0 + threadIdx.x * kUnstuffPerThread;
    uint32_t keep = 0;
    for (int k = 0; k < kUnstuffPerThread; ++k)
      if (i0 + k < n && keep_byte(in, i0 + k, n)) keep |= 1u << k;
    int total;
    int o = base + block_excl_scan(__popc(keep), sh, &total);
    for (int k = 0; k < kUnstuffPerThread; ++k)
      if (keep >> k & 1u) out[o++] = in[i0 + k];
    base += total;
  }
}

__device__ __forceinline__ int find_seg(const int32_t* segsub, int n_segs, int q) {  // last s with segsub[s] <= q
  int lo = 0, hi = n_segs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (segsub[mid] <= q) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// pair scan for the DC prediction: (restart seen, sum since the last restart)
__device__ __forceinline__ void seg_scan(int& f, unsigned& s, int* shf, unsigned* shs) {
  shf[threadIdx.x] = f;
  shs[threadIdx.x] = s;
  __syncthreads();
  for (int o = 1; o < kThreads; o <<= 1) {
    int pf = 0;
    unsigned ps = 0;
    if (threadIdx.x >= o) {
      pf = shf[threadIdx.x - o];
      ps = shs[threadIdx.x - o];
    }
    __syncthreads();
    if (threadIdx.x >= o) {
      s = f ? s : s + ps;
      f |= pf;
      shf[threadIdx.x] = f;
      shs[threadIdx.x] = s;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kThreads) huffman_kernel(const y3_jpeg_desc* __restrict__ descs, int32_t* __restrict__ err_flags) {
  __shared__ Tables T;
  __shared__ uint8_t nat[64];
  __shared__ uint8_t canon[8];
  __shared__ int sh[32];
  __shared__ int shf[kThreads];
  __shared__ unsigned shs[kThreads];
  __shared__ int s_err;
  pdl_entry();
  const y3_jpeg_desc& d = descs[blockIdx.x];
  const y3_jpeg_geom g = d.geom;
  const Layout L = layout(g);
  uint8_t* ws = static_cast<uint8_t*>(d.ws);
  const uint8_t* un = ws + L.unst;
  int32_t* segsub = reinterpret_cast<int32_t*>(ws + L.segsub);
  uint64_t* entry = reinterpret_cast<uint64_t*>(ws + L.entry);
  uint64_t* exitv = reinterpret_cast<uint64_t*>(ws + L.exitv);
  int32_t* count = reinterpret_cast<int32_t*>(ws + L.count);
  int32_t* flags = reinterpret_cast<int32_t*>(ws + L.flags);
  int16_t* coef = reinterpret_cast<int16_t*>(ws + L.coef);
  const int32_t* segs = static_cast<const int32_t*>(d.segs);
  {
    const uint2* src = static_cast<const uint2*>(d.tables);
    uint2* dst = reinterpret_cast<uint2*>(&T);
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(Tables) / 8); i += kThreads) dst[i] = src[i];
  }
  if (threadIdx.x == 0) {
    zigzag_table(nat);
    s_err = 0;
  }
  if (threadIdx.x < g.blocks_per_mcu) canon[threadIdx.x] = static_cast<uint8_t>(canonical_block(g, threadIdx.x));
  // subsequences per segment -> segsub (exclusive prefix, n_segs + 1 entries)
  int base = 0;
  for (int s0 = 0; s0 < g.n_segs; s0 += kThreads) {
    const int s = s0 + threadIdx.x;
    const int ns = s < g.n_segs ? max(1, segs[2 * s + 1] * 8 / kSubBits) : 0;
    int total;
    const int pre = block_excl_scan(ns, sh, &total);
    if (s < g.n_segs) segsub[s] = base + pre;
    base += total;
  }
  if (threadIdx.x == 0) segsub[g.n_segs] = base;
  const int n_sub = base;
  __syncthreads();
  auto args = [&](int q, int& s, int& i, int& end, bool& last) {
    s = find_seg(segsub, g.n_segs, q);
    i = q - segsub[s];
    last = q + 1 == segsub[s + 1];
    end = last ? segs[2 * s + 1] * 8 : (i + 1) * kSubBits;
  };
  for (int q = threadIdx.x; q < n_sub; q += kThreads) {
    int s, i, end;
    bool last;
    args(q, s, i, end, last);
    entry[q] = pack_state(i * kSubBits, 0, 0);
    flags[q] = 1;
  }
  __syncthreads();
  // phase 1: rounds until every entry equals its predecessor's exit
  for (;;) {
    for (int q = threadIdx.x; q < n_sub; q += kThreads) {
      if (!(flags[q] & 1)) continue;
      int s, i, end;
      bool last;
      args(q, s, i, end, last);
      const SubResult r = decode_sub<false>(g, T, nat, canon, un + segs[2 * s], segs[2 * s + 1], end, last, entry[q], nullptr, 0);
      exitv[q] = r.exit;
      count[q] = r.blocks;
      flags[q] = r.err ? 2 : 0;
    }
    __syncthreads();
    int changed = 0;
    for (int q = threadIdx.x; q < n_sub; q += kThreads) {
      if (q == 0 || q == segsub[find_seg(segsub, g.n_segs, q)]) continue;
      const uint64_t e = exitv[q - 1];
      if (entry[q] != e) {
        entry[q] = e;
        flags[q] |= 1;
        changed = 1;
      }
    }
    if (!__syncthreads_or(changed)) break;
  }
  // phase 2: block index of each subsequence (exclusive scan of the counts, in place), checked at segment starts
  const int per = (n_sub + kThreads - 1) / kThreads;
  const int q0 = min(n_sub, threadIdx.x * per), q1 = min(n_sub, q0 + per);
  int local = 0, bad = 0;
  for (int q = q0; q < q1; ++q) {
    local += count[q];
    bad |= flags[q] >> 1;
  }
  int total;
  int run = block_excl_scan(local, sh, &total);
  for (int q = q0; q < q1; ++q) {
    const int c = count[q];
    count[q] = run;
    const int s = find_seg(segsub, g.n_segs, q);
    if (g.restart_interval && q == segsub[s] &&
        static_cast<int64_t>(run) != static_cast<int64_t>(s) * g.restart_interval * g.blocks_per_mcu)
      bad = 1;
    run += c;
  }
  if (total != g.n_blocks) bad = 1;
  if (bad) s_err = 1;
  __syncthreads();
  if (s_err) {
    if (threadIdx.x == 0) err_flags[blockIdx.x] = 1;
    return;
  }
  // phase 3: decode again from the synchronised entries, writing the coefficients
  for (int q = threadIdx.x; q < n_sub; q += kThreads) {
    int s, i, end;
    bool last;
    args(q, s, i, end, last);
    decode_sub<true>(g, T, nat, canon, un + segs[2 * s], segs[2 * s + 1], end, last, entry[q], coef, count[q]);
  }
  __syncthreads();
  // DC prediction: per component, in MCU order, reset at each restart; a wrapping sum stored as 16 bits
  const int mcus = g.mcus_x * g.mcus_y;
  for (int c = 0; c < g.ncomp; ++c) {
    const int pc = c == 0 ? g.hmax * g.vmax : 1, off = c == 0 ? 0 : g.hmax * g.vmax + c - 1;
    const int nc = mcus * pc;
    const int chunk = (nc + kThreads - 1) / kThreads;
    const int i0 = min(nc, threadIdx.x * chunk), i1 = min(nc, i0 + chunk);
    auto dc_at = [&](int i) -> int16_t* {
      const int mcu = i / pc;
      return coef + (static_cast<int64_t>(mcu) * g.blocks_per_mcu + off + (i - mcu * pc)) * 64;
    };
    auto reset = [&](int i) {
      const int mcu = i / pc;
      return i == mcu * pc && (g.restart_interval ? mcu % g.restart_interval == 0 : mcu == 0);
    };
    int f = 0;
    unsigned sum = 0;
    for (int i = i0; i < i1; ++i) {
      if (reset(i)) {
        f = 1;
        sum = 0;
      }
      sum += static_cast<unsigned>(static_cast<int>(*dc_at(i)));
    }
    seg_scan(f, sum, shf, shs);  // inclusive over the threads' chunks
    unsigned acc = threadIdx.x ? shs[threadIdx.x - 1] : 0u;
    __syncthreads();
    for (int i = i0; i < i1; ++i) {
      if (reset(i)) acc = 0;
      int16_t* p = dc_at(i);
      acc += static_cast<unsigned>(static_cast<int>(*p));
      *p = static_cast<int16_t>(acc);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) err_flags[blockIdx.x] = 0;
}

constexpr int kIdctBlocks = kThreads / 8;

__global__ void __launch_bounds__(kThreads) idct_kernel(const y3_jpeg_desc* __restrict__ descs,
                                                        const int32_t* __restrict__ err_flags) {
  __shared__ int ws[kIdctBlocks][64];
  pdl_entry();
  const y3_jpeg_desc& d = descs[blockIdx.y];
  const y3_jpeg_geom& g = d.geom;
  const int blk = blockIdx.x * kIdctBlocks + (threadIdx.x >> 3), lane = threadIdx.x & 7;
  if (blk >= g.n_blocks || err_flags[blockIdx.y]) return;  // the 8 threads of a DCT block leave together
  const Layout L = layout(g);
  uint8_t* base = static_cast<uint8_t*>(d.ws);
  const int16_t* coef = reinterpret_cast<const int16_t*>(base + L.coef) + static_cast<int64_t>(blk) * 64;
  int c, bx, by;
  block_place(g, blk, c, bx, by);
  const uint16_t* q = static_cast<const Tables*>(d.tables)->quant[c];
  int* w = ws[threadIdx.x >> 3];
  idct_col(coef, q, lane, w);
  __syncwarp(0xFFu << (threadIdx.x & 24));
  const int pitch = c == 0 ? L.pitch[0] : (c == 1 ? L.pitch[1] : L.pitch[2]);
  const int64_t poff = c == 0 ? L.plane[0] : (c == 1 ? L.plane[1] : L.plane[2]);
  uint8_t row[8];
  idct_row(w, lane, row);
  uint2 v;
  v.x = row[0] | row[1] << 8 | row[2] << 16 | static_cast<uint32_t>(row[3]) << 24;
  v.y = row[4] | row[5] << 8 | row[6] << 16 | static_cast<uint32_t>(row[7]) << 24;
  *reinterpret_cast<uint2*>(base + poff + static_cast<int64_t>(by + lane) * pitch + bx) = v;
}

__global__ void __launch_bounds__(kThreads) color_kernel(const y3_jpeg_desc* __restrict__ descs,
                                                         const int32_t* __restrict__ err_flags) {
  pdl_entry();
  const y3_jpeg_desc& d = descs[blockIdx.z];
  const y3_jpeg_geom g = d.geom;
  const int x = blockIdx.x * kThreads + threadIdx.x, y = blockIdx.y;
  if (x >= g.width || y >= g.height || err_flags[blockIdx.z]) return;
  const Layout L = layout(g);
  const uint8_t* base = static_cast<const uint8_t*>(d.ws);
  const uint8_t* planes[3] = {base + L.plane[0], base + L.plane[1], base + L.plane[2]};
  uint8_t bgr[3];
  pixel_bgr(g, planes, L.pitch, x, y, bgr);
  uint8_t* o = static_cast<uint8_t*>(d.dst) + static_cast<int64_t>(y) * d.dst_pitch + x * 3;
  o[0] = bgr[0];
  o[1] = bgr[1];
  o[2] = bgr[2];
}

}  // namespace
}  // namespace y3

extern "C" int y3_jpeg_parse(const uint8_t* buf, int64_t len, y3_jpeg_info* info, int32_t* segs, int32_t seg_cap) {
  Y3_REQUIRE(buf && info && len >= 0 && seg_cap >= 0 && (segs || seg_cap == 0), "jpeg_parse: bad arguments");
  y3::jpeg::parse(buf, len, info, segs, seg_cap);
  return Y3_OK;
}

extern "C" int64_t y3_jpeg_workspace_bytes(const y3_jpeg_geom* geom) {
  if (!geom) return -1;
  return y3::jpeg::layout(*geom).total;
}

extern "C" int y3_jpeg_decode_batched(const y3_jpeg_desc* descs, const y3_jpeg_desc* host_descs, int32_t n, void* workspace,
                                      int64_t ws_bytes, int32_t* err_flags, y3_stream_t stream) {
  Y3_REQUIRE(descs && host_descs && workspace && err_flags && n > 0 && n <= 65535 && ws_bytes > 0,
             "jpeg_decode: bad arguments (n %d)", n);
  const uintptr_t w0 = reinterpret_cast<uintptr_t>(workspace), w1 = w0 + static_cast<uintptr_t>(ws_bytes);
  int max_blocks = 0, max_h = 0, max_w = 0;
  for (int i = 0; i < n; ++i) {
    const y3_jpeg_desc& d = host_descs[i];
    const y3_jpeg_geom& g = d.geom;
    Y3_REQUIRE(g.ncomp == 1 || g.ncomp == 3, "jpeg_decode: item %d: %d components", i, g.ncomp);
    Y3_REQUIRE(g.src_h > 0 && g.src_w > 0 && g.orientation >= 1 && g.orientation <= 8 &&
                   g.height == (g.orientation >= 5 ? g.src_w : g.src_h) && g.width == (g.orientation >= 5 ? g.src_h : g.src_w),
               "jpeg_decode: item %d: bad size / orientation", i);
    Y3_REQUIRE(g.hmax >= 1 && g.vmax >= 1 && g.mcus_x == (g.src_w + 8 * g.hmax - 1) / (8 * g.hmax) &&
                   g.mcus_y == (g.src_h + 8 * g.vmax - 1) / (8 * g.vmax) &&
                   g.blocks_per_mcu == (g.ncomp == 3 ? g.hmax * g.vmax + 2 : 1) &&
                   static_cast<int64_t>(g.n_blocks) == static_cast<int64_t>(g.mcus_x) * g.mcus_y * g.blocks_per_mcu,
               "jpeg_decode: item %d: inconsistent MCU geometry", i);
    Y3_REQUIRE(g.n_segs >= 1 && g.data_len >= 0 && g.unstuffed_len >= 0 && g.unstuffed_len <= g.data_len &&
                   g.comp_dc[0] >= 0 && g.comp_dc[0] <= 1 && g.comp_dc[1] >= 0 && g.comp_dc[1] <= 1 && g.comp_dc[2] >= 0 &&
                   g.comp_dc[2] <= 1 && g.comp_ac[0] >= 0 && g.comp_ac[0] <= 1 && g.comp_ac[1] >= 0 && g.comp_ac[1] <= 1 &&
                   g.comp_ac[2] >= 0 && g.comp_ac[2] <= 1,
               "jpeg_decode: item %d: bad stream description", i);
    Y3_REQUIRE(d.data && d.segs && d.dst && d.dst_pitch >= 3 * g.width && (reinterpret_cast<uintptr_t>(d.tables) & 7) == 0 &&
                   d.tables,
               "jpeg_decode: item %d: bad pointer or pitch", i);
    const uintptr_t a = reinterpret_cast<uintptr_t>(d.ws);
    Y3_REQUIRE((a & 255) == 0 && a >= w0 && a + static_cast<uintptr_t>(y3::jpeg::layout(g).total) <= w1,
               "jpeg_decode: item %d: workspace outside [workspace, workspace + ws_bytes) or not 256-byte aligned", i);
    max_blocks = max(max_blocks, g.n_blocks);
    max_h = max(max_h, g.height);
    max_w = max(max_w, g.width);
  }
  Y3_REQUIRE(max_h <= 65535, "jpeg_decode: image too tall (%d rows)", max_h);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::unstuff_kernel, dim3(n), dim3(y3::kThreads), 0, s, descs));
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::huffman_kernel, dim3(n), dim3(y3::kThreads), 0, s, descs, err_flags));
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::idct_kernel, dim3((max_blocks + y3::kIdctBlocks - 1) / y3::kIdctBlocks, n),
                                 dim3(y3::kThreads), 0, s, descs, static_cast<const int32_t*>(err_flags)));
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::color_kernel, dim3((max_w + y3::kThreads - 1) / y3::kThreads, max_h, n),
                                 dim3(y3::kThreads), 0, s, descs, static_cast<const int32_t*>(err_flags)));
  return Y3_OK;
}
