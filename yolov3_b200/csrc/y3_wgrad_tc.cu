// yolov3_b200 — weight gradient of a conv on the Hopper tensor cores (wgmma); every training conv runs it.
//   dW[co, tap, ci] += sum over padded pixels p of dy[p, co] * x[p + shift(tap), ci]
// is a GEMM whose K dimension is the PIXEL index: both operands sit in memory pixel-major with channels contiguous, i.e.
// "MN-major" (transposed) wgmma operands: shared-memory descriptors of the canonical MN-major swizzled layout — 64
// channels (128 B) contiguous, 8 pixel rows per swizzle atom, SBO = bytes between 8-row groups, LBO = bytes between
// 64-channel blocks.  The same TMA boxes as the forward conv ([64 pixels x 64 channels], the x box shifted by the tap)
// land in exactly that layout — no transposition anywhere.
// One CTA = one (128-co block, N-ci block, tap) output tile over a range of pixels (split-K): warp 8 streams the boxes,
// warpgroups 0 and 1 accumulate co rows [0, 64) and [64, 128) in registers and finish with 8-byte fp32 vector reductions
// (or plain stores) into dW laid out [co][taps][ci], the flat gradient buffer's order
// (reference: autograd of Conv.forward, models/common.py:71-75).
#include <cuda_bf16.h>

#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {
namespace {

constexpr int kWgM = 128;     // co per tile
constexpr int kWgK = 64;      // pixels per pipeline stage (flat mode); the stride-2 patch mode uses 80 = tw x th
constexpr int kWgThreads = 288;  // warpgroups 0-1 wgmma + epilogue, warp 8 producer (no idle warps)
constexpr int kWgProducerWarp = 8;

struct WgTcArgs {
  int co, ci, taps, wp;
  int n_ci_tiles;       // ci tiles of width N
  int kblocks_total;    // ceil(rows / 64)
  int kblocks_per_cta;  // pixel blocks one CTA accumulates (split-K)
  int dy_coff, x_coff;
  float* dw;            // [co][taps][ci]
  int single;           // 1: this CTA is the only contributor to its dW tile AND dw need not be accumulated into (plain stores)
  int* err;
  uint32_t lbo_a, lbo_b, sbo_a, sbo_b;  // descriptor strides in bytes
  // stride-2 "patch" mode (KB = 80): a K block is a tw x th patch of OUTPUT pixels; dy comes through a 4-D map of its padded
  // grid, x through the 5-D parity view the forward stride-2 conv uses (one box per tap)
  int s2, tw, th, tiles_w, tiles_per_img, x_ld;
};

template <int N, int KB>
struct WgCfg {
  static constexpr int kBCols = N >= 64 ? 64 : N;            // channels per B box
  static constexpr uint32_t kStage = 2 * KB * 128 + (N / kBCols) * KB * kBCols * 2;
  static constexpr int kStages = (200 * 1024) / kStage > 6 ? 6 : (200 * 1024) / kStage;
  static constexpr size_t kSmemBytes = size_t(kStages) * kStage + 1024 + 256;
  static_assert(kStages >= 2, "wgrad: the ring needs two stages");
};

// N = ci tile width (32 .. 128); KB = pixels per K block
template <int N, int KB>
__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_x, const WgTcArgs p) {
  constexpr int kBCols = WgCfg<N, KB>::kBCols;
  constexpr int kBBoxes = N / kBCols;
  constexpr uint32_t kABox = KB * 128;                // one A box: KB pixel rows x 64 channels
  constexpr uint32_t kABytes = 2 * kABox;             // co 0-63 | co 64-127
  constexpr uint32_t kBBox = KB * kBCols * 2;
  constexpr uint32_t kStage = WgCfg<N, KB>::kStage;
  constexpr int STAGES = WgCfg<N, KB>::kStages;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * kStage);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.y;  // co tile * n_ci_tiles + ci tile
  const int co0 = (tile / p.n_ci_tiles) * kWgM, ci0 = (tile % p.n_ci_tiles) * N;
  const int tap = blockIdx.z;
  const int shift = p.taps == 9 ? (tap / 3 - 1) * p.wp + (tap % 3 - 1) : 0;
  const int kb0 = blockIdx.x * p.kblocks_per_cta;
  const int kb1 = min(kb0 + p.kblocks_per_cta, p.kblocks_total);
  const int k_iters = kb1 - kb0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_dy);
    tma_prefetch_desc(&map_x);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // prologue above overlaps the previous kernel's tail (y3_common.cuh)
  pdl_trigger();
  if (k_iters <= 0) return;

  if (warp == kWgProducerWarp) {
    uint32_t stage = 0, phase = 0;
    for (int it = 0; it < k_iters; ++it) {
      mbar_wait(&empty_bar[stage], phase ^ 1u, p.err, 11);
      if (elect_one()) {
        uint8_t* a_dst = smem + stage * kStage;
        uint8_t* b_dst = a_dst + kABytes;
        mbar_expect_tx(&full_bar[stage], kStage);
        if (KB == 80) {  // stride-2 patch mode
          const int kb = kb0 + it;
          const int img = kb / p.tiles_per_img, t = kb - img * p.tiles_per_img;
          const int oy0 = (t / p.tiles_w) * p.th, ox0 = (t % p.tiles_w) * p.tw;
          const int r = tap / 3, sx = tap - r * 3;
          tma_load_4d(a_dst, &map_dy, &full_bar[stage], p.dy_coff + co0, 1 + ox0, 1 + oy0, img);
          tma_load_4d(a_dst + kABox, &map_dy, &full_bar[stage], p.dy_coff + co0 + 64, 1 + ox0, 1 + oy0, img);
#pragma unroll
          for (int b = 0; b < kBBoxes; ++b)  // input pixel of output (oy, ox), tap (r, sx): padded (2 oy + r, 2 ox + sx)
            tma_load_5d(b_dst + b * kBBox, &map_x, &full_bar[stage], (sx & 1) * p.x_ld + p.x_coff + ci0 + b * kBCols,
                        ox0 + (sx >> 1), r & 1, oy0 + (r >> 1), img);
        } else {
          const int row = (kb0 + it) * KB;
          tma_load_2d(a_dst, &map_dy, &full_bar[stage], p.dy_coff + co0, row);
          tma_load_2d(a_dst + kABox, &map_dy, &full_bar[stage], p.dy_coff + co0 + 64, row);
#pragma unroll
          for (int b = 0; b < kBBoxes; ++b)
            tma_load_2d(b_dst + b * kBBox, &map_x, &full_bar[stage], p.x_coff + ci0 + b * kBCols, row + shift);
        }
      }
      __syncwarp();
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
  } else {
    const int wg = warp >> 2;  // co rows [64 wg, 64 wg + 64) of the tile
    const uint32_t hi_a = wgmma_desc_hi(p.sbo_a, 128);
    const uint32_t hi_b = wgmma_desc_hi(p.sbo_b, kBCols * 2);
    const uint32_t a0 = smem_u32(smem) + uint32_t(wg) * kABox, b0 = smem_u32(smem) + kABytes;
    constexpr uint32_t kRowA = 128, kRowB = kBCols * 2;  // bytes per pixel row inside a box
    float acc[N / 2];
    uint32_t stage = 0, phase = 0, prev = 0;
    for (int it = 0; it < k_iters; ++it) {
      mbar_wait(&full_bar[stage], phase, p.err, 12);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KB / 16; ++ks) {
        const uint64_t adesc = wgmma_desc(hi_a, a0 + stage * kStage + ks * 16 * kRowA, p.lbo_a);
        const uint64_t bdesc = wgmma_desc(hi_b, b0 + stage * kStage + ks * 16 * kRowB, p.lbo_b);
        Wgmma<N>::template mma<1, 1>(acc, adesc, bdesc, (it | ks) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous stage's MMAs have completed: its slot may be refilled
      if (it > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);

    // epilogue: accumulator row = co, column = ci; fp32 vector reductions (or plain stores) into dW.  ci and this thread's
    // column c are even, so ci0 + c < ci puts both columns of the pair inside the row; columns past ci are discarded.
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int co = co0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (co >= p.co) continue;
      float* dst = p.dw + (static_cast<long long>(co) * p.taps + tap) * p.ci + ci0;
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        const int c = 8 * j + cq;
        if (ci0 + c >= p.ci) continue;
        const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        float* q = dst + c;
        if (p.single)  // this CTA is the only contributor: plain 8-byte store
          *reinterpret_cast<float2*>(q) = make_float2(v0, v1);
        else
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(q), "f"(v0), "f"(v1) : "memory");
      }
    }
  }
}

template <int N, int KB>
int wgrad_tc_launch(const CUtensorMap& mdy, const CUtensorMap& mx, const WgTcArgs& a, dim3 grid, cudaStream_t stream) {
  constexpr size_t smem = WgCfg<N, KB>::kSmemBytes;
  auto kern = wgrad_tc_kernel<N, KB>;
  static bool attr_set = false;
  if (!attr_set) {
    Y3_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    attr_set = true;
  }
  Y3_CHECK_CUDA(launch_pdl(kern, grid, dim3(kWgThreads), smem, stream, mdy, mx, a));
  return Y3_OK;
}

}  // namespace

// (tw, th) with tw * th == 80 for the stride-2 patch mode: the fewest tw x th patches over the ho x wo output, ties to the
// smallest th.  An exact tiling, when one exists, is the unique minimum (ceil(ho/th) * ceil(wo/tw) >= ho * wo / 80, with
// equality only when both divide), so it is the one chosen.
static void s2_patch(int ho, int wo, int* tw, int* th) {
  long long best = -1;
  for (int cand_th = 1; cand_th <= 80; ++cand_th) {
    if (80 % cand_th) continue;
    const int cand_tw = 80 / cand_th;
    const long long patches = static_cast<long long>((ho + cand_th - 1) / cand_th) * ((wo + cand_tw - 1) / cand_tw);
    if (best < 0 || patches < best) {
      best = patches;
      *tw = cand_tw;
      *th = cand_th;
    }
  }
}

static int wgrad_tc_s2(const y3_wgrad_desc& d, cudaStream_t stream) {
  // dW[co, tap, ci] += sum over OUTPUT pixels p of dy[p, co] * x[2p + tap, ci]: no zero-stuffed copy of dy, a quarter of the
  // K extent of the stride-1 formulation on the input grid (which multiplied 75 % zeros).
  // A patch that overhangs the output reads dy's zero halo (column wo + 1, row ho + 1) and past it the map's out-of-bounds
  // zero fill, so its extra pixels add exactly 0.  The x map's channel extent is 2 * x_ld (the parity view), so B columns
  // past ci read neighbouring channels: column n of the product depends only on column n of B, and the epilogue discards
  // those columns.
  Y3_REQUIRE(d.ksize == 3 && d.h % 2 == 0 && d.w % 2 == 0, "wgrad: the stride-2 form needs a 3x3 conv and even h, w");
  const int ho = d.h / 2, wo = d.w / 2;
  int tw = 0, th = 0;
  s2_patch(ho, wo, &tw, &th);
  const int n_tile = d.ci >= 128 ? 128 : (d.ci >= 64 ? 64 : 32);
  const uint32_t bcols = n_tile >= 64 ? 64 : n_tile;
  CUtensorMap mdy, mx;
  {
    const uint64_t ld = static_cast<uint64_t>(d.dy_ld);
    const uint64_t dims[4] = {static_cast<uint64_t>(d.dy_coff + d.co), static_cast<uint64_t>(wo + 2), static_cast<uint64_t>(ho + 2),
                              static_cast<uint64_t>(d.n)};
    const uint64_t strides[4] = {0, ld * 2, static_cast<uint64_t>(wo + 2) * ld * 2, static_cast<uint64_t>(ho + 2) * (wo + 2) * ld * 2};
    const uint32_t box[4] = {64, static_cast<uint32_t>(tw), static_cast<uint32_t>(th), 1};
    int rc = encode_tensor_map_bf16(&mdy, d.dy, 4, dims, strides, box, 128);
    if (rc) return rc;
  }
  {
    const uint64_t ld = static_cast<uint64_t>(d.x_ld);
    const int hp = d.h + 2, wp = d.w + 2;
    const uint64_t dims[5] = {2 * ld, static_cast<uint64_t>(wp / 2), 2, static_cast<uint64_t>(hp / 2), static_cast<uint64_t>(d.n)};
    const uint64_t strides[5] = {0, 2 * ld * 2, static_cast<uint64_t>(wp) * ld * 2, 2ull * wp * ld * 2,
                                 static_cast<uint64_t>(hp) * wp * ld * 2};
    const uint32_t box[5] = {bcols, static_cast<uint32_t>(tw), 1, static_cast<uint32_t>(th), 1};
    int rc = encode_tensor_map_bf16(&mx, d.x, 5, dims, strides, box, bcols * 2);
    if (rc) return rc;
  }
  WgTcArgs a{};
  a.co = d.co;
  a.ci = d.ci;
  a.taps = 9;
  a.wp = d.w + 2;
  a.n_ci_tiles = (d.ci + n_tile - 1) / n_tile;
  a.s2 = 1;
  a.tw = tw;
  a.th = th;
  a.tiles_w = (wo + tw - 1) / tw;
  a.tiles_per_img = a.tiles_w * ((ho + th - 1) / th);
  a.x_ld = d.x_ld;
  a.kblocks_total = d.n * a.tiles_per_img;
  a.dy_coff = d.dy_coff;
  a.x_coff = d.x_coff;
  a.dw = d.dw;
  a.err = nullptr;
  a.lbo_a = 80 * 128;
  a.lbo_b = 80 * bcols * 2;
  a.sbo_a = 1024;
  a.sbo_b = 8 * bcols * 2;
  const int tiles = ((d.co + kWgM - 1) / kWgM) * a.n_ci_tiles;
  // split the pixel dimension so that the grid is ONE wave of CTAs, one per SM (floor, not ceil: a grid a few CTAs over a
  // wave costs a whole extra wave)
  long long want = static_cast<long long>(num_sms()) / (static_cast<long long>(tiles) * 9);
  long long max_split = (a.kblocks_total + 7) / 8;
  if (want > max_split) want = max_split;
  if (want < 1 || d.deterministic) want = 1;
  a.kblocks_per_cta = static_cast<int>((a.kblocks_total + want - 1) / want);
  const unsigned splits = static_cast<unsigned>((a.kblocks_total + a.kblocks_per_cta - 1) / a.kblocks_per_cta);
  a.single = (splits == 1 && !d.accumulate) ? 1 : 0;
  const dim3 grid(splits, static_cast<unsigned>(tiles), 9u);
  switch (n_tile) {
    case 128: return wgrad_tc_launch<128, 80>(mdy, mx, a, grid, stream);
    case 64: return wgrad_tc_launch<64, 80>(mdy, mx, a, grid, stream);
    default: return wgrad_tc_launch<32, 80>(mdy, mx, a, grid, stream);
  }
}

int wgrad_tc(const y3_wgrad_desc& d, cudaStream_t stream) {
  if (d.stride == 2) return wgrad_tc_s2(d, stream);
  const int taps = d.ksize * d.ksize;
  const long long rows = static_cast<long long>(d.n) * (d.h + 2) * (d.w + 2);
  Y3_REQUIRE(rows < (1ll << 31) - 4096, "wgrad: too many pixels");
  const int n_tile = d.ci >= 128 ? 128 : (d.ci >= 64 ? 64 : 32);
  CUtensorMap mdy, mx;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(d.dy_coff + d.co), static_cast<uint64_t>(rows)};
    const uint64_t strides[2] = {0, static_cast<uint64_t>(d.dy_ld) * 2};
    const uint32_t box[2] = {64, static_cast<uint32_t>(kWgK)};
    int rc = encode_tensor_map_bf16(&mdy, d.dy, 2, dims, strides, box, 128);
    if (rc) return rc;
  }
  const uint32_t bcols = n_tile >= 64 ? 64 : n_tile;
  {
    // the extent x_coff + ci clips the last ci tile: its B columns past ci are zero-filled
    const uint64_t dims[2] = {static_cast<uint64_t>(d.x_coff + d.ci), static_cast<uint64_t>(rows)};
    const uint64_t strides[2] = {0, static_cast<uint64_t>(d.x_ld) * 2};
    const uint32_t box[2] = {bcols, static_cast<uint32_t>(kWgK)};
    int rc = encode_tensor_map_bf16(&mx, d.x, 2, dims, strides, box, bcols * 2);
    if (rc) return rc;
  }
  WgTcArgs a{};
  a.co = d.co;
  a.ci = d.ci;
  a.taps = taps;
  a.wp = d.w + 2;
  a.n_ci_tiles = (d.ci + n_tile - 1) / n_tile;
  a.kblocks_total = static_cast<int>((rows + kWgK - 1) / kWgK);
  a.dy_coff = d.dy_coff;
  a.x_coff = d.x_coff;
  a.dw = d.dw;
  a.err = nullptr;
  a.lbo_a = kWgK * 128;          // bytes between 64-channel boxes
  a.lbo_b = kWgK * bcols * 2;
  a.sbo_a = 1024;                 // 8 pixel rows of 128 B
  a.sbo_b = 8 * bcols * 2;        // 8 pixel rows of a B box
  const int tiles = ((d.co + kWgM - 1) / kWgM) * a.n_ci_tiles;
  // split the pixel dimension into one wave of CTAs, one per SM (floor: a grid a few CTAs over a wave costs a whole extra
  // wave); at least 8 pixel blocks per CTA
  long long want = static_cast<long long>(num_sms()) / (static_cast<long long>(tiles) * taps);
  long long max_split = (a.kblocks_total + 7) / 8;
  if (want > max_split) want = max_split;
  if (want < 1) want = 1;
  if (d.deterministic) want = 1;  // one CTA per dW tile: a single adder per address, bit-reproducible (slow on early layers)
  a.kblocks_per_cta = static_cast<int>((a.kblocks_total + want - 1) / want);
  const unsigned splits = static_cast<unsigned>((a.kblocks_total + a.kblocks_per_cta - 1) / a.kblocks_per_cta);
  a.single = (splits == 1 && !d.accumulate) ? 1 : 0;
  const dim3 grid(splits, static_cast<unsigned>(tiles), static_cast<unsigned>(taps));
  switch (n_tile) {
    case 128: return wgrad_tc_launch<128, kWgK>(mdy, mx, a, grid, stream);
    case 64: return wgrad_tc_launch<64, kWgK>(mdy, mx, a, grid, stream);
    default: return wgrad_tc_launch<32, kWgK>(mdy, mx, a, grid, stream);
  }
}

}  // namespace y3
