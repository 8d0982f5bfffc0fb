// yolov3_b200 — implicit-GEMM convolution on the Hopper tensor cores (wgmma, fp32 accumulators in registers), operands
// staged by TMA, folded-BN bias + SiLU (+ residual, + nearest-2x upsample, + concat-offset / Detect store) fused into the
// epilogue.  Replaces Conv.forward_fuse (reference models/common.py:77-81) and the adds/copies around it.
//
// GEMM view:  D[pixel, cout] = sum_{tap, c} A[pixel shifted by tap, c] * W[cout, tap, c]
//   * activations are bf16 "padded NHWC" [n, h+2, w+2, ld] with an all-zero halo, so for a stride-1 conv the A tile
//     of filter tap (r,s) is simply the [128 pixels x BLOCK_K channels] box of the flat pixel list shifted by
//     (r-1)*(w+2)+(s-1) rows: one 2-D TMA box per (tap, k-block), zero quantisation waste, no im2col buffer
//     ("flat" mode; halo pixels are computed but never stored).
//   * a stride-2 conv reads the same buffer through a 5-D view (2*ld, (w+2)/2, 2, (h+2)/2, n) that splits rows and
//     columns by parity; the A tile of tap (r,s) for a TH x TW patch of output pixels is one 5-D TMA box ("patch").
//   * weights are bf16 [cout_pad, taps*cin] (K-major); B tile = [BLOCK_N x BLOCK_K] box.
// Warp roles (288 threads, 1 CTA/SM, persistent over tiles): warp 8 = TMA producer (the whole warp runs the loop, one elected
// lane issues); warpgroups 0 and 1 (warps 0-7) = consumers, each owning 64 of the tile's 128 rows: it issues the
// m64 x BLOCK_N wgmma of its rows for every stage of the smem ring, releases a stage as soon as the MMAs that read it have
// completed, and after the last k-block converts its accumulators straight from the registers (bias, SiLU, residual,
// bf16 / fp32 stores).  While the consumers run the epilogue the producer already fills the ring for their next tile.
#include <cuda_bf16.h>

#include <cstdlib>
#include <type_traits>

#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {

namespace {

constexpr int kBlockM = 128;
// two consumer warpgroups + one producer warp: no idle warps, up to 224 registers per thread (the N = 256 tiles keep 128
// accumulators each)
constexpr int kThreads = 288;
constexpr int kProducerWarp = 8;
constexpr int kSmemBudget = 221 * 1024;  // ring (+ resident weights); alignment slack and barriers come on top (227 KB max)

// HALO = true (stride-1 3x3, BLOCK_K = 64 or 32): one pipeline stage covers a whole filter ROW (3 taps): the A operand is
// ONE TMA box of 128+2 consecutive pixels and the three taps read it at row offsets 0/1/2 through wgmma descriptors whose
// start address is not aligned to the swizzle pattern (the swizzle is a function of the absolute shared-memory address,
// so the descriptor's base offset stays 0).  A rows fetched per k-block drop from 9*128 to 3*130 and the producer runs a
// third of the pipeline stages.
template <int BLOCK_N, int BLOCK_K, bool HALO>
struct Cfg {
  static constexpr uint32_t kARows = HALO ? kBlockM + 2 : kBlockM;
  static constexpr uint32_t kATxBytes = kARows * BLOCK_K * 2;                         // bytes one A box delivers (flat mode)
  static constexpr uint32_t kABytes = (kATxBytes + 1023u) / 1024u * 1024u;            // slot size, 1 KB aligned
  static constexpr uint32_t kTaps = HALO ? 3 : 1;                                     // filter taps per stage
  static constexpr uint32_t kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr uint32_t kStageBytes = kABytes + kTaps * kBBytes;
  static constexpr int kMaxStages = 8;
  static constexpr int kStagesRaw = kSmemBudget / kStageBytes;
  static constexpr int kStages = kStagesRaw > kMaxStages ? kMaxStages : kStagesRaw;
  // B-resident mode: `steps` weight boxes of kBBytes stay in shared memory for the whole kernel; the ring carries A only
  __host__ __device__ static constexpr uint32_t bres_bytes(int steps) { return (uint32_t(steps) * kBBytes + 1023u) / 1024u * 1024u; }
  __host__ __device__ static constexpr int bres_stages(int steps) {
    const int s = (int(kSmemBudget) - int(bres_bytes(steps))) / int(kABytes);
    return s > kMaxStages ? kMaxStages : s;
  }
  static constexpr uint32_t kSwizzleBytes = BLOCK_K * 2;  // 32 / 64 / 128: one smem row of an operand tile
  static constexpr uint32_t kSbo = 8 * kSwizzleBytes;
  static constexpr uint32_t kBarBytes = 256;              // mbarriers
  static constexpr size_t kSmemBytes = size_t(kSmemBudget) + 1024 /*align*/ + kBarBytes;
  static_assert(kStages >= 2, "pipeline needs at least two stages");
  static_assert(!HALO || BLOCK_K >= 32, "halo reuse: rows of 64 or 128 bytes");
};

// bias (+ SiLU) of one accumulator.  SiLU(x) = h + h*tanh(h) with h = x/2 = fma(acc, 0.5, b/2): `b` holds b/2 for SiLU
// layers, so bias add and halving are one FFMA (bit-identical: scaling by 0.5 is exact) — one MUFU op per element.
__device__ __forceinline__ float bias_act(float a, float b, bool silu) {
  if (!silu) return a + b;
  const float h = fmaf(a, 0.5f, b);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}

// exact n / d for any 32-bit n with a precomputed (multiplier, shift) pair (host: fast_div_for)
__device__ __forceinline__ uint32_t fast_div(uint32_t n, uint32_t mul, uint32_t shr) {
  const uint32_t t = __umulhi(n, mul);
  return (t + ((n - t) >> (shr ? 1 : 0))) >> (shr ? shr - 1 : 0);
}

// where accumulator row m of tile (mt, n0) goes: null pointers for halo / out-of-range rows
struct RowOut {
  __nv_bfloat16* out;       // bf16 output (first of the 4 upsampled copies)
  float* f32;               // fp32 pixel-major output (Detect heads)
  const __nv_bfloat16* res; // residual
};

__device__ __forceinline__ RowOut row_out(const ConvTcArgs& p, int mt, int n0, int m) {
  RowOut o{nullptr, nullptr, nullptr};
  bool valid;
  int img, oy, ox;  // image, UNPADDED output coordinates
  if (p.mode == 0) {
    const int row = mt * kBlockM + m;
    const int plane = p.hp * p.wp;
    img = static_cast<int>(fast_div(static_cast<uint32_t>(row), p.plane_mul, p.plane_shr));
    const int rem = row - img * plane;
    const int yp = static_cast<int>(fast_div(static_cast<uint32_t>(rem), p.wp_mul, p.wp_shr)), xp = rem - yp * p.wp;
    valid = row < p.rows_total && yp >= 1 && yp <= p.hp - 2 && xp >= 1 && xp <= p.wp - 2;
    oy = yp - 1;
    ox = xp - 1;
  } else {
    const int per_img = p.tiles_w * p.tiles_h;
    img = mt / per_img;
    const int t = mt - img * per_img;
    const int ty = m / p.tw, tx = m - ty * p.tw;
    oy = (t / p.tiles_w) * p.th + ty;
    ox = (t % p.tiles_w) * p.tw + tx;
    valid = ty < p.th && oy < p.ho && ox < p.wo;
  }
  if (!valid) return o;
  const int oh = p.mode == 0 ? p.hp - 2 : p.ho;  // conv-output height/width (unpadded)
  const int ow = p.mode == 0 ? p.wp - 2 : p.wo;
  long long conv_row = (static_cast<long long>(img) * (oh + 2) + oy + 1) * (ow + 2) + ox + 1;
  if (p.phase)  // one parity class of a transposed stride-2 conv: (oy, ox) -> (2 oy + a, 2 ox + b) of the 2x grid
    conv_row = (static_cast<long long>(img) * (2 * oh + 2) + 2 * oy + p.ph_a + 1) * (2 * ow + 2) + 2 * ox + p.ph_b + 1;
  if (p.res) o.res = p.res + conv_row * p.res_ld + p.res_coff + n0;
  if (p.out_f32) {
    o.f32 = p.out_f32 + ((static_cast<long long>(img) * oh + oy) * ow + ox) * p.out_f32_ld + n0;
  } else if (p.upsample) {
    const long long r00 = (static_cast<long long>(img) * (2 * oh + 2) + 2 * oy + 1) * (2 * ow + 2) + 2 * ox + 1;
    o.out = p.out + r00 * p.out_ld + p.out_coff + n0;
  } else {
    o.out = p.out + conv_row * p.out_ld + p.out_coff + n0;
  }
  return o;
}

template <int BLOCK_N, int BLOCK_K, bool HALO>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const ConvTcArgs p) {
  using C = Cfg<BLOCK_N, BLOCK_K, HALO>;
  const int STAGES = p.stages;
  const bool bres = p.bres != 0;
  constexpr uint32_t kBStage = C::kTaps * C::kBBytes;  // B bytes per stage (ring mode)
  const int b_steps = p.taps * p.kblocks;             // weight boxes of one N tile (resident mode keeps them all)

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);  // swizzled TMA / wgmma tiles need 1 KB alignment
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * C::kABytes;  // ring of B stages, or the resident weight tile
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_b + (bres ? C::bres_bytes(b_steps) : uint32_t(STAGES) * kBStage));
  uint64_t* empty_bar = full_bar + C::kMaxStages;
  uint64_t* bres_bar = empty_bar + C::kMaxStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    mbar_init(bres_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  // everything above touched only shared memory and the kernel parameters: it may run while the previous kernel of the
  // stream drains.  From here on global memory is read and written.
  pdl_wait();
  pdl_trigger();

  const int total_tiles = p.m_tiles * p.n_tiles;
  const int k_iters = HALO ? 3 * p.kblocks : p.taps * p.kblocks;  // HALO: one iteration = one filter row of one k-block

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------------ TMA producer
    // The WHOLE warp runs the loop in warp-uniform control flow and one elected lane issues the copies: with a single
    // active thread (if (lane == 0)) the compiler cannot prove that the TMA operands are uniform.
    uint32_t stage = 0, phase = 0;
    if (bres && int(blockIdx.x) < total_tiles && elect_one()) {
      // resident weights (single N tile): every (k-block, tap) box once, all credited to one barrier
      mbar_expect_tx(bres_bar, uint32_t(b_steps) * C::kBBytes);
      for (int st = 0; st < b_steps; ++st) {
        const int kb = st / p.taps, tap = st - kb * p.taps;
        tma_load_2d(smem_b + st * C::kBBytes, &map_b, bres_bar, (p.custom_taps ? p.tap_wcol[tap] : tap) * p.cin + kb * BLOCK_K, 0);
      }
    }
    __syncwarp();
    // loop-invariant parameters in registers, and one copy of the tile loop per addressing mode
    const int n_tiles = p.n_tiles, wp = p.wp, cin = p.cin, a_coff = p.a_coff, a_ld = p.a_ld;
    const int taps_it = HALO ? 3 : p.taps;  // HALO: tap = filter row r
    const bool xpair = p.xpair != 0, nine = p.taps == 9, custom = p.custom_taps != 0;
    const int taps_w = xpair ? 2 : 3;       // taps per filter row
    const uint32_t stage_tx = p.a_tx_bytes + (bres ? 0u : kBStage);
    auto run = [&](auto mode_tag) {
      constexpr int MODE = decltype(mode_tag)::value;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = tile % n_tiles;
        const int mt = tile / n_tiles;
        const int n0 = nt * BLOCK_N;
        int row0 = 0, img = 0, oh0 = 0, ow0 = 0;
        if (MODE == 0) {
          row0 = mt * kBlockM;
        } else {
          const int per_img = p.tiles_w * p.tiles_h;
          img = mt / per_img;
          const int t = mt - img * per_img;
          oh0 = (t / p.tiles_w) * p.th;
          ow0 = (t % p.tiles_w) * p.tw;
        }
        // (k-block kb, tap) advance incrementally: a runtime division per stage was a quarter of the loop
        int kb = 0, tap = 0, r = 0, s = 0;  // tap = r * taps_w + s  (1x1: always 0)
        for (int it = 0; it < k_iters; ++it) {
          mbar_wait(&empty_bar[stage], phase ^ 1u, p.err, 1);
          if (elect_one()) {
            uint8_t* a_dst = smem_a + stage * C::kABytes;
            uint8_t* b_dst = smem_b + stage * kBStage;
            const int kcol = kb * BLOCK_K;
            // flat mode: the tap's A box is the tile's pixel rows shifted by (r-1)*wp + (s-1) (HALO: a whole filter row)
            const int shift = HALO ? (tap - 1) * wp - 1 : (custom ? p.tap_shift[tap] : (nine ? (r - 1) * wp + (s - 1) : 0));
            // patch mode: filter row r, column s.  x-paired weights (stride 2, in_ld == c_in): one box covers the two
            // horizontally adjacent taps (r, 2s) and (r, 2s+1), which are contiguous channels of the parity view
            const int c0 = xpair ? a_coff : (s & 1) * a_ld + a_coff + kcol;
            const int c1 = xpair ? s : (s >> 1);
            const int bcol = (HALO ? tap * 3 : (custom ? p.tap_wcol[tap] : tap)) * cin + kcol;
            mbar_expect_tx(&full_bar[stage], stage_tx);
            if (MODE == 0)
              tma_load_2d(a_dst, &map_a, &full_bar[stage], a_coff + kcol, row0 + shift);
            else
              tma_load_5d(a_dst, &map_a, &full_bar[stage], c0, ow0 + c1, r & 1, oh0 + (r >> 1), img);
            if (!bres) {
#pragma unroll
              for (uint32_t t = 0; t < C::kTaps; ++t)
                tma_load_2d(b_dst + t * C::kBBytes, &map_b, &full_bar[stage], bcol + int(t) * cin, n0);
            }
          }
          __syncwarp();
          if (++stage == uint32_t(STAGES)) {
            stage = 0;
            phase ^= 1u;
          }
          if (++s == taps_w) {
            s = 0;
            ++r;
          }
          if (++tap == taps_it) {
            tap = 0;
            r = 0;
            s = 0;
            ++kb;
          }
        }
      }
    };
    if (p.mode == 0)
      run(std::integral_constant<int, 0>{});
    else
      run(std::integral_constant<int, 1>{});
  } else {
    // ------------------------------------------------------------------ consumers: wgmma + epilogue (warpgroups 0, 1)
    const int wg = warp >> 2;                             // tile rows [64 wg, 64 wg + 64)
    const int m0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's accumulator rows: m0 and m0 + 8
    const int cq = 2 * (lane & 3);                        // ... and columns 8 j + cq, 8 j + cq + 1
    constexpr uint32_t kDescHi = wgmma_desc_hi(C::kSbo, C::kSwizzleBytes);
    const uint32_t a_base = smem_u32(smem_a) + uint32_t(wg) * 64u * C::kSwizzleBytes;
    const uint32_t b_base = smem_u32(smem_b);
    uint32_t stage = 0, phase = 0;
    if (bres && int(blockIdx.x) < total_tiles) mbar_wait(bres_bar, 0, p.err, 6);  // resident weights have landed
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      float acc[BLOCK_N / 2];
      uint32_t prev = 0;
      for (int it = 0; it < k_iters; ++it) {
        mbar_wait(&full_bar[stage], phase, p.err, 3);  // TMA bytes have landed
        const uint32_t a_st = a_base + stage * C::kABytes;
        const uint32_t b_st = b_base + (bres ? uint32_t(it) : stage) * kBStage;
        wgmma_fence();
#pragma unroll
        for (uint32_t t = 0; t < C::kTaps; ++t) {
#pragma unroll
          for (int k = 0; k < BLOCK_K / 16; ++k) {
            // HALO: tap t reads the A box shifted by t pixel rows (start address off the swizzle pattern)
            const uint64_t adesc = wgmma_desc(kDescHi, a_st + t * C::kSwizzleBytes + k * 32);
            const uint64_t bdesc = wgmma_desc(kDescHi, b_st + t * C::kBBytes + k * 32);
            Wgmma<BLOCK_N>::template mma<0, 0>(acc, adesc, bdesc, (it != 0 || t != 0 || k != 0) ? 1u : 0u);
          }
        }
        wgmma_commit();
        // the previous stage's MMAs have completed: its slot may be refilled
        wgmma_wait<1>();
        if (it > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == uint32_t(STAGES)) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      // ---- epilogue straight from the accumulator registers
      const int nt = tile % p.n_tiles, mt = tile / p.n_tiles;
      const int n0 = nt * BLOCK_N;
      const long long up_row_stride = static_cast<long long>(2 * (p.mode == 0 ? p.wp - 2 : p.wo) + 2) * p.out_ld;
      // read from the kernel parameters here rather than kept live through the main loop
      const bool silu = p.act == Y3_ACT_SILU;
      const float bscale = silu ? 0.5f : 1.0f;
      const int reps = p.upsample ? 4 : 1;
      // one row at a time: only that row's three output pointers are live beside the accumulators (N = 256 keeps 128)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const RowOut ro = row_out(p, mt, n0, m0 + 8 * h);
        if (!ro.f32 && !ro.out) continue;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int c = 8 * j + cq;
          if (!p.out_f32 && n0 + c >= p.cout) continue;  // c_out % 32 == 0: a column pair is either inside or outside
          const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + c));
          float x0 = bias_act(acc[4 * j + 2 * h], bscale * b.x, silu);
          float x1 = bias_act(acc[4 * j + 2 * h + 1], bscale * b.y, silu);
          if (ro.f32) {
            *reinterpret_cast<float2*>(ro.f32 + c) = make_float2(x0, x1);
          } else {
            if (ro.res) {
              const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(ro.res + c));
              x0 += f.x;
              x1 += f.y;
            }
            const uint32_t v = pack_bf16x2(x0, x1);
            for (int rep = 0; rep < reps; ++rep)
              *reinterpret_cast<uint32_t*>(ro.out + (rep >> 1) * up_row_stride + (rep & 1) * p.out_ld + c) = v;
          }
        }
      }
    }
  }
}

template <int BLOCK_N, int BLOCK_K, bool HALO = false>
int launch_cfg(const ConvTcPlan& plan, cudaStream_t stream) {
  using C = Cfg<BLOCK_N, BLOCK_K, HALO>;
  auto kern = conv_tc_kernel<BLOCK_N, BLOCK_K, HALO>;
  static bool attr_set = false;  // benign race: idempotent attribute
  if (!attr_set) {
    Y3_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(C::kSmemBytes)));
    attr_set = true;
  }
  ConvTcArgs args = plan.args;
  args.bres = plan.bres;
  args.stages = plan.bres ? C::bres_stages(args.taps * args.kblocks) : C::kStages;
  if (args.stages < 3) {  // not enough ring left beside the resident weights: fall back to streaming them
    args.bres = 0;
    args.stages = C::kStages;
  }
  // the kernel parks at pdl_wait() after its prologue (y3_common.cuh)
  Y3_CHECK_CUDA(launch_pdl(kern, dim3(plan.grid), dim3(kThreads), C::kSmemBytes, stream, plan.map_a, plan.map_b, args));
  return Y3_OK;
}

int pick_block_n(int cout) { return cout <= 32 ? 32 : (cout <= 64 ? 64 : (cout <= 128 ? 128 : 256)); }

}  // namespace

int conv_tc_launch(const ConvTcPlan& plan, cudaStream_t stream) {
#define Y3_DISPATCH_K(BN)                                              \
  switch (plan.block_k) {                                              \
    case 64: return launch_cfg<BN, 64>(plan, stream);                  \
    case 32: return launch_cfg<BN, 32>(plan, stream);                  \
    case 16: return launch_cfg<BN, 16>(plan, stream);                  \
  }                                                                    \
  break;
  if (plan.halo) {  // stride-1 3x3: K = 64 with N <= 128, K = 32 (c_in = 32 layers, 64-byte rows) with N <= 64
    if (plan.block_k == 64) {
      if (plan.block_n == 128) return launch_cfg<128, 64, true>(plan, stream);
      if (plan.block_n == 64) return launch_cfg<64, 64, true>(plan, stream);
      if (plan.block_n == 32) return launch_cfg<32, 64, true>(plan, stream);
    } else if (plan.block_k == 32) {
      if (plan.block_n == 64) return launch_cfg<64, 32, true>(plan, stream);
      if (plan.block_n == 32) return launch_cfg<32, 32, true>(plan, stream);
    }
    return set_error(Y3_ERR_BAD_ARG, "conv_tc: no halo kernel for tile N=%d K=%d", plan.block_n, plan.block_k);
  }
  switch (plan.block_n) {
    case 32: Y3_DISPATCH_K(32)
    case 64: Y3_DISPATCH_K(64)
    case 128: Y3_DISPATCH_K(128)
    case 256: Y3_DISPATCH_K(256)
  }
#undef Y3_DISPATCH_K
  return set_error(Y3_ERR_BAD_ARG, "conv_tc: no kernel for tile N=%d K=%d", plan.block_n, plan.block_k);
}

// Y3_CONV_HALO=0 disables the halo-reuse A path (A/B measurements).
static bool halo_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("Y3_CONV_HALO");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

// Y3_CONV_BRES=0 streams the weights through the ring everywhere (A/B measurements).
static bool bres_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("Y3_CONV_BRES");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

// Layer 1 of yolov3 (32 -> 64, stride 2 at 640x640) moved 64-byte rows through 9 five-dimensional TMA boxes per tile
// and ran at 0.2 PFLOP/s; paired, the same tile is 6 boxes of full 128-byte rows and one K = 64 MMA group per box.
// (mul, shr) such that n / d == (t + ((n - t) >> 1)) >> (shr - 1), t = umulhi(n, mul), for every 32-bit n (d >= 2);
// d == 1: mul = 0, shr = 0 (identity).  Granlund-Montgomery round-up method.
static void fast_div_for(uint32_t d, uint32_t* mul, uint32_t* shr) {
  if (d <= 1) {
    *mul = 0;
    *shr = 0;
    return;
  }
  uint32_t l = 0;
  while ((1ull << l) < d) ++l;
  *mul = static_cast<uint32_t>(((1ull << 32) * ((1ull << l) - d)) / d + 1);
  *shr = l;
}

static bool conv_prefers_xpair(const y3_conv_desc& d) {
  return d.ksize == 3 && d.stride == 2 && (d.c_in == 32 || d.c_in == 16) && d.in_ld == d.c_in && d.in_coff == 0;
}

// select_only: tile / mode selection without encoding the tensor maps (y3_conv_plan: host-side tests of the heuristics)
int conv_tc_prepare(const y3_conv_desc& d, ConvTcPlan* plan, bool select_only, const ConvTcExtra* extra) {
  Y3_REQUIRE(d.n > 0 && d.h > 0 && d.w > 0, "conv: empty shape");
  Y3_REQUIRE((d.ksize == 1 && d.stride == 1) || (d.ksize == 3 && (d.stride == 1 || d.stride == 2)),
             "conv: ksize/stride %d/%d unsupported (1x1 s1, 3x3 s1, 3x3 s2)", d.ksize, d.stride);
  Y3_REQUIRE(d.c_in % 16 == 0 && d.c_in >= 16, "conv: c_in=%d must be a multiple of 16", d.c_in);
  Y3_REQUIRE(d.in_ld % 8 == 0 && d.in_coff % 8 == 0 && d.in_coff + d.c_in <= d.in_ld, "conv: bad input slice");
  Y3_REQUIRE(d.in && d.weight && d.bias, "conv: null pointer");
  Y3_REQUIRE((reinterpret_cast<uintptr_t>(d.in) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.weight) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(d.bias) & 15) == 0,
             "conv: pointers must be 16-byte aligned");
  const bool head = d.out_f32 != nullptr;
  if (head) {
    Y3_REQUIRE(d.stride == 1 && !d.upsample && !d.res, "conv: fp32 output supports plain stride-1 convs only");
    Y3_REQUIRE(d.out_f32_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(d.out_f32) & 15) == 0, "conv: bad fp32 output");
  } else {
    Y3_REQUIRE(d.out != nullptr, "conv: null output");
    Y3_REQUIRE(d.c_out % 32 == 0, "conv: c_out=%d must be a multiple of 32", d.c_out);
    Y3_REQUIRE(d.out_ld % 8 == 0 && d.out_coff % 8 == 0 && d.out_coff + d.c_out <= d.out_ld, "conv: bad output slice");
    Y3_REQUIRE((reinterpret_cast<uintptr_t>(d.out) & 15) == 0, "conv: out must be 16-byte aligned");
    if (d.res)
      Y3_REQUIRE(d.res_ld % 8 == 0 && d.res_coff % 8 == 0 && (reinterpret_cast<uintptr_t>(d.res) & 15) == 0,
                 "conv: bad residual slice");
  }
  if (d.stride == 2) Y3_REQUIRE(d.h % 2 == 0 && d.w % 2 == 0, "conv: stride-2 needs even h, w");

  const bool xpair = d.weight_layout == Y3_W_XPAIR;
  if (xpair) Y3_REQUIRE(conv_prefers_xpair(d), "conv: x-paired weights need ksize 3, stride 2, c_in 16|32 == in_ld, in_coff 0");
  else Y3_REQUIRE(d.weight_layout == Y3_W_TAPS, "conv: unknown weight_layout %d", d.weight_layout);
  const int bn = pick_block_n(d.c_out);
  // x-paired: the GEMM sees 3 x 2 taps of 2*c_in channels (the phantom 4th column carries zero weights)
  const int gemm_cin = xpair ? 2 * d.c_in : d.c_in;
  const int bk = gemm_cin % 64 == 0 ? 64 : (gemm_cin % 32 == 0 ? 32 : 16);
  const int cout_pad = (d.c_out + bn - 1) / bn * bn;
  const int taps = extra ? extra->ntaps : (xpair ? 6 : d.ksize * d.ksize);
  const int hp = d.h + 2, wp = d.w + 2;
  if (extra) Y3_REQUIRE(d.stride == 1 && !xpair && !head && !d.upsample && extra->ntaps >= 1 && extra->ntaps <= 4, "conv: bad custom tap list");

  ConvTcArgs& a = plan->args;
  a = ConvTcArgs{};
  plan->block_n = bn;
  plan->block_k = bk;
  a.taps = taps;
  a.kblocks = gemm_cin / bk;
  a.cin = gemm_cin;
  a.xpair = xpair ? 1 : 0;
  a.a_coff = d.in_coff;
  a.a_ld = d.in_ld;
  a.n_tiles = cout_pad / bn;
  a.bias = d.bias;
  a.cout = d.c_out;
  a.act = d.act;
  a.out = static_cast<__nv_bfloat16*>(d.out);
  a.out_ld = d.out_ld;
  a.out_coff = d.out_coff;
  a.upsample = d.upsample;
  a.res = static_cast<const __nv_bfloat16*>(d.res);
  a.res_ld = d.res_ld;
  a.res_coff = d.res_coff;
  a.out_f32 = d.out_f32;
  a.out_f32_ld = d.out_f32_ld;
  a.err = d.err;
  if (head) {
    a.out = nullptr;
    Y3_REQUIRE(d.out_f32_ld >= (d.c_out + pick_block_n(d.c_out) - 1) / pick_block_n(d.c_out) * pick_block_n(d.c_out),
               "conv: out_f32_ld must cover the padded c_out");
  }

  int rc;
  if (d.stride == 1) {
    a.mode = 0;
    a.hp = hp;
    a.wp = wp;
    fast_div_for(static_cast<uint32_t>(hp) * wp, &a.plane_mul, &a.plane_shr);
    fast_div_for(static_cast<uint32_t>(wp), &a.wp_mul, &a.wp_shr);
    const long long rows = static_cast<long long>(d.n) * hp * wp;
    Y3_REQUIRE(rows < (1ll << 31) - 4096, "conv: too many pixels");
    a.rows_total = static_cast<int>(rows);
    a.m_tiles = static_cast<int>((rows + kBlockM - 1) / kBlockM);
    // halo reuse needs >= 2 stages of (17 KB + 3 B tiles): N <= 128 (N = 256 would leave room for one stage)
    plan->halo = (!extra && taps == 9 && ((bk == 64 && bn <= 128) || (bk == 32 && bn <= 64)) && halo_enabled()) ? 1 : 0;
    if (extra) {
      a.custom_taps = 1;
      for (int t = 0; t < extra->ntaps; ++t) {
        a.tap_shift[t] = extra->dr[t] * wp + extra->ds[t];
        a.tap_wcol[t] = extra->wcol[t];
      }
      a.phase = extra->phase;
      a.ph_a = extra->ph_a;
      a.ph_b = extra->ph_b;
    }
    const uint32_t a_rows = plan->halo ? kBlockM + 2 : kBlockM;
    a.a_tx_bytes = a_rows * bk * 2;
    const uint64_t dims[2] = {static_cast<uint64_t>(d.in_ld), static_cast<uint64_t>(rows)};
    const uint64_t strides[2] = {0, static_cast<uint64_t>(d.in_ld) * 2};
    const uint32_t box[2] = {static_cast<uint32_t>(bk), a_rows};
    rc = select_only ? Y3_OK : encode_tensor_map_bf16(&plan->map_a, d.in, 2, dims, strides, box, bk * 2);
    if (rc) return rc;
  } else {
    plan->halo = 0;
    a.mode = 1;
    a.ho = d.h / 2;
    a.wo = d.w / 2;
    // pick the TH x TW (<=128 pixels) output patch that wastes the least MMA rows
    int best_tw = 1, best_th = 1;
    long long best_tiles = -1;
    for (int tw = 1; tw <= 128 && tw <= 256; ++tw) {
      const int th = 128 / tw;
      if (th < 1) break;
      const int thc = th > a.ho ? a.ho : th;
      const long long tiles = static_cast<long long>((a.wo + tw - 1) / tw) * ((a.ho + thc - 1) / thc);
      if (best_tiles < 0 || tiles < best_tiles || (tiles == best_tiles && tw > best_tw)) {
        best_tiles = tiles;
        best_tw = tw;
        best_th = thc;
      }
    }
    a.tw = best_tw;
    a.th = best_th;
    a.tiles_w = (a.wo + a.tw - 1) / a.tw;
    a.tiles_h = (a.ho + a.th - 1) / a.th;
    a.m_tiles = d.n * a.tiles_w * a.tiles_h;
    a.a_tx_bytes = static_cast<uint32_t>(a.tw) * a.th * bk * 2;
    const uint64_t ld = static_cast<uint64_t>(d.in_ld);
    const uint64_t dims[5] = {2 * ld, static_cast<uint64_t>(wp / 2), 2, static_cast<uint64_t>(hp / 2),
                              static_cast<uint64_t>(d.n)};
    const uint64_t strides[5] = {0, 2 * ld * 2, static_cast<uint64_t>(wp) * ld * 2, 2ull * wp * ld * 2,
                                 static_cast<uint64_t>(hp) * wp * ld * 2};
    const uint32_t box[5] = {static_cast<uint32_t>(bk), static_cast<uint32_t>(a.tw), 1, static_cast<uint32_t>(a.th), 1};
    rc = select_only ? Y3_OK : encode_tensor_map_bf16(&plan->map_a, d.in, 5, dims, strides, box, bk * 2);
    if (rc) return rc;
  }
  {
    const uint64_t ktot = static_cast<uint64_t>(extra ? d.ksize * d.ksize : taps) * gemm_cin;  // the whole weight matrix
    const uint64_t dims[2] = {ktot, static_cast<uint64_t>(cout_pad)};
    const uint64_t strides[2] = {0, ktot * 2};
    const uint32_t box[2] = {static_cast<uint32_t>(bk), static_cast<uint32_t>(bn)};
    rc = select_only ? Y3_OK : encode_tensor_map_bf16(&plan->map_b, d.weight, 2, dims, strides, box, bk * 2);
    if (rc) return rc;
  }
  {
    // resident weights: one N tile whose (taps x k-blocks) boxes fit beside a useful A ring.  The TMA unit's row rate
    // (not bytes) bounds the thin layers, and re-fetching the same <= 96 KB of weights for every M tile was most of it.
    const long long b_bytes = static_cast<long long>(taps) * a.kblocks * bn * bk * 2;
    plan->bres = (a.n_tiles == 1 && b_bytes <= 96 * 1024 && bres_enabled()) ? 1 : 0;
  }
  const int sms = num_sms();
  const long long total = static_cast<long long>(a.m_tiles) * a.n_tiles;
  plan->grid = static_cast<int>(total < sms ? total : sms);
  return Y3_OK;
}

}  // namespace y3

extern "C" int y3_conv_plan(const y3_conv_desc* d, y3_conv_plan_info* out) {
  if (!d || !out) return y3::set_error(Y3_ERR_BAD_ARG, "conv_plan: null argument");
  y3::ConvTcPlan plan;
  int rc = y3::conv_tc_prepare(*d, &plan, true);
  if (rc) return rc;
  out->block_n = plan.block_n;
  out->block_k = plan.block_k;
  out->halo = plan.halo;
  out->resident_weights = plan.bres;
  out->xpair = plan.args.xpair;
  out->m_tiles = plan.args.m_tiles;
  out->n_tiles = plan.args.n_tiles;
  out->k_blocks = plan.args.kblocks;
  out->grid = plan.grid;
  return Y3_OK;
}

extern "C" int y3_conv_weight_layout(const y3_conv_desc* d) {
  if (!d) return y3::set_error(Y3_ERR_BAD_ARG, "conv: null descriptor");
  static int enabled = -1;  // Y3_CONV_XPAIR=0 keeps the plain tap-major layout everywhere (A/B measurements)
  if (enabled < 0) {
    const char* e = getenv("Y3_CONV_XPAIR");
    enabled = (e && e[0] == '0') ? 0 : 1;
  }
  return (enabled && y3::conv_prefers_xpair(*d)) ? Y3_W_XPAIR : Y3_W_TAPS;
}

extern "C" int y3_conv_cout_pad(int32_t c_out) {
  const int bn = y3::pick_block_n(c_out);
  return (c_out + bn - 1) / bn * bn;
}

// Input gradient of a stride-2 3x3 conv as FOUR parity-class convolutions on the un-stuffed dy (transposed convolution by
// phases): dx[2i+a, 2j+b] = sum over the taps (r, s) with r = a+1 (mod 2), s = b+1 (mod 2) of dy[i + (a && r == 0), j + (b && s == 0)]
// * W[r, s]^T — 1, 2, 2 and 4 taps.  The stride-1 convolution of the zero-stuffed dy it replaces multiplied 75 % zeros.
extern "C" int y3_conv_dgrad_s2(const y3_conv_desc* d, y3_stream_t stream) {
  if (!d) return y3::set_error(Y3_ERR_BAD_ARG, "conv: null descriptor");
  Y3_REQUIRE(d->ksize == 3 && d->stride == 1 && !d->upsample && !d->out_f32 && d->weight_layout == Y3_W_TAPS,
             "dgrad_s2: describe the 3x3 transposed conv on dy's own grid (stride 1 in the descriptor), bf16 output");
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      y3::ConvTcExtra ex{};
      ex.phase = 1;
      ex.ph_a = a;
      ex.ph_b = b;
      const int rs[2][2] = {{1, -1}, {0, 2}};  // taps r of parity class a (second entry -1: none)
      for (int ri = 0; ri < 2; ++ri) {
        const int r = rs[a][ri];
        if (r < 0) continue;
        for (int si = 0; si < 2; ++si) {
          const int s = rs[b][si];
          if (s < 0) continue;
          const int t = ex.ntaps++;
          ex.dr[t] = (a == 1 && r == 0) ? 1 : 0;
          ex.ds[t] = (b == 1 && s == 0) ? 1 : 0;
          ex.wcol[t] = (2 - r) * 3 + (2 - s);  // the dgrad pack stores W[r, s]^T at the flipped tap
        }
      }
      y3::ConvTcPlan plan;
      int rc = y3::conv_tc_prepare(*d, &plan, false, &ex);
      if (rc) return rc;
      rc = y3::conv_tc_launch(plan, static_cast<cudaStream_t>(stream));
      if (rc) return rc;
    }
  return Y3_OK;
}

extern "C" int y3_conv_bn_act_fwd(const y3_conv_desc* d, y3_stream_t stream) {
  if (!d) return y3::set_error(Y3_ERR_BAD_ARG, "conv: null descriptor");
  y3::ConvTcPlan plan;
  int rc = y3::conv_tc_prepare(*d, &plan);
  if (rc) return rc;
  return y3::conv_tc_launch(plan, static_cast<cudaStream_t>(stream));
}
