// yolov3_b200 — the optimizer step of the training loop as three bandwidth-bound launches over ONE flat parameter buffer
// (SURVEY §8(f) row f3).  Replaces, for the reference's train.py:411-421 + utils/torch_utils.py:207-237:
//   scaler.unscale_/clip_grad_norm_(model.parameters(), max_norm=10.0)   -> grad_sumsq (two-stage, bit-reproducible) + the
//                                                                           clip coefficient applied inside the update
//   optimizer.step()  (SGD, momentum 0.937, nesterov, 3 param groups:      -> sgd_step: p, g, momentum buffer streamed once;
//                      conv/linear weights with decay, BN weights, biases)    group id per 256-element chunk
//   ema.update(model) (ModelEMA: v = d*v + (1-d)*p over the state_dict)   -> fused into the same pass (and over the buffers)
//   optimizer.step()  (Adam / AdamW, train.py --optimizer, same groups)  -> adam_step: p, g, exp_avg, exp_avg_sq streamed once,
//                                                                           bias corrections per parameter from a host table
// All hyper-parameters are read from a small DEVICE array so the launches are CUDA-graph capturable while the scheduler
// changes lr / momentum every iteration (warm-up: train.py:364-375).
#include "y3_common.cuh"
#include "y3_internal.h"

namespace y3 {
namespace {

constexpr int kChunk = 256;  // elements per group-map entry; every parameter's slot in the flat buffer is a multiple of it

// first stage: partial[b] = sum of g^2 over block b's grid-stride range (fixed association order per block).  group
// (optional): the chunks it does not tag trainable (< 3) are left out — frozen parameters, whose slot of g may hold anything,
// count in the clip norm no more than they do in clip_grad_norm_, which skips a parameter whose .grad is None
__global__ void __launch_bounds__(256) sumsq_partial_kernel(const float* __restrict__ g, const uint8_t* __restrict__ group,
                                                            long long n4, float* __restrict__ partial) {
  pdl_entry();
  float acc = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (group && group[(i * 4) / kChunk] >= 3) continue;
    const float4 v = __ldg(reinterpret_cast<const float4*>(g) + i);
    acc = fmaf(v.x, v.x, acc);
    acc = fmaf(v.y, v.y, acc);
    acc = fmaf(v.z, v.z, acc);
    acc = fmaf(v.w, v.w, acc);
  }
  __shared__ float sh[256];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}
// second stage (one block): out[0] = sum_b partial[b], pairwise in a fixed order
__global__ void __launch_bounds__(256) sumsq_final_kernel(const float* __restrict__ partial, int nblk, float* __restrict__ out) {
  pdl_entry();
  __shared__ float sh[256];
  float acc = 0.f;
  for (int b = threadIdx.x; b < nblk; b += 256) acc += partial[b];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = sh[0];
}

// hp (device): [0..2] lr of groups 0/1/2, [3..5] weight decay, [6] momentum, [7] nesterov (0/1), [8] max_norm (0 = no clip),
//              [9] ema decay d of this update (ignored when ema == nullptr), [10] gradient pre-scale (1/world for a SUM
//              all-reduce, 1 otherwise)
__global__ void __launch_bounds__(256) sgd_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                       float* __restrict__ ema, const uint8_t* __restrict__ group,
                                                       long long n4, const float* __restrict__ hp,
                                                       const float* __restrict__ gsumsq) {
  pdl_entry();
  const float mom = hp[6], nesterov = hp[7], max_norm = hp[8], d = hp[9], gscale = hp[10];
  float clip = gscale;
  if (max_norm > 0.f) {
    // torch.nn.utils.clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), clamped to 1 (the norm is of the scaled grads)
    const float total = sqrtf(gsumsq[0]) * gscale;
    const float coef = max_norm / (total + 1e-6f);
    clip = gscale * (coef < 1.f ? coef : 1.f);
  }
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int grp = group[(i * 4) / kChunk];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    if (grp < 3) {  // trainable; a frozen parameter (G_FROZEN in the map) keeps p and its momentum, and still takes the EMA
      const float lr = hp[grp], wd = hp[3 + grp];
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g) + i);
      float4 mv = reinterpret_cast<float4*>(m)[i];
      float pe[4] = {pv.x, pv.y, pv.z, pv.w}, ge[4] = {gv.x, gv.y, gv.z, gv.w}, me[4] = {mv.x, mv.y, mv.z, mv.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        // torch.optim.SGD (dampening 0): d_p = g + wd*p; buf = mom*buf + d_p; d_p = nesterov ? d_p + mom*buf : buf; p -= lr*d_p
        float dp = fmaf(wd, pe[k], ge[k] * clip);
        me[k] = fmaf(mom, me[k], dp);
        dp = nesterov != 0.f ? fmaf(mom, me[k], dp) : me[k];
        pe[k] = fmaf(-lr, dp, pe[k]);
      }
      pv = make_float4(pe[0], pe[1], pe[2], pe[3]);
      reinterpret_cast<float4*>(p)[i] = pv;
      reinterpret_cast<float4*>(m)[i] = make_float4(me[0], me[1], me[2], me[3]);
    }
    if (ema) {  // ModelEMA.update over every floating-point state_dict entry (parameters AND BatchNorm buffers)
      float4 ev = reinterpret_cast<float4*>(ema)[i];
      ev.x = fmaf(d, ev.x - pv.x, pv.x);  // d*e + (1-d)*p
      ev.y = fmaf(d, ev.y - pv.y, pv.y);
      ev.z = fmaf(d, ev.z - pv.z, pv.z);
      ev.w = fmaf(d, ev.w - pv.w, pv.w);
      reinterpret_cast<float4*>(ema)[i] = ev;
    }
  }
}

// This file is compiled with --use_fast_math, which the SGD step's numbers are pinned to.  The Adam step restates torch's
// CUDA arithmetic instead (IEEE division and square root, no flush of subnormals, a*b+c contracted to one fma as nvcc
// contracts it in torch's foreach kernels), so it spells those operations as PTX without .ftz / .approx.
__device__ __forceinline__ float f_mul(float a, float b) { float r; asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float f_add(float a, float b) { float r; asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float f_sub(float a, float b) { float r; asm("sub.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float f_div(float a, float b) { float r; asm("div.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float f_sqrt(float a) { float r; asm("sqrt.rn.f32 %0, %1;" : "=f"(r) : "f"(a)); return r; }
__device__ __forceinline__ float f_fma(float a, float b, float c) {
  float r;
  asm("fma.rn.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
  return r;
}

// hp (device): [0..2] weight decay added to the gradient (Adam) of groups 0/1/2, [3..5] decoupled decay factor
//              fp32(1 - lr*wd) (AdamW; 1 = none), [8] max_norm, [9] ema decay d, [10] gradient pre-scale (as sgd_step),
//              [12..14] 1 - beta1, [15..17] beta2, [18..20] 1 - beta2, [21..23] eps;
// tab (device): per parameter slot k, {step_size_k = -lr / (1 - beta1^t_k), sqrt(1 - beta2^t_k)} from the host, where t_k is
//              the slot's own step count; slot[c] = slot of chunk c (trainable chunks only)
// Per element, torch.optim.adam._multi_tensor_adam (non-capturable) in its order: clip, weight decay, moments, update.
__global__ void __launch_bounds__(256) adam_step_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                        float* __restrict__ m, float* __restrict__ v, float* __restrict__ ema,
                                                        const uint8_t* __restrict__ group, const int32_t* __restrict__ slot,
                                                        long long n4, const float* __restrict__ hp,
                                                        const float* __restrict__ tab, const float* __restrict__ gsumsq) {
  pdl_entry();
  const float d = hp[9], max_norm = hp[8], gscale = hp[10];
  // sgd_step_kernel's clip factor in torch's own fp32 operations (clip_grads_with_norm_: coef = (1 / (total_norm + 1e-6)) * max_norm,
  // clamped to 1): Adam's step is ill-conditioned where the decayed gradient nearly cancels, so a coefficient a few ulp away
  // from torch's moves those parameters beyond rounding; given the same norm, this one is torch's bit for bit
  float clip = gscale;
  if (max_norm > 0.f) {
    const float coef = f_mul(f_div(1.f, f_add(f_mul(f_sqrt(gsumsq[0]), gscale), 1e-6f)), max_norm);
    clip = f_mul(gscale, coef < 1.f ? coef : 1.f);
  }
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long c = (i * 4) / kChunk;
    const int grp = group[c];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    if (grp < 3) {  // trainable; a frozen parameter keeps p, m, v (and its step count, on the host), and still takes the EMA
      const int k = slot[c];
      const float step_size = tab[2 * k], bc2_sqrt = tab[2 * k + 1];
      const float wd = hp[grp], decay = hp[3 + grp], w1 = hp[12 + grp], beta2 = hp[15 + grp], omb2 = hp[18 + grp],
                  eps = hp[21 + grp];
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g) + i);
      float4 mv = reinterpret_cast<float4*>(m)[i];
      float4 vv = reinterpret_cast<float4*>(v)[i];
      float pe[4] = {pv.x, pv.y, pv.z, pv.w}, ge[4] = {gv.x, gv.y, gv.z, gv.w};
      float me[4] = {mv.x, mv.y, mv.z, mv.w}, ve[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float gk = f_mul(ge[e], clip);
        if (wd != 0.f) gk = f_fma(wd, pe[e], gk);          // _foreach_add(grads, params, alpha=wd)
        if (decay != 1.f) pe[e] = f_mul(pe[e], decay);     // _foreach_mul_(params, 1 - lr*wd)
        // _foreach_lerp_(exp_avgs, grads, 1 - beta1): at::lerp's two forms, chosen by |weight| < 0.5
        me[e] = w1 < 0.5f ? f_fma(w1, f_sub(gk, me[e]), me[e]) : f_sub(gk, f_mul(f_sub(gk, me[e]), f_sub(1.f, w1)));
        ve[e] = f_fma(omb2, f_mul(gk, gk), f_mul(ve[e], beta2));  // _foreach_mul_(beta2), _foreach_addcmul_(g, g, 1 - beta2)
        const float denom = f_add(f_div(f_sqrt(ve[e]), bc2_sqrt), eps);
        pe[e] = f_fma(step_size, f_div(me[e], denom), pe[e]);  // _foreach_addcdiv_(params, exp_avgs, denom, step_size)
      }
      pv = make_float4(pe[0], pe[1], pe[2], pe[3]);
      reinterpret_cast<float4*>(p)[i] = pv;
      reinterpret_cast<float4*>(m)[i] = make_float4(me[0], me[1], me[2], me[3]);
      reinterpret_cast<float4*>(v)[i] = make_float4(ve[0], ve[1], ve[2], ve[3]);
    }
    if (ema) {  // as in sgd_step_kernel
      float4 ev = reinterpret_cast<float4*>(ema)[i];
      ev.x = fmaf(d, ev.x - pv.x, pv.x);
      ev.y = fmaf(d, ev.y - pv.y, pv.y);
      ev.z = fmaf(d, ev.z - pv.z, pv.z);
      ev.w = fmaf(d, ev.w - pv.w, pv.w);
      reinterpret_cast<float4*>(ema)[i] = ev;
    }
  }
}

int blocks_for(long long n4) {
  long long b = (n4 + 255) / 256;
  const long long cap = 8ll * num_sms();
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace
}  // namespace y3

extern "C" int32_t y3_sumsq_blocks(void) { return 1024; }

extern "C" int y3_grad_sumsq(const float* g, const uint8_t* group, int64_t n, float* partial, float* out, y3_stream_t stream_) {
  Y3_REQUIRE(g && partial && out && n > 0 && n % 4 == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0,
             "grad_sumsq: n must be a multiple of 4, g 16-byte aligned");
  Y3_REQUIRE(!group || n % y3::kChunk == 0, "grad_sumsq: with a group map n must be a multiple of 256");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int nblk = y3_sumsq_blocks();  // fixed: the partial sums — and so the result — do not depend on the device
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::sumsq_partial_kernel, dim3(nblk), dim3(256), 0, stream, g, group, n / 4, partial));
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::sumsq_final_kernel, dim3(1), dim3(256), 0, stream, partial, nblk, out));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_sgd_step(float* p, const float* g, float* m, float* ema, const uint8_t* group, int64_t n, const float* hp_dev,
                           const float* gsumsq, y3_stream_t stream) {
  Y3_REQUIRE(p && g && m && group && hp_dev && n > 0 && n % y3::kChunk == 0, "sgd_step: n must be a multiple of 256");
  Y3_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
               reinterpret_cast<uintptr_t>(ema)) & 15) == 0, "sgd_step: buffers must be 16-byte aligned");
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::sgd_step_kernel, dim3(y3::blocks_for(n / 4)), dim3(256), 0, static_cast<cudaStream_t>(stream), p, g, m, ema, group, n / 4, hp_dev,
                                                                                            gsumsq));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}

extern "C" int y3_adam_step(float* p, const float* g, float* m, float* v, float* ema, const uint8_t* group, const int32_t* slot,
                            int64_t n, const float* hp_dev, const float* tab_dev, const float* gsumsq, y3_stream_t stream) {
  Y3_REQUIRE(p && g && m && v && group && slot && hp_dev && tab_dev && n > 0 && n % y3::kChunk == 0,
             "adam_step: n must be a multiple of 256");
  Y3_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
               reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(ema)) & 15) == 0,
             "adam_step: buffers must be 16-byte aligned");
  Y3_CHECK_CUDA(::y3::launch_pdl(y3::adam_step_kernel, dim3(y3::blocks_for(n / 4)), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), p, g, m, v, ema, group, slot, n / 4, hp_dev, tab_dev, gsumsq));
  Y3_CHECK_CUDA(cudaGetLastError());
  return Y3_OK;
}
