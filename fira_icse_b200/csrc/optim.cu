// Adam over ONE flat parameter buffer (the optimizer step of run_model.py:101-109, torch.optim.Adam semantics:
// no weight decay, no amsgrad), one launch for all parameters:
//
//   g' = g / *grad_scale                       (grad_scale: device scalar or NULL -- the data-parallel step divides the
//                                               summed gradients by the global token count here)
//   m  = b1 m + (1 - b1) g' ;  v = b2 v + (1 - b2) g'^2
//   p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)          t = *step (device scalar, already incremented)
//   p16 = bf16(p)                              (the GEMM-operand mirror of the throughput mode; may be NULL)
//   e   = fma(d, e, fl(c * p))                 (ema: exponential moving average of the stored p, may be NULL;
//                                               c = fl(1 - d), fl() = fp32 rounding, fma = one rounding)
//
// Memory-bound: 16 B read + 12 B written per parameter + 2 B mirror = 30 B; with ema 20 B read + 16 B written + 2 B = 38 B.
// 8 parameters per thread, 16-byte accesses.  The EMA is a second instantiation of the kernel: the Adam arithmetic of
// both is the same source, so p, m, v and the mirror do not depend on whether ema is set.
//
// Global-norm gradient clipping (fira_adam_flat_clip, the CLIP instantiations) runs in three launches per step:
//   grad_sumsq     per member buffer: float64 sum of g^2 per CTA -> partials (grid fixed by n alone: 4 B read/param)
//   clip_finalize  one CTA: S = sum of every member's partials in order; norm = sqrt(S) / s; S not finite -> skip the
//                  step (flag 0, skipped += 1); else coef = fl32(min(1, c / (norm + 1e-6))), clipped += (coef < 1), and
//                  every member's step counter += 1
//   adam (CLIP)    reads coef and the flag; a skipped step returns before any store; else g' = fl(fl(g / s) * coef)
// coef == 1 multiplies by 1.0f, so an unclipped step is the same bits as fira_adam_flat.
#include "common.cuh"
#include "fira_b200.h"

namespace {

// clip: the FiraClip state of clip_finalize (include/fira_b200.h), read by the CLIP instantiations only; it is the last
// parameter so that the other instantiations keep their parameter layout
template <bool EMA, bool CLIP>
__global__ void __launch_bounds__(256) adam_flat_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                        float* __restrict__ m, float* __restrict__ v,
                                                        __nv_bfloat16* __restrict__ p16, float* __restrict__ ema,
                                                        long n8, float lr, float b1, float b2, float eps,
                                                        const float* __restrict__ step,
                                                        const float* __restrict__ grad_scale, float ema_decay,
                                                        const double* __restrict__ clip) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  float coef = 1.f;
  if constexpr (CLIP) {
    if (clip[FIRA_CLIP_TAKEN] == 0.0) return;                         // skipped step: nothing is written
    coef = (float)clip[FIRA_CLIP_COEF];                               // already an fp32 value
  }
  const float t = *step;
  const float bc1 = 1.f - powf(b1, t), bc2 = 1.f - powf(b2, t);
  const float step_size = lr / bc1, rsq_bc2 = rsqrtf(bc2);
  const float inv_scale = grad_scale ? 1.f / *grad_scale : 1.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    float pv[8], gv[8], mv[8], vv[8];
    Act<float>::load8(p + i * 8, pv);
    Act<float>::load8(g + i * 8, gv);
    Act<float>::load8(m + i * 8, mv);
    Act<float>::load8(v + i * 8, vv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float gj = gv[j] * inv_scale;
      if constexpr (CLIP) gj = __fmul_rn(gj, coef);
      if constexpr (CLIP) {
        // the lines below, with each multiply-add written as the one fma the compiler forms for it in the other
        // instantiations (left to contraction here, it fuses the other product of m's line and the bits differ)
        mv[j] = __fmaf_rn(mv[j], b1, __fmul_rn(1.f - b1, gj));
        vv[j] = __fmaf_rn(__fmul_rn(1.f - b2, gj), gj, __fmul_rn(b2, vv[j]));
        pv[j] = __fmaf_rn(mv[j] / __fmaf_rn(sqrtf(vv[j]), rsq_bc2, eps), -step_size, pv[j]);
        continue;
      }
      mv[j] = b1 * mv[j] + (1.f - b1) * gj;
      vv[j] = b2 * vv[j] + (1.f - b2) * gj * gj;
      const float denom = sqrtf(vv[j]) * rsq_bc2 + eps;
      pv[j] -= step_size * (mv[j] / denom);
    }
    Act<float>::store8(p + i * 8, pv);
    Act<float>::store8(m + i * 8, mv);
    Act<float>::store8(v + i * 8, vv);
    if (p16) Act<__nv_bfloat16>::store8(p16 + i * 8, pv);
    if constexpr (EMA) {
      const float c = 1.f - ema_decay;
      float ev[8];
      Act<float>::load8(ema + i * 8, ev);
#pragma unroll
      for (int j = 0; j < 8; ++j) ev[j] = __fmaf_rn(ema_decay, ev[j], __fmul_rn(c, pv[j]));
      Act<float>::store8(ema + i * 8, ev);
    }
  }
}

__global__ void __launch_bounds__(256) cast_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long n8) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    float v[8];
    Act<float>::load8(x + i * 8, v);
    Act<__nv_bfloat16>::store8(y + i * 8, v);
  }
}

int grid_for(long n8) {
  long g = (n8 + 255) / 256;
  const long cap = (long)fira_num_sms() * 8;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// ---- global-norm clipping
constexpr long kSumsqMaxBlocks = 1024;        // about one wave of 256-thread CTAs on 132 SMs; NOT sized from the SM
                                              // count, so the partials and their sum are the same on every device

long sumsq_blocks(long n8) {
  const long g = (n8 + 255) / 256;
  return g < 1 ? 1 : (g > kSumsqMaxBlocks ? kSumsqMaxBlocks : g);
}

// sum of v over a 256-thread CTA in a fixed order (butterfly per warp, then warps 0..7); the result is thread 0's
__device__ __forceinline__ double block_sum_f64(double v) {
  __shared__ double warp_part[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0) {
    t = warp_part[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) t += warp_part[w];
  }
  return t;
}

__global__ void __launch_bounds__(256) grad_sumsq_kernel(const float* __restrict__ g, long n8, double* __restrict__ partials) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  double acc = 0.0;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    float gv[8];
    Act<float>::load8(g + i * 8, gv);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fma((double)gv[j], (double)gv[j], acc);     // g^2 is exact in float64
  }
  const double s = block_sum_f64(acc);
  if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

__global__ void __launch_bounds__(256) clip_finalize_kernel(const double* __restrict__ partials, long n_partials,
                                                            const float* __restrict__ grad_scale, double max_norm,
                                                            double* __restrict__ clip, float* const* __restrict__ steps,
                                                            int n_steps) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  double acc = 0.0;
  for (long i = threadIdx.x; i < n_partials; i += blockDim.x) acc += partials[i];
  const double S = block_sum_f64(acc);
  if (threadIdx.x != 0) return;
  const double s = grad_scale ? (double)*grad_scale : 1.0;
  const double norm = sqrt(S) / s;
  clip[FIRA_CLIP_NORM] = norm;
  if (!isfinite(S)) {
    clip[FIRA_CLIP_TAKEN] = 0.0;
    clip[FIRA_CLIP_SKIPPED] += 1.0;
    return;
  }
  const float coef = (float)fmin(1.0, max_norm / (norm + 1e-6));
  clip[FIRA_CLIP_COEF] = (double)coef;
  clip[FIRA_CLIP_TAKEN] = 1.0;
  if (coef < 1.f) clip[FIRA_CLIP_CLIPPED] += 1.0;
  for (int k = 0; k < n_steps; ++k) *steps[k] += 1.f;
}

}  // namespace

extern "C" {

int fira_adam_flat(float* p, const float* g, float* m, float* v, void* p_bf16, long n, float lr, float beta1, float beta2,
                   float eps, const float* step, const float* grad_scale, float* ema, float ema_decay, void* stream) {
  FIRA_CHECK_ARG(p && g && m && v && step, FIRA_ERR_ARG, "adam_flat: null argument");
  FIRA_CHECK_ARG(n > 0 && n % 8 == 0, FIRA_ERR_SHAPE, "adam_flat: n %ld must be a positive multiple of 8", n);
  FIRA_CHECK_ARG(fira_aligned16(p) && fira_aligned16(g) && fira_aligned16(m) && fira_aligned16(v) && fira_aligned16(p_bf16) &&
                 fira_aligned16(ema), FIRA_ERR_ALIGN, "adam_flat: 16-B alignment");
  if (ema) {
    FIRA_CHECK_ARG(ema_decay > 0.f && ema_decay < 1.f, FIRA_ERR_ARG,       // NaN fails both comparisons
                   "adam_flat: ema_decay %g must be a finite number in (0, 1)", (double)ema_decay);
    launch_k(adam_flat_kernel<true, false>, dim3(grid_for(n / 8)), dim3(256), 0, (cudaStream_t)stream, p, g, m, v,
             (__nv_bfloat16*)p_bf16, ema, n / 8, lr, beta1, beta2, eps, step, grad_scale, ema_decay,
             (const double*)nullptr);
  } else {
    launch_k(adam_flat_kernel<false, false>, dim3(grid_for(n / 8)), dim3(256), 0, (cudaStream_t)stream, p, g, m, v,
             (__nv_bfloat16*)p_bf16, (float*)nullptr, n / 8, lr, beta1, beta2, eps, step, grad_scale, 0.f,
             (const double*)nullptr);
  }
  FIRA_CHECK_LAUNCH("fira_adam_flat");
  return FIRA_OK;
}

int fira_adam_flat_clip(float* p, const float* g, float* m, float* v, void* p_bf16, long n, float lr, float beta1,
                        float beta2, float eps, const float* step, const float* grad_scale, float* ema, float ema_decay,
                        const double* clip, void* stream) {
  FIRA_CHECK_ARG(p && g && m && v && step && clip, FIRA_ERR_ARG, "adam_flat_clip: null argument");
  FIRA_CHECK_ARG(n > 0 && n % 8 == 0, FIRA_ERR_SHAPE, "adam_flat_clip: n %ld must be a positive multiple of 8", n);
  FIRA_CHECK_ARG(fira_aligned16(p) && fira_aligned16(g) && fira_aligned16(m) && fira_aligned16(v) && fira_aligned16(p_bf16) &&
                 fira_aligned16(ema) && ((uintptr_t)clip & 7u) == 0, FIRA_ERR_ALIGN, "adam_flat_clip: 16-B alignment");
  if (ema) {
    FIRA_CHECK_ARG(ema_decay > 0.f && ema_decay < 1.f, FIRA_ERR_ARG,       // NaN fails both comparisons
                   "adam_flat_clip: ema_decay %g must be a finite number in (0, 1)", (double)ema_decay);
    launch_k(adam_flat_kernel<true, true>, dim3(grid_for(n / 8)), dim3(256), 0, (cudaStream_t)stream, p, g, m, v,
             (__nv_bfloat16*)p_bf16, ema, n / 8, lr, beta1, beta2, eps, step, grad_scale, ema_decay, clip);
  } else {
    launch_k(adam_flat_kernel<false, true>, dim3(grid_for(n / 8)), dim3(256), 0, (cudaStream_t)stream, p, g, m, v,
             (__nv_bfloat16*)p_bf16, (float*)nullptr, n / 8, lr, beta1, beta2, eps, step, grad_scale, 0.f, clip);
  }
  FIRA_CHECK_LAUNCH("fira_adam_flat_clip");
  return FIRA_OK;
}

int fira_grad_sumsq_blocks(long n) { return n > 0 && n % 8 == 0 ? (int)sumsq_blocks(n / 8) : 0; }

int fira_grad_sumsq(const float* g, long n, double* partials, void* stream) {
  FIRA_CHECK_ARG(g && partials, FIRA_ERR_ARG, "grad_sumsq: null argument");
  FIRA_CHECK_ARG(n > 0 && n % 8 == 0, FIRA_ERR_SHAPE, "grad_sumsq: n %ld must be a positive multiple of 8", n);
  FIRA_CHECK_ARG(fira_aligned16(g) && ((uintptr_t)partials & 7u) == 0, FIRA_ERR_ALIGN, "grad_sumsq: 16-B alignment");
  launch_k(grad_sumsq_kernel, dim3((unsigned)sumsq_blocks(n / 8)), dim3(256), 0, (cudaStream_t)stream, g, n / 8, partials);
  FIRA_CHECK_LAUNCH("fira_grad_sumsq");
  return FIRA_OK;
}

int fira_grad_clip_finalize(const double* partials, long n_partials, const float* grad_scale, double max_norm,
                            double* clip, float* const* steps, int n_steps, void* stream) {
  FIRA_CHECK_ARG(partials && clip && (steps || n_steps == 0), FIRA_ERR_ARG, "grad_clip_finalize: null argument");
  FIRA_CHECK_ARG(n_partials > 0 && n_steps >= 0, FIRA_ERR_SHAPE, "grad_clip_finalize: n_partials %ld, n_steps %d",
                 n_partials, n_steps);
  FIRA_CHECK_ARG(max_norm > 0.0, FIRA_ERR_ARG,                               // NaN fails the comparison; inf is allowed
                 "grad_clip_finalize: max_norm %g must be > 0 (inf = never clip)", max_norm);
  FIRA_CHECK_ARG(((uintptr_t)partials & 7u) == 0 && ((uintptr_t)clip & 7u) == 0 && ((uintptr_t)steps & 7u) == 0,
                 FIRA_ERR_ALIGN, "grad_clip_finalize: 8-B alignment");
  launch_k(clip_finalize_kernel, dim3(1), dim3(256), 0, (cudaStream_t)stream, partials, n_partials, grad_scale, max_norm,
           clip, steps, n_steps);
  FIRA_CHECK_LAUNCH("fira_grad_clip_finalize");
  return FIRA_OK;
}

int fira_cast_bf16(const float* x, void* y, long n, void* stream) {
  FIRA_CHECK_ARG(x && y, FIRA_ERR_ARG, "cast_bf16: null argument");
  FIRA_CHECK_ARG(n > 0 && n % 8 == 0, FIRA_ERR_SHAPE, "cast_bf16: n %ld must be a positive multiple of 8", n);
  FIRA_CHECK_ARG(fira_aligned16(x) && fira_aligned16(y), FIRA_ERR_ALIGN, "cast_bf16: 16-B alignment");
  launch_k(cast_bf16_kernel, dim3(grid_for(n / 8)), dim3(256), 0, (cudaStream_t)stream, x, (__nv_bfloat16*)y, n / 8);
  FIRA_CHECK_LAUNCH("fira_cast_bf16");
  return FIRA_OK;
}

}  // extern "C"
