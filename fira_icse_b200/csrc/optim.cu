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
#include "common.cuh"
#include "fira_b200.h"

namespace {

template <bool EMA>
__global__ void __launch_bounds__(256) adam_flat_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                        float* __restrict__ m, float* __restrict__ v,
                                                        __nv_bfloat16* __restrict__ p16, float* __restrict__ ema,
                                                        long n8, float lr, float b1, float b2, float eps,
                                                        const float* __restrict__ step,
                                                        const float* __restrict__ grad_scale, float ema_decay) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
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
      const float gj = gv[j] * inv_scale;
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
    launch_k(adam_flat_kernel<true>, dim3(grid_for(n / 8)), dim3(256), 0, (cudaStream_t)stream, p, g, m, v,
             (__nv_bfloat16*)p_bf16, ema, n / 8, lr, beta1, beta2, eps, step, grad_scale, ema_decay);
  } else {
    launch_k(adam_flat_kernel<false>, dim3(grid_for(n / 8)), dim3(256), 0, (cudaStream_t)stream, p, g, m, v,
             (__nv_bfloat16*)p_bf16, (float*)nullptr, n / 8, lr, beta1, beta2, eps, step, grad_scale, 0.f);
  }
  FIRA_CHECK_LAUNCH("fira_adam_flat");
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
