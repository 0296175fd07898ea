// Shared device/host helpers for libfira_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#define FIRA_OK 0
#define FIRA_ERR_SHAPE 1
#define FIRA_ERR_ALIGN 2
#define FIRA_ERR_CUDA 3
#define FIRA_ERR_DTYPE 4
#define FIRA_ERR_ARG 5

#define FIRA_F32 0
#define FIRA_BF16 1

// set by every entry point on failure; read by fira_last_error_string()
void fira_set_error(int code, const char* fmt, ...);

#define FIRA_CHECK_ARG(cond, code, ...)                      \
  do {                                                       \
    if (!(cond)) {                                           \
      fira_set_error((code), __VA_ARGS__);                   \
      return (code);                                         \
    }                                                        \
  } while (0)

#define FIRA_CHECK_LAUNCH(name)                                                   \
  do {                                                                            \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) {                                                     \
      fira_set_error(FIRA_ERR_CUDA, "%s: %s", (name), cudaGetErrorString(e__));   \
      return FIRA_ERR_CUDA;                                                       \
    }                                                                             \
  } while (0)

// streaming multiprocessors of the current device (api.cu, cached per device): every grid of the library is sized
// from this one query
extern "C" int fira_num_sms(void);

static inline bool fira_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// launch mode of every kernel of the library (api.cu; fira_set_pdl / FIRA_PDL): 1 = programmatic dependent launch
int fira_pdl_on();

#ifdef __CUDACC__

// ---- programmatic dependent launch (PDL).  Every kernel of the library starts with pdl_wait() -- before its first
//      global-memory access -- and pdl_trigger(): launched with the programmatic-serialization attribute (launch_k
//      below), its CTAs are scheduled while the previous kernel of the stream drains, run their on-chip prologue
//      (barrier init, tensor-map prefetch), and block in griddepcontrol.wait until that kernel has
//      completed and flushed.  Because EVERY kernel waits before touching memory, completion is transitive along the
//      stream.  Inside a captured CUDA graph the attribute becomes a programmatic edge; after a non-kernel node or a
//      cross-stream join it degrades to a full dependency.  Without the attribute both instructions are no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = fira_pdl_on() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

constexpr int kWarp = 32;
constexpr float kLnEps = 1e-5f;
constexpr float kMaskFill = -1e9f;   // gnn_transformer.py:153, Model.py:61

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- activation storage type traits: fp32 (parity mode) and bf16 (throughput mode) ----
template <typename T> struct Act;
template <> struct Act<float> {
  // 8 consecutive elements <-> 8 floats
  static __device__ __forceinline__ void load8(const float* p, float* v) {
    float4 a = *reinterpret_cast<const float4*>(p);
    float4 b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  static __device__ __forceinline__ void store8(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
  static __device__ __forceinline__ float ld(const float* p) { return *p; }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
template <> struct Act<__nv_bfloat16> {
  static __device__ __forceinline__ void load8(const __nv_bfloat16* p, float* v) {
    uint4 r = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
  }
  static __device__ __forceinline__ void store8(__nv_bfloat16* p, const float* v) {
    uint4 r;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = r;
  }
  static __device__ __forceinline__ float ld(const __nv_bfloat16* p) { return __bfloat162float(*p); }
  static __device__ __forceinline__ void st(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
};

// ---- counter-based dropout RNG (Philox4x32-7): mask is a pure function of (seed, stream, index)
//      so backward recomputes it instead of storing it.  Not bit-compatible with torch's stream
//      order (SURVEY.md K13); tests/philox_rule.py restates this rule in numpy, and tests/test_gpu_dropout_rule.py /
//      tests/test_gpu_train_dropout.py check the kernels and the dropout-on training step against it.
__device__ __forceinline__ uint4 philox4(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                         uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 7; ++r) {
    uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += W0; k1 += W1;
  }
  return make_uint4(c0, c1, c2, c3);
}
// keep-mask for 8 consecutive elements starting at element index idx8*8.
// Returns an 8-bit mask; element i kept iff bit i set.  p_drop in [0,1).
// ONE Philox4x32-7 call serves the 8 elements: 16 random bits per element, compared against p with 2^-16 resolution
// (p = 0.1 -> 0.100006, p = 0.2 -> 0.199997).  Every dropout site (LayerNorm blocks, Combination gate, fused GCN
// epilogue) and its backward draw their masks through this one function, so they agree by construction.
__device__ __forceinline__ uint32_t dropout_keep8(uint64_t seed, uint32_t stream, uint64_t idx8, float p_drop) {
  const uint4 r = philox4((uint32_t)idx8, (uint32_t)(idx8 >> 32), stream, 0u, (uint32_t)seed, (uint32_t)(seed >> 32));
  const uint32_t thr = (uint32_t)(p_drop * 65536.0f);
  uint32_t m = 0;
  m |= ((r.x & 0xffffu) >= thr) << 0; m |= ((r.x >> 16) >= thr) << 1;
  m |= ((r.y & 0xffffu) >= thr) << 2; m |= ((r.y >> 16) >= thr) << 3;
  m |= ((r.z & 0xffffu) >= thr) << 4; m |= ((r.z >> 16) >= thr) << 5;
  m |= ((r.w & 0xffffu) >= thr) << 6; m |= ((r.w >> 16) >= thr) << 7;
  return m;
}

#endif  // __CUDACC__
