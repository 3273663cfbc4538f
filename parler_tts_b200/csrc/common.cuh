// common.cuh -- shared helpers for the sm_90a kernels (device math, dtype traits, error plumbing).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/ptts_b200.h"

namespace ptts {

typedef __nv_bfloat16 bf16;

// ---- host-side error plumbing -------------------------------------------------------------------
void set_error(const std::string& msg);
int fail(int code, const char* fmt, ...);

#define PTTS_CHECK_CUDA(expr)                                                                      \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return ::ptts::fail(PTTS_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#define PTTS_REQUIRE(cond, ...)                                                                    \
  do {                                                                                             \
    if (!(cond)) return ::ptts::fail(PTTS_EINVAL, __VA_ARGS__);                                    \
  } while (0)

#define PTTS_LAUNCH_CHECK() PTTS_CHECK_CUDA(cudaGetLastError())

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// ---- device control block (lives in the workspace) ----------------------------------------------
// All step kernels read it; ptts_sample's last block advances it.  Keeping the step index on the
// device lets one captured CUDA graph be replayed for every decode step without a host round trip.
struct Ctrl {
  int cur_len;        // columns in raw_ids (1 after begin; +1 per sampled token)
  int active;         // 1 while any row is unfinished and cur_len < max_length
  int n_unfinished;
  int done_blocks;    // last-block-done counter for ptts_sample
  int steps_run;      // decode steps actually executed (not no-op'd)
  int launch_gen;     // fused step kernel launches so far (selects the barrier counter)
  int pad_[26];
  unsigned bar[32];   // barrier counters of the fused step kernel (own 128 B line): slot s uses bar[16 s + (launch_gen & 1)]
};
static_assert(sizeof(Ctrl) == 256, "Ctrl layout");

// Ragged continuation (ptts_generate_begin_ids2): batch row b continues from shift[b] fewer input columns than the longest row,
// so its history column and cache position are the batch's minus shift[b] -- what the row alone would have.  The array is
// written once by the begin kernel; shift == nullptr (every row at the batch's own column) reads nothing.
__device__ __forceinline__ int row_shift(const int* shift, int b) { return shift != nullptr ? shift[b] : 0; }

// ---- dtype traits -------------------------------------------------------------------------------
template <typename T> struct DT;
template <> struct DT<bf16> {
  static constexpr int code = PTTS_BF16;
  __device__ __forceinline__ static float to_f(bf16 v) { return __bfloat162float(v); }
  __device__ __forceinline__ static bf16 from_f(float v) { return __float2bfloat16_rn(v); }
  // round-trip through the storage type: mimics torch rounding every op output to the model dtype
  __device__ __forceinline__ static float rnd(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
};
template <> struct DT<float> {
  static constexpr int code = PTTS_F32;
  __device__ __forceinline__ static float to_f(float v) { return v; }
  __device__ __forceinline__ static float from_f(float v) { return v; }
  __device__ __forceinline__ static float rnd(float v) { return v; }
};

// 8 consecutive elements -> 8 floats (16 B for bf16, 32 B for f32)
__device__ __forceinline__ void load8(const bf16* p, float (&v)[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    float2 f = __bfloat1622float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  float4 a = *reinterpret_cast<const float4*>(p);
  float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; i++) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ void store8(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

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

// activation_function (configuration_parler_tts.py:118; ACT2FN at modeling_parler_tts.py:958)
__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case 0: return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));  // gelu (erf)
    case 1: return fmaxf(x, 0.0f);
    case 2: return x / (1.0f + expf(-x));
    default: {
      const float k = 0.7978845608028654f;
      return 0.5f * x * (1.0f + tanhf(k * (x + 0.044715f * x * x * x)));
    }
  }
}

// K/V cache rows are stored SWIZZLED: element d of the 64-wide row of key t lives at position kv_swz(t, d) -- the 8-element
// (16-byte bf16) chunk index XORed with t & 7.  A contiguous bulk copy of 8n rows then lands in shared memory as a
// bank-conflict-free ldmatrix tile (what a SWIZZLE_128B tensor map would produce) with no tensor map: the tensor-core attention
// of the cluster step kernel depends on it, every other reader / writer of the caches just applies the same index map.
__host__ __device__ __forceinline__ int kv_swz(int t, int d) { return ((((d >> 3) ^ t) & 7) << 3) | (d & 7); }

// Programmatic dependent launch: everything before pdl_wait() overlaps the previous kernel's tail.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

}  // namespace ptts
