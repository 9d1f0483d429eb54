// Shared device/host helpers for the tfx_b200 kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace tfx {

// ---- error plumbing for the C ABI (never throws across the boundary)
void set_error(const char* fmt, ...);
int check_launch(const char* what);     // cudaGetLastError -> 0 / negative code

#define TFX_REQUIRE(cond, ...) do { if (!(cond)) { tfx::set_error(__VA_ARGS__); return -1; } } while (0)

constexpr int WARPS_PER_BLOCK = 8;
constexpr int ROW_THREADS = WARPS_PER_BLOCK * 32;

// grid of the warp-per-row kernels (their warps stride over the rows): one warp per row, at most 8 blocks per SM
inline int row_grid(int M, int sms) {
  long long blocks = ((long long)M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
  long long cap = (long long)sms * 8;
  return (int)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

// accurate tanh from two MUFU ops (ex2 + rcp): abs error ~1e-7, needed because the attention soft-cap (50) and the LASER clamp (15) multiply it
__device__ __forceinline__ float tanh_acc(float x) {
  const float e = __expf(2.f * x);
  return 1.f - __fdividef(2.f, 1.f + e);
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

__device__ __forceinline__ uint32_t pack2_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack2_bf16(uint32_t w) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&w);
  return __bfloat1622float2(t);
}

// Row access pattern for "one warp per token" kernels: D = 128 * NCH, lane owns 4 consecutive floats
// in each 128-wide chunk -> every warp-level access is one contiguous 512 B (fp32) / 256 B (bf16) run.
template <int NCH>
__device__ __forceinline__ void load_row_f32(const float* __restrict__ base, int lane, float (&v)[NCH * 4]) {
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const float4 t = *reinterpret_cast<const float4*>(base + c * 128 + lane * 4);
    v[c * 4] = t.x; v[c * 4 + 1] = t.y; v[c * 4 + 2] = t.z; v[c * 4 + 3] = t.w;
  }
}
template <int NCH>
__device__ __forceinline__ void store_row_f32(float* __restrict__ base, int lane, const float (&v)[NCH * 4]) {
#pragma unroll
  for (int c = 0; c < NCH; ++c)
    *reinterpret_cast<float4*>(base + c * 128 + lane * 4) = make_float4(v[c * 4], v[c * 4 + 1], v[c * 4 + 2], v[c * 4 + 3]);
}
template <int NCH>
__device__ __forceinline__ void load_row_bf16(const __nv_bfloat16* __restrict__ base, int lane, float (&v)[NCH * 4]) {
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const uint2 t = *reinterpret_cast<const uint2*>(base + c * 128 + lane * 4);
    const float2 a = unpack2_bf16(t.x), b = unpack2_bf16(t.y);
    v[c * 4] = a.x; v[c * 4 + 1] = a.y; v[c * 4 + 2] = b.x; v[c * 4 + 3] = b.y;
  }
}
template <int NCH>
__device__ __forceinline__ void store_row_bf16(__nv_bfloat16* __restrict__ base, int lane, const float (&v)[NCH * 4]) {
#pragma unroll
  for (int c = 0; c < NCH; ++c)
    *reinterpret_cast<uint2*>(base + c * 128 + lane * 4) = make_uint2(pack2_bf16(v[c * 4], v[c * 4 + 1]), pack2_bf16(v[c * 4 + 2], v[c * 4 + 3]));
}
// atomically add a register row into a global fp32 row (used for per-condition-row / per-parameter reductions)
template <int NCH>
__device__ __forceinline__ void red_row_f32(float* __restrict__ base, int lane, const float (&v)[NCH * 4]) {
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    float* d = base + c * 128 + lane * 4;
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d), "f"(v[c * 4]), "f"(v[c * 4 + 1]), "f"(v[c * 4 + 2]), "f"(v[c * 4 + 3]) : "memory");
  }
}

// cp.async pieces for the per-warp row rings of the depth-serial kernels (rowops.cu: AttentionResidual forward / deferred backward)
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async_8(uint32_t dst, const void* src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async_4(uint32_t dst, const void* src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }

// dispatch on model dim D = 128 * NCH: 128, 256, 384, 512, 768, 1024, 1536 or 2048 (transfusion.py MODEL_DIMS lists the same widths)
#define TFX_DISPATCH_NCH(D, ...)                                                       \
  do {                                                                                 \
    switch ((D) / 128) {                                                               \
      case 1: { constexpr int NCH = 1; __VA_ARGS__; } break;                           \
      case 2: { constexpr int NCH = 2; __VA_ARGS__; } break;                           \
      case 3: { constexpr int NCH = 3; __VA_ARGS__; } break;                           \
      case 4: { constexpr int NCH = 4; __VA_ARGS__; } break;                           \
      case 6: { constexpr int NCH = 6; __VA_ARGS__; } break;                           \
      case 8: { constexpr int NCH = 8; __VA_ARGS__; } break;                           \
      case 12: { constexpr int NCH = 12; __VA_ARGS__; } break;                         \
      case 16: { constexpr int NCH = 16; __VA_ARGS__; } break;                         \
      default: tfx::set_error("unsupported model dim %d (need 128, 256, 384, 512, 768, 1024, 1536 or 2048)", (int)(D)); return -1; \
    }                                                                                  \
  } while (0)

}  // namespace tfx
