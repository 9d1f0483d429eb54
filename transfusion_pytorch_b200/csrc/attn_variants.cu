// Optional attention variants of the reference's Attention.forward (transfusion.py:918-1039) as HBM-bound row kernels around the fused
// attention kernels (one warp per token; DH / 8 lanes share a head with 16-byte bf16 accesses, 32 / (DH / 8) heads per pass - the layout of
// attn_bwd_prep).  The per-head kernels are templates on the head dim DH, instantiated at 64 and 128:
//
//   LASER (T.py:981-983, 1021-1022; laser_softclamp_value = 15):   v' = exp(15 tanh(v / 15))  ->  attention  ->  out = log(out) [* sigmoid(gate)]
//       the kv cache keeps the RAW value (T.py:976-977 stacks before the transform); the transformed copy is a second slab written in place;
//   learned value residual (T.py:956-960, 1234):   v = v * mix + v_first_layer * (1 - mix),  mix = sigmoid(Linear(dim -> heads, bias)(x)) per token and head.
//       The Linear lives in the pad rows of the packed QKVG weight (its pre-activation is written by the QKVG epilogue, its gradient goes through the
//       packed dqkvg matrix), only the bias and the mixing are here.
#include "common.cuh"
#include "../../include/tfx_b200.h"
#include <math.h>

namespace tfx {

int num_sms();

__device__ __forceinline__ float sigmoid_v(float x) { return 1.f / (1.f + __expf(-x)); }

// One warp per token; DH / 8 lanes share a head (a lane owns 8 consecutive dims: 16-byte bf16 accesses), 32 / (DH / 8) heads per pass.
#define VAR_ROW_LOOP(DH)                                                                               \
  constexpr int LPH = (DH) / 8, HPP = 32 / LPH;                                                        \
  const int lane = threadIdx.x & 31, sub = lane % LPH, hq = (lane >> 3) / (LPH / 8);                  \
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5; \
  for (int row = warp0; row < M; row += nwarps)                                                        \
    for (int h0 = 0; h0 < H; h0 += HPP)

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&x)[8]) {
  const uint4 t = *reinterpret_cast<const uint4*>(p);
  const float2 a = unpack2_bf16(t.x), b = unpack2_bf16(t.y), c = unpack2_bf16(t.z), d = unpack2_bf16(t.w);
  x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y; x[4] = c.x; x[5] = c.y; x[6] = d.x; x[7] = d.y;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&x)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack2_bf16(x[0], x[1]), pack2_bf16(x[2], x[3]), pack2_bf16(x[4], x[5]), pack2_bf16(x[6], x[7]));
}
// sum over the LPH lanes of a head.  The same butterfly at both widths, spelled per width: each spelling keeps the generated code its width was
// measured with (the loop form reschedules the 64-wide kernels, the unrolled form the 128-wide ones).
template <int LPH>
__device__ __forceinline__ float sum_head_lanes(float s) {
  if constexpr (LPH == 8) {
    s += __shfl_xor_sync(0xffffffffu, s, 1); s += __shfl_xor_sync(0xffffffffu, s, 2); s += __shfl_xor_sync(0xffffffffu, s, 4);
  } else {
#pragma unroll
    for (int o = 1; o < LPH; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  return s;
}

// laser_v_fwd / laser_v_bwd are elementwise and serve any head dim (a 128-wide head is two 64-wide ones).
// v' = exp(c tanh(v / c)); rows (optional): cache row of token `row` (source and destination are then cache slabs)
__global__ void __launch_bounds__(ROW_THREADS) laser_v_fwd_k(const __nv_bfloat16* __restrict__ v, long long ld_v, const int* __restrict__ rows, __nv_bfloat16* __restrict__ vl,
                                                            long long ld_vl, int M, int H, float c) {
  VAR_ROW_LOOP(64) {
    const int h = h0 + hq;
    if (h >= H) continue;
    const long long r = rows ? rows[row] : row;
    float x[8];
    ld8(v + r * ld_v + h * 64 + sub * 8, x);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = __expf(c * tanh_acc(x[e] / c));
    st8(vl + r * ld_vl + h * 64 + sub * 8, x);
  }
}

// dv = dv' * v' * (1 - tanh^2(v / c)), in place on dv'
__global__ void __launch_bounds__(ROW_THREADS) laser_v_bwd_k(__nv_bfloat16* __restrict__ dv, long long ld_dv, const __nv_bfloat16* __restrict__ v, long long ld_v, int M, int H, float c) {
  VAR_ROW_LOOP(64) {
    const int h = h0 + hq;
    if (h >= H) continue;
    float g[8], x[8];
    ld8(dv + (long long)row * ld_dv + h * 64 + sub * 8, g);
    ld8(v + (long long)row * ld_v + h * 64 + sub * 8, x);
#pragma unroll
    for (int e = 0; e < 8; ++e) { const float t = tanh_acc(x[e] / c); g[e] *= __expf(c * t) * (1.f - t * t); }
    st8(dv + (long long)row * ld_dv + h * 64 + sub * 8, g);
  }
}

// att = log(o) * sigmoid(gate)
template <int DH>
__global__ void __launch_bounds__(ROW_THREADS) laser_out_fwd_k(const __nv_bfloat16* __restrict__ o, const float* __restrict__ gates, __nv_bfloat16* __restrict__ att, int M, int H) {
  const long long HI = (long long)H * DH;
  VAR_ROW_LOOP(DH) {
    const int h = h0 + hq;
    if (h >= H) continue;
    const long long off = row * HI + h * DH + sub * 8;
    const float sg = gates ? sigmoid_v(gates[(long long)row * H + h]) : 1.f;
    float x[8];
    ld8(o + off, x);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = __logf(fmaxf(x[e], 1e-30f)) * sg;
    st8(att + off, x);
  }
}

// backward of att = log(o) * sg:  dO = dAtt * sg / o ;  D[h][row] = sum_d dO * o = sum_d dAtt * sg ;  gate sums[row][h] = sum_d dAtt * att  (d gate_pre = (1 - sg) * that)
template <int DH>
__global__ void __launch_bounds__(ROW_THREADS) laser_bwd_prep_k(const __nv_bfloat16* __restrict__ datt, const __nv_bfloat16* __restrict__ o, const float* __restrict__ gates,
                                                               __nv_bfloat16* __restrict__ dop, float* __restrict__ dsum, float* __restrict__ dsum_rowmajor,
                                                               float* __restrict__ dq_zero, int M, int H) {
  const long long HI = (long long)H * DH;
  VAR_ROW_LOOP(DH) {
    const int h = h0 + hq;
    const bool act = h < H;
    const long long off = row * HI + (act ? h : 0) * DH + sub * 8;
    const float sg = (act && gates) ? sigmoid_v(gates[(long long)row * H + h]) : 1.f;
    float a[8], b[8], w[8];
    ld8(datt + off, a); ld8(o + off, b);
    float s = 0.f, gsum = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float oo = fmaxf(b[e], 1e-30f);
      s += a[e] * sg;
      gsum += a[e] * __logf(oo) * sg;
      w[e] = a[e] * sg / oo;
    }
    s = sum_head_lanes<LPH>(s); gsum = sum_head_lanes<LPH>(gsum);
    if (act) {
      st8(dop + off, w);
      if (sub == 0) { dsum[(long long)h * M + row] = s; if (dsum_rowmajor) dsum_rowmajor[(long long)row * H + h] = gsum; }
      if (dq_zero) {
        *reinterpret_cast<float4*>(dq_zero + off) = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(dq_zero + off + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  }
}

// v = v * mix + v0 * (1 - mix), in place; rows (optional) = cache row of the token in both v and v0
template <int DH>
__global__ void __launch_bounds__(ROW_THREADS) vmix_fwd_k(__nv_bfloat16* __restrict__ v, long long ld_v, const int* __restrict__ rows, const __nv_bfloat16* __restrict__ v0,
                                                         long long ld_v0, const float* __restrict__ mixpre, const float* __restrict__ bias, int M, int H) {
  VAR_ROW_LOOP(DH) {
    const int h = h0 + hq;
    if (h >= H) continue;
    const long long r = rows ? rows[row] : row;
    const float mix = sigmoid_v(mixpre[(long long)row * H + h] + bias[h]);
    float a[8], b[8];
    ld8(v + r * ld_v + h * DH + sub * 8, a); ld8(v0 + r * ld_v0 + h * DH + sub * 8, b);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] = a[e] * mix + b[e] * (1.f - mix);
    st8(v + r * ld_v + h * DH + sub * 8, a);
  }
}

// backward of the mix (dv holds d v_mixed on entry, d v_raw on exit):  dv_raw = dvm * mix ;  dv0 += dvm * (1 - mix) ;
// d mix_pre = sum_d dvm (v_raw - v0) mix (1 - mix) = sum_d dvm (v_mixed - v0) (1 - mix)        [v_mixed - v0 = (v_raw - v0) mix]
template <int DH>
__global__ void __launch_bounds__(ROW_THREADS) vmix_bwd_k(__nv_bfloat16* __restrict__ dv, long long ld_dv, const __nv_bfloat16* __restrict__ vm, long long ld_v,
                                                         const __nv_bfloat16* __restrict__ v0, long long ld_v0, const float* __restrict__ mixpre, const float* __restrict__ bias,
                                                         float* __restrict__ dv0_acc, __nv_bfloat16* __restrict__ dmix, long long ld_dmix, int M, int H) {
  const long long HI = (long long)H * DH;
  VAR_ROW_LOOP(DH) {
    const int h = h0 + hq;
    const bool act = h < H;
    const int hh = act ? h : 0;
    const float mix = sigmoid_v(mixpre[(long long)row * H + hh] + bias[hh]);
    float g[8], a[8], b[8];
    ld8(dv + (long long)row * ld_dv + hh * DH + sub * 8, g);
    ld8(vm + (long long)row * ld_v + hh * DH + sub * 8, a);
    ld8(v0 + (long long)row * ld_v0 + hh * DH + sub * 8, b);
    float s = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) s += g[e] * (a[e] - b[e]);
    s = sum_head_lanes<LPH>(s) * (1.f - mix);
    if (act) {
      float* acc = dv0_acc + row * HI + h * DH + sub * 8;
      const float4 c0 = *reinterpret_cast<const float4*>(acc), c1 = *reinterpret_cast<const float4*>(acc + 4);
      const float om = 1.f - mix;
      *reinterpret_cast<float4*>(acc) = make_float4(c0.x + g[0] * om, c0.y + g[1] * om, c0.z + g[2] * om, c0.w + g[3] * om);
      *reinterpret_cast<float4*>(acc + 4) = make_float4(c1.x + g[4] * om, c1.y + g[5] * om, c1.z + g[6] * om, c1.w + g[7] * om);
#pragma unroll
      for (int e = 0; e < 8; ++e) g[e] *= mix;
      st8(dv + (long long)row * ld_dv + h * DH + sub * 8, g);
      if (sub == 0) dmix[(long long)row * ld_dmix + h] = __float2bfloat16(s);
    }
  }
}

// dst(bf16) += src(fp32): first-layer value gradient += what the later layers' value residuals sent back
__global__ void __launch_bounds__(ROW_THREADS) add_f32_into_bf16_k(__nv_bfloat16* __restrict__ dst, long long ld_dst, const float* __restrict__ src, long long ld_src, int M, int N) {
  const int per_row = N / 8;
  const long long total = (long long)M * per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / per_row; const int c = (int)(i - r * per_row) * 8;
    float x[8];
    ld8(dst + r * ld_dst + c, x);
    const float4 a = *reinterpret_cast<const float4*>(src + r * ld_src + c), b = *reinterpret_cast<const float4*>(src + r * ld_src + c + 4);
    x[0] += a.x; x[1] += a.y; x[2] += a.z; x[3] += a.w; x[4] += b.x; x[5] += b.y; x[6] += b.z; x[7] += b.w;
    st8(dst + r * ld_dst + c, x);
  }
}

}  // namespace tfx

using namespace tfx;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)

// launchers of the per-head kernels, behind each entry point and its _d128 twin; `name` is the entry point's name for error messages
template <int DH>
static int laser_out_fwd(const char* name, const void* o_laser, const float* gates, void* att, int M, int H, void* stream) {
  if (M <= 0) return 0;
  laser_out_fwd_k<DH><<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>(CBF(o_laser), gates, BF(att), M, H);
  return check_launch(name);
}

template <int DH>
static int laser_bwd_prep(const char* name, const void* d_att, const void* o_laser, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero,
                          int M, int H, void* stream) {
  if (M <= 0) return 0;
  laser_bwd_prep_k<DH><<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>(CBF(d_att), CBF(o_laser), gates, BF(do_pre), dsum_hm, dsum_mh, dq_zero, M, H);
  return check_launch(name);
}

template <int DH>
static int vmix_fwd(const char* name, void* v_inout, long long ld_v, const int* rows, const void* v_first, long long ld_v0, const float* mix_pre,
                    const float* mix_bias, int M, int H, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(ld_v % 8 == 0 && ld_v0 % 8 == 0 && mix_pre && mix_bias, "%s: bad arguments", name);
  vmix_fwd_k<DH><<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>(BF(v_inout), ld_v, rows, CBF(v_first), ld_v0, mix_pre, mix_bias, M, H);
  return check_launch(name);
}

template <int DH>
static int vmix_bwd(const char* name, void* dv_inout, long long ld_dv, const void* v_mixed, long long ld_v, const void* v_first, long long ld_v0,
                    const float* mix_pre, const float* mix_bias, float* dv_first_acc, void* dmix_bf16, long long ld_dmix, int M, int H, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(ld_v % 8 == 0 && ld_v0 % 8 == 0 && ld_dv % 8 == 0, "%s: row pitches must be multiples of 8 bf16", name);
  vmix_bwd_k<DH><<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>(BF(dv_inout), ld_dv, CBF(v_mixed), ld_v, CBF(v_first), ld_v0, mix_pre, mix_bias, dv_first_acc,
                                                                         BF(dmix_bf16), ld_dmix, M, H);
  return check_launch(name);
}

extern "C" {

int tfx_laser_v_fwd(const void* v, long long ld_v, const int* rows, void* v_laser, long long ld_vl, int M, int H, float clamp, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(clamp > 0.f && ld_v % 8 == 0 && ld_vl % 8 == 0, "laser_v_fwd: clamp must be > 0 and row pitches multiples of 8 bf16");
  laser_v_fwd_k<<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>(CBF(v), ld_v, rows, BF(v_laser), ld_vl, M, H, clamp);
  return check_launch("laser_v_fwd");
}

int tfx_laser_v_bwd(void* dv_inout, long long ld_dv, const void* v, long long ld_v, int M, int H, float clamp, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(clamp > 0.f && ld_v % 8 == 0 && ld_dv % 8 == 0, "laser_v_bwd: clamp must be > 0 and row pitches multiples of 8 bf16");
  laser_v_bwd_k<<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>(BF(dv_inout), ld_dv, CBF(v), ld_v, M, H, clamp);
  return check_launch("laser_v_bwd");
}

int tfx_laser_out_fwd(const void* o_laser, const float* gates, void* att, int M, int H, void* stream) {
  return laser_out_fwd<64>("laser_out_fwd", o_laser, gates, att, M, H, stream);
}

int tfx_laser_out_fwd_d128(const void* o_laser, const float* gates, void* att, int M, int H, void* stream) {
  return laser_out_fwd<128>("laser_out_fwd_d128", o_laser, gates, att, M, H, stream);
}

int tfx_laser_bwd_prep(const void* d_att, const void* o_laser, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero, int M, int H, void* stream) {
  return laser_bwd_prep<64>("laser_bwd_prep", d_att, o_laser, gates, do_pre, dsum_hm, dsum_mh, dq_zero, M, H, stream);
}

int tfx_laser_bwd_prep_d128(const void* d_att, const void* o_laser, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero, int M, int H, void* stream) {
  return laser_bwd_prep<128>("laser_bwd_prep_d128", d_att, o_laser, gates, do_pre, dsum_hm, dsum_mh, dq_zero, M, H, stream);
}

int tfx_vmix_fwd(void* v_inout, long long ld_v, const int* rows, const void* v_first, long long ld_v0, const float* mix_pre, const float* mix_bias, int M, int H, void* stream) {
  return vmix_fwd<64>("vmix_fwd", v_inout, ld_v, rows, v_first, ld_v0, mix_pre, mix_bias, M, H, stream);
}

int tfx_vmix_fwd_d128(void* v_inout, long long ld_v, const int* rows, const void* v_first, long long ld_v0, const float* mix_pre, const float* mix_bias, int M, int H, void* stream) {
  return vmix_fwd<128>("vmix_fwd_d128", v_inout, ld_v, rows, v_first, ld_v0, mix_pre, mix_bias, M, H, stream);
}

int tfx_vmix_bwd(void* dv_inout, long long ld_dv, const void* v_mixed, long long ld_v, const void* v_first, long long ld_v0, const float* mix_pre, const float* mix_bias,
                 float* dv_first_acc, void* dmix_bf16, long long ld_dmix, int M, int H, void* stream) {
  return vmix_bwd<64>("vmix_bwd", dv_inout, ld_dv, v_mixed, ld_v, v_first, ld_v0, mix_pre, mix_bias, dv_first_acc, dmix_bf16, ld_dmix, M, H, stream);
}

int tfx_vmix_bwd_d128(void* dv_inout, long long ld_dv, const void* v_mixed, long long ld_v, const void* v_first, long long ld_v0, const float* mix_pre, const float* mix_bias,
                      float* dv_first_acc, void* dmix_bf16, long long ld_dmix, int M, int H, void* stream) {
  return vmix_bwd<128>("vmix_bwd_d128", dv_inout, ld_dv, v_mixed, ld_v, v_first, ld_v0, mix_pre, mix_bias, dv_first_acc, dmix_bf16, ld_dmix, M, H, stream);
}

int tfx_add_f32_into_bf16(void* dst_bf16, long long ld_dst, const float* src, long long ld_src, int M, int N, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  TFX_REQUIRE(N % 8 == 0 && ld_dst % 8 == 0 && ld_src % 4 == 0, "add_f32_into_bf16: N and the pitches must keep 16-byte alignment");
  const long long total = (long long)M * (N / 8);
  long long blocks = (total + 255) / 256, cap = (long long)num_sms() * 8;
  add_f32_into_bf16_k<<<(int)(blocks < cap ? blocks : cap), 256, 0, ST(stream)>>>(BF(dst_bf16), ld_dst, src, ld_src, M, N);
  return check_launch("add_f32_into_bf16");
}

}  // extern "C"
