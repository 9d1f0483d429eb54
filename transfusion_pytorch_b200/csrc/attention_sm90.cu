// wgmma / TMA attention for sm_90a: the "bounded-logit" fast path of the span-masked, soft-capped
// attention (semantics: attention.cu; reference transfusion.py:998-1027, mask :452-470).
//
// Why a separate path.  q and k are RMS-normalised per head (T.py:950-952), so |q.k| * dh^-1/2 <= 8 * max|gq+1| * max|gk+1|
// is known from the two 64-element gamma vectors before the kernel runs.  When that bound keeps the soft-cap argument
// y = s/cap inside |y| <= 0.75 (true for any gamma product <= 4.6; gamma is 0 at init) two things follow:
//   * tanh(y) is a degree-9 odd polynomial to 2.6e-7 absolute - same accuracy as the MUFU ex2+rcp formulation of the
//     general kernel, but on the FMA pipe (the MUFU pipe is what bounds the general kernel);
//   * the soft-capped logits are bounded by m = cap * y_max <= 37.5, so softmax can use the FIXED maximum m: no running max,
//     no rescaling of the output accumulator - O accumulates untouched in registers across all KV tiles.
// `tfx_attn_fast_params` evaluates the bound on the device; both this kernel and the general one are launched and the one
// whose precondition fails returns immediately (no host synchronisation).
//
// Forward (one CTA = 128 query rows x one head, two consumer warpgroups of 64 rows, 2 CTAs / SM):
//   S = Q K_j^T (wgmma 64x128x16, both operands from shared memory) -> p = 2^(x*poly(x^2) - m2) in registers -> P packed to bf16
//   in the accumulator-fragment order, which is the register A operand of O += P V_j (wgmma 64x64x16, V read MN-major).
//   K_j / V_j arrive by TMA into a two-deep ring; one thread of the CTA issues the loads.
#include "sm90_ptx.cuh"
#include "common.cuh"
#include "gemm_sm90.cuh"
#include "../../include/tfx_b200.h"

namespace tfx {

int num_sms();

constexpr int FA_BM = 128, FA_BN = 128;
constexpr int FA_THREADS = 256;
constexpr int FA_SMEM = 16384 * 5 + 1024 /*align*/ + 256 /*barriers*/;
constexpr float FA_YMAX = 0.75f;

// tanh(y) ~= y * (C0 + C1 u + C2 u^2 + C3 u^3 + C4 u^4), u = y^2, |y| <= 0.75, abs err 2.6e-7 (minimax fit, fp32 Horner)
#define FA_C0 9.9999722832e-01f
#define FA_C1 -3.3323076483e-01f
#define FA_C2 1.3226091649e-01f
#define FA_C3 -4.9280448379e-02f
#define FA_C4 1.2318833231e-02f

// params[0] = 1 if the fast path is valid for this layer, params[1] = m (upper bound of the soft-capped logits, natural units)
__global__ void attn_fast_params_k(const float* __restrict__ gq, const float* __restrict__ gk, int n, float scale, float cap, float* __restrict__ params) {
  const int lane = threadIdx.x;
  float a = 0.f, b = 0.f;
  for (int i = lane; i < n; i += 32) { a = fmaxf(a, fabsf(gq[i] + 1.f)); b = fmaxf(b, fabsf(gk[i] + 1.f)); }
  a = warp_max(a); b = warp_max(b);
  if (lane == 0) {
    // |q| <= sqrt(n) * a, |k| <= sqrt(n) * b (RMSNorm scale sqrt(n), rotation preserves norms); 1.01 covers the bf16 rounding of q, k
    const float xmax = 1.01f * (float)n * a * b * scale;
    const float ymax = xmax / cap;
    params[0] = (ymax <= FA_YMAX && isfinite(ymax)) ? 1.f : 0.f;
    params[1] = xmax;
  }
}

__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// coefficients of e2(x) = x * (a0 + a1 X + a2 X^2 + a3 X^3 + a4 X^4) = cap * log2(e) * tanh(x * scale / cap), X = x^2
struct FaPoly {
  float a0, a1, a2, a3, a4;
  __device__ __forceinline__ FaPoly(float scale, float cap) {
    const float k1 = scale / cap, KL = cap * 1.4426950408889634f, k2 = k1 * k1;
    a0 = KL * k1 * FA_C0; a1 = KL * k1 * k2 * FA_C1; a2 = KL * k1 * k2 * k2 * FA_C2; a3 = KL * k1 * k2 * k2 * k2 * FA_C3; a4 = KL * k1 * k2 * k2 * k2 * k2 * FA_C4;
  }
  __device__ __forceinline__ float operator()(float x) const { return x * tail(x); }
  // e2(x) - m, the subtraction folded into the last multiply
  __device__ __forceinline__ float minus(float x, float m) const { return fmaf(x, tail(x), -m); }
  __device__ __forceinline__ float tail(float x) const {
    const float X = x * x;
    float g = fmaf(a4, X, a3);
    g = fmaf(g, X, a2);
    g = fmaf(g, X, a1);
    return fmaf(g, X, a0);
  }
};

// p = 2^(e2(x) - m2) of one 128-key tile for this thread's rows (a, b), row sums, P packed into the A fragments of the PV product
// (16 keys per fragment).  MASKED = false: the warp's 16 rows see every key of the tile.
template <bool MASKED>
__device__ __forceinline__ void fwd_p(const float (&s)[64], uint32_t (&pf)[8][4], float& l_a, float& l_b, int key0, int lim_a, int lim_b,
                                      const FaPoly& poly, float m2, int t) {
#pragma unroll
  for (int n8 = 0; n8 < 16; ++n8) {
    const int key = key0 + n8 * 8 + 2 * t;
    float p0 = ex2_approx(poly.minus(s[4 * n8], m2)), p1 = ex2_approx(poly.minus(s[4 * n8 + 1], m2));
    float p2 = ex2_approx(poly.minus(s[4 * n8 + 2], m2)), p3 = ex2_approx(poly.minus(s[4 * n8 + 3], m2));
    if (MASKED) {
      p0 = key <= lim_a ? p0 : 0.f; p1 = key + 1 <= lim_a ? p1 : 0.f;
      p2 = key <= lim_b ? p2 : 0.f; p3 = key + 1 <= lim_b ? p3 : 0.f;
    }
    l_a += p0 + p1; l_b += p2 + p3;
    pf[n8 >> 1][(n8 & 1) * 2] = pack_bf16(p0, p1);
    pf[n8 >> 1][(n8 & 1) * 2 + 1] = pack_bf16(p2, p3);
  }
}

__global__ void __launch_bounds__(FA_THREADS, 2)
attn_fwd_tc_k(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
              const float* __restrict__ gates, int H, const int* __restrict__ kv_limit, const int* __restrict__ tile_q0, const int* __restrict__ tile_qend,
              const int* __restrict__ tile_kv0, const int* __restrict__ tile_kvend, __nv_bfloat16* __restrict__ o, long long ld_o, float* __restrict__ lse,
              int M, float scale, float cap, const float* __restrict__ fast) {
  if (fast[0] == 0.f) return;                       // precondition of this path does not hold: the general kernel does the work
  extern __shared__ uint8_t fa_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(fa_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                                // [128 rows][128 B]
  uint8_t* sK = smem + 16384;                        // [2][128 keys][128 B]
  uint8_t* sV = smem + 49152;                        // [2][128 keys][128 B]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 81920);
  uint64_t *q_full = bars, *kv_full = bars + 1;     // kv_full[2]

  const int tile = gridDim.x - 1 - blockIdx.x;      // heavy (late) tiles first
  const int head = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cwg = warp >> 2, w4 = warp & 3, g = lane >> 2, t = lane & 3;
  const int q0 = tile_q0[tile], q_end = tile_qend[tile], kv0 = tile_kv0[tile], kv_end = tile_kvend[tile];
  const int n_kv = (kv_end - kv0 + FA_BN - 1) / FA_BN;

  if (tid == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1); mbar_init(&kv_full[0], 1); mbar_init(&kv_full[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(q_full, 16384);
    tma_load_2d(&tmQ, q_full, sQ, head * 64, q0);
    for (int j = 0; j < 2 && j < n_kv; ++j) {
      mbar_expect_tx(&kv_full[j], 32768);
      tma_load_2d(&tmK, &kv_full[j], sK + j * 16384, head * 64, kv0 + j * FA_BN);
      tma_load_2d(&tmV, &kv_full[j], sV + j * 16384, head * 64, kv0 + j * FA_BN);
    }
  }

  const int row_a = q0 + cwg * 64 + w4 * 16 + g, row_b = row_a + 8;
  const int lim_a = row_a < q_end ? kv_limit[row_a] : -1;
  const int lim_b = row_b < q_end ? kv_limit[row_b] : -1;
  const FaPoly poly(scale, cap);
  const float m2 = fast[1] * 1.4426950408889634f;
  float oacc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) oacc[i] = 0.f;
  float l_a = 0.f, l_b = 0.f;
  const uint32_t aQ = smem_u32(sQ) + cwg * 8192;
  mbar_wait(q_full, 0);

  for (int j = 0; j < n_kv; ++j) {
    const int b = j & 1;
    mbar_wait(&kv_full[b], (j >> 1) & 1);
    const uint32_t aK = smem_u32(sK + b * 16384), aV = smem_u32(sV + b * 16384);
    float s[64];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n128_ss<0, 0>(s, wgmma_desc_sw128(aQ + k * 32, 16, 1024), wgmma_desc_sw128(aK + k * 32, 16, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(s);
    // ---- p = 2^(e2(x) - m2), span mask only where some row of the warp does not see the whole tile
    const int key0 = kv0 + j * FA_BN;
    uint32_t pf[8][4];
    if (__all_sync(0xffffffffu, key0 + FA_BN - 1 <= min(lim_a, lim_b))) fwd_p<false>(s, pf, l_a, l_b, key0, lim_a, lim_b, poly, m2, t);
    else fwd_p<true>(s, pf, l_a, l_b, key0, lim_a, lim_b, poly, m2, t);
    // ---- O += P V_j
    wgmma_reg_fence(oacc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_m64n64_rs<1>(oacc, pf[kk], wgmma_desc_sw128(aV + kk * 2048, 8192, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(oacc);
    __syncthreads();                                 // both warpgroups are done with K_j / V_j: refill the slot with tile j + 2
    if (tid == 0 && j + 2 < n_kv) {
      mbar_expect_tx(&kv_full[b], 32768);
      tma_load_2d(&tmK, &kv_full[b], sK + b * 16384, head * 64, kv0 + (j + 2) * FA_BN);
      tma_load_2d(&tmV, &kv_full[b], sV + b * 16384, head * 64, kv0 + (j + 2) * FA_BN);
    }
  }
  // ---- epilogue: O / l * sigmoid(gate) -> bf16
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1); l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1); l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
  float ga = l_a > 0.f ? 1.f / l_a : 0.f, gb = l_b > 0.f ? 1.f / l_b : 0.f;
  if (gates) {
    if (row_a < q_end) ga *= 1.f / (1.f + __expf(-gates[(long long)row_a * H + head]));
    if (row_b < q_end) gb *= 1.f / (1.f + __expf(-gates[(long long)row_b * H + head]));
  }
  if (row_a < q_end) {
    __nv_bfloat16* dst = o + (long long)row_a * ld_o + head * 64 + 2 * t;
#pragma unroll
    for (int n8 = 0; n8 < 8; ++n8) *reinterpret_cast<uint32_t*>(dst + n8 * 8) = pack_bf16(oacc[4 * n8] * ga, oacc[4 * n8 + 1] * ga);
    if (t == 0 && lse) lse[(long long)head * M + row_a] = fast[1] + logf(l_a);
  }
  if (row_b < q_end) {
    __nv_bfloat16* dst = o + (long long)row_b * ld_o + head * 64 + 2 * t;
#pragma unroll
    for (int n8 = 0; n8 < 8; ++n8) *reinterpret_cast<uint32_t*>(dst + n8 * 8) = pack_bf16(oacc[4 * n8 + 2] * gb, oacc[4 * n8 + 3] * gb);
    if (t == 0 && lse) lse[(long long)head * M + row_b] = fast[1] + logf(l_b);
  }
}


// ================================================================================================ backward (bounded-logit path)
// One CTA = one 128-key tile x one head; it sweeps the 64-row query steps that can see those keys.  Two warpgroups, 64 keys each.
// Q, dO and the step's kv_limit, lse and D rows arrive by TMA in a FB_STAGES-deep ring (full / empty mbarriers; a slot is released by
// one arrival per warp and refilled by thread 0 two steps later, so the warpgroups never meet at a CTA-wide barrier).  There is no
// producer warp: with one, ptxas caps the block at 168 registers (also after setmaxnreg) and the consumers need more.
// Transposed scores put the keys on the accumulator rows, so dV and dK accumulate in registers:
//   S^T = K Q^T, dP^T = V dO^T                     (wgmma 64x64x16, shared-memory operands; two commit groups, so p starts under dP^T)
//   p = 2^(e2(x) - lse2), ds = p (dp - D) scale (1 - tanh^2)   (mask key <= kv_limit[query] only on steps a warp does not fully see)
//   dV += P^T dO, dK += dS^T Q                     (P^T / dS^T as register A operands, dO / Q read MN-major)
//   dQ = dS K over all 128 keys                    (one warpgroup per step, alternating: both dS^T halves from shared memory, MN-major A)
// dQ goes to a swizzled fp32 tile and into dq by one bulk tensor reduce-add, so each dq element gets one add per CTA step.
constexpr int FB_BQ = 64;
constexpr int FB_THREADS = 256;
constexpr int FB_STAGES = 4;
constexpr int FB_STAGE = 16384;                                     // Q [64][128 B] then dO [64][128 B]
constexpr int FB_RING = 32768;                                      // after K, V
// per stage: kv_limit, lse, D of the step's queries, each as a box of FB_ROW_BOX elements that starts at the 16-byte boundary at or
// below the step's first query (TMA tile starts must be 16-byte aligned; sequences start anywhere)
constexpr int FB_ROW_BOX = FB_BQ + 4;
constexpr int FB_ROW_SLOT = 384, FB_ROWS_STAGE = 3 * FB_ROW_SLOT;
constexpr int FB_ROWS = FB_RING + FB_STAGES * FB_STAGE;
constexpr int FB_DS = FB_ROWS + ((FB_STAGES * FB_ROWS_STAGE + 1023) & ~1023); // dS^T [2 buffers][128 keys][64 queries] bf16, 128B-swizzled
constexpr int FB_DQ = FB_DS + 2 * 16384;                            // dQ fp32 [2 warpgroups][2 column halves][64 rows][32], 128B-swizzled
constexpr int FB_BAR = FB_DQ + 2 * 16384;
constexpr int FB_SMEM = FB_BAR + 256 + 1024 /*align*/;
// named barriers: 1 + b dS^T buffer b written by both warpgroups, 3 + b buffer b read by its dQ product, 5 + cw dQ tile of warpgroup cw
constexpr int FB_BAR_DS_FULL = 1, FB_BAR_DS_EMPTY = 3, FB_BAR_DQ = 5;

// P^T / dS^T of one 64-query step for this thread's keys key_a, key_b (accumulator rows) and queries 8 n8 + 2 t + {0, 1} (columns).
// Pass 1 (S^T ready): p, packed into pf; sacc becomes w = p scale (1 - tanh^2).  Pass 2 (dP^T ready): ds = w (dp - D), packed into dsf.
template <bool MASKED>
__device__ __forceinline__ void bwd_p(float (&sacc)[32], uint32_t (&pf)[4][4], const int* sLim, const float* sLse, int key_a, int key_b, int qvalid,
                                      const FaPoly& poly, float oms_c, float scale, int t) {
#pragma unroll
  for (int n8 = 0; n8 < 8; ++n8) {
    const int c0 = n8 * 8 + 2 * t;
    const float lse2[2] = {sLse[c0] * 1.4426950408889634f, sLse[c0 + 1] * 1.4426950408889634f};   // (rows are not 8-byte aligned)
    int lim[2] = {0, 0};
    if (MASKED) {
      lim[0] = c0 < qvalid ? sLim[c0] : -1;
      lim[1] = c0 + 1 < qvalid ? sLim[c0 + 1] : -1;
    }
    float pv[4];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int e = 4 * n8 + 2 * r + c;
        const float e2 = poly(sacc[e]);
        float p = ex2_approx(e2 - lse2[c]);
        if (MASKED) p = ((r == 0 ? key_a : key_b) <= lim[c]) ? p : 0.f;
        pv[2 * r + c] = p;
        sacc[e] = p * fmaf(e2 * e2, oms_c, scale);
      }
    pf[n8 >> 1][(n8 & 1) * 2] = pack_bf16(pv[0], pv[1]);
    pf[n8 >> 1][(n8 & 1) * 2 + 1] = pack_bf16(pv[2], pv[3]);
  }
}

__global__ void __launch_bounds__(FB_THREADS, 1)
attn_bwd_tc_k(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
              const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ CUtensorMap tmLim, const __grid_constant__ CUtensorMap tmLse,
              const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmDQ,
              const int* __restrict__ kt_kv0, const int* __restrict__ kt_kvend, const int* __restrict__ kt_q0, const int* __restrict__ kt_qend,
              const int* __restrict__ kt_order, float* __restrict__ dk, __nv_bfloat16* __restrict__ dv, long long ld_dv, int M, int H, float scale, float cap,
              const float* __restrict__ fast) {
  if (fast[0] == 0.f) return;
  extern __shared__ uint8_t fb_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(fb_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;                                // [128 keys][128 B]
  uint8_t* sV = smem + 16384;
  uint8_t* sDS = smem + FB_DS;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FB_BAR);
  uint64_t *full = bars, *empty = bars + FB_STAGES, *kv_full = bars + 2 * FB_STAGES;

  const int idx = blockIdx.x;
  const int tt = idx / H;
  const int tile = kt_order ? kt_order[tt] : tt;
  const int head = idx - tt * H;
  const int kv0 = kt_kv0[tile], kv_end = kt_kvend[tile], q_begin = kt_q0[tile], q_end = kt_qend[tile];
  const int n_q = (q_end - q_begin + FB_BQ - 1) / FB_BQ;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmDO);
    for (int s = 0; s < FB_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_init(kv_full, 1);
    mbar_fence_init();
  }
  __syncthreads();

  // Q / dO / row loads of step j into ring slot j % FB_STAGES (issued by thread 0)
  auto load_step = [&](int j) {
    const int sl = j % FB_STAGES;
    const int qb = q_begin + j * FB_BQ;
    uint8_t* st = smem + FB_RING + sl * FB_STAGE;
    uint8_t* rows = smem + FB_ROWS + sl * FB_ROWS_STAGE;
    mbar_expect_tx(&full[sl], FB_STAGE + 3 * FB_ROW_BOX * 4);
    tma_load_2d(&tmQ, &full[sl], st, head * 64, qb);
    tma_load_2d(&tmDO, &full[sl], st + 8192, head * 64, qb);
    // per-query rows (zero-filled past the end of the array; queries past q_end are masked)
    tma_load_1d(&tmLim, &full[sl], rows, qb & ~3);
    tma_load_1d(&tmLse, &full[sl], rows + FB_ROW_SLOT, (head * M + qb) & ~3);
    tma_load_1d(&tmD, &full[sl], rows + 2 * FB_ROW_SLOT, (head * M + qb) & ~3);
  };
  if (tid == 0) {
    mbar_expect_tx(kv_full, 32768);
    tma_load_2d(&tmK, kv_full, sK, head * 64, kv0);
    tma_load_2d(&tmV, kv_full, sV, head * 64, kv0);
    for (int j = 0; j < FB_STAGES && j < n_q; ++j) load_step(j);
  }
  const int cwg = warp >> 2, w4 = warp & 3, g = lane >> 2, t = lane & 3;
  const bool leader = (tid & 127) == 0;
  const FaPoly poly(scale, cap);
  const float KL = cap * 1.4426950408889634f;
  const float oms_c = -scale / (KL * KL);            // scale * (1 - tanh^2) = fma(e2^2, oms_c, scale)
  const int key_a = kv0 + cwg * 64 + w4 * 16 + g, key_b = key_a + 8;
  const int warp_key_last = kv0 + cwg * 64 + w4 * 16 + 15;
  float dvacc[32], dkacc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dvacc[i] = 0.f; dkacc[i] = 0.f; }
  const uint32_t aK = smem_u32(sK) + cwg * 8192, aV = smem_u32(sV) + cwg * 8192, aKall = smem_u32(sK);
  const int ds_row0 = cwg * 64 + w4 * 16 + g;        // this thread's two dS^T rows: ds_row0, ds_row0 + 8
  uint8_t* sDQ = smem + FB_DQ + cwg * 16384;
  mbar_wait(kv_full, 0);

  int s = 0; uint32_t phase = 0;
  for (int i = 0; i < n_q; ++i) {
    const int b = i & 1;                             // dS^T buffer of this step; warpgroup b computes its dQ
    const int qb = q_begin + i * FB_BQ;
    mbar_wait(&full[s], phase);
    const uint32_t aQ = smem_u32(smem + FB_RING + s * FB_STAGE), aDO = aQ + 8192;
    const int* sLim = reinterpret_cast<const int*>(smem + FB_ROWS + s * FB_ROWS_STAGE) + (qb & 3);
    const float* sLse = reinterpret_cast<const float*>(smem + FB_ROWS + s * FB_ROWS_STAGE + FB_ROW_SLOT) + ((head * M + qb) & 3);
    const float* sD = reinterpret_cast<const float*>(smem + FB_ROWS + s * FB_ROWS_STAGE + 2 * FB_ROW_SLOT) + ((head * M + qb) & 3);
    float sacc[32], pacc[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64_ss<0, 0>(sacc, wgmma_desc_sw128(aK + k * 32, 16, 1024), wgmma_desc_sw128(aQ + k * 32, 16, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64_ss<0, 0>(pacc, wgmma_desc_sw128(aV + k * 32, 16, 1024), wgmma_desc_sw128(aDO + k * 32, 16, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    // refill the slot of step i - 2 (both warpgroups have released it, or will shortly) with step i - 2 + FB_STAGES
    if (tid == 0 && i >= 2 && i - 2 + FB_STAGES < n_q) {
      mbar_wait(&empty[(i - 2) % FB_STAGES], ((i - 2) / FB_STAGES) & 1);
      load_step(i - 2 + FB_STAGES);
    }
    // this warp's 16 keys are visible to all 64 queries of the step: no mask
    const int qvalid = q_end - qb;
    const bool full_vis = qvalid >= FB_BQ && warp_key_last <= __reduce_min_sync(0xffffffffu, min(sLim[lane], sLim[lane + 32]));
    wgmma_wait<1>();
    wgmma_reg_fence(sacc);
    uint32_t pf[4][4], dsf[4][4];
    if (full_vis) bwd_p<false>(sacc, pf, sLim, sLse, key_a, key_b, qvalid, poly, oms_c, scale, t);
    else bwd_p<true>(sacc, pf, sLim, sLse, key_a, key_b, qvalid, poly, oms_c, scale, t);
    wgmma_wait<0>();
    wgmma_reg_fence(pacc);
#pragma unroll
    for (int n8 = 0; n8 < 8; ++n8) {
      const float d0 = sD[n8 * 8 + 2 * t], d1 = sD[n8 * 8 + 2 * t + 1];
      dsf[n8 >> 1][(n8 & 1) * 2] = pack_bf16(sacc[4 * n8] * (pacc[4 * n8] - d0), sacc[4 * n8 + 1] * (pacc[4 * n8 + 1] - d1));
      dsf[n8 >> 1][(n8 & 1) * 2 + 1] = pack_bf16(sacc[4 * n8 + 2] * (pacc[4 * n8 + 2] - d0), sacc[4 * n8 + 3] * (pacc[4 * n8 + 3] - d1));
    }
    // ---- dS^T -> shared buffer b (this warpgroup's 64 rows), once the dQ product of step i - 2 has finished reading it
    uint8_t* dsb = sDS + b * 16384;
    if (cwg != b && i >= 2) named_bar_sync(FB_BAR_DS_EMPTY + b, 256);
#pragma unroll
    for (int n8 = 0; n8 < 8; ++n8) {
      const int r0 = ds_row0, r1 = ds_row0 + 8;
      *reinterpret_cast<uint32_t*>(dsb + r0 * 128 + ((n8 ^ (r0 & 7)) << 4) + t * 4) = dsf[n8 >> 1][(n8 & 1) * 2];
      *reinterpret_cast<uint32_t*>(dsb + r1 * 128 + ((n8 ^ (r1 & 7)) << 4) + t * 4) = dsf[n8 >> 1][(n8 & 1) * 2 + 1];
    }
    fence_proxy_async_smem();
    if (cwg == b) named_bar_sync(FB_BAR_DS_FULL + b, 256);
    else named_bar_arrive(FB_BAR_DS_FULL + b, 256);
    // ---- dV += P^T dO, dK += dS^T Q (this warpgroup's keys); on its steps, dQ = dS K (all 128 keys)
    wgmma_reg_fence(dvacc);
    wgmma_reg_fence(dkacc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64_rs<1>(dvacc, pf[kk], wgmma_desc_sw128(aDO + kk * 2048, 8192, 1024), 1u);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64_rs<1>(dkacc, dsf[kk], wgmma_desc_sw128(aQ + kk * 2048, 8192, 1024), 1u);
    wgmma_commit();
    if (cwg == b) {
      float qacc[32];
      const uint32_t aDS = smem_u32(dsb);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_m64n64_ss<1, 1>(qacc, wgmma_desc_sw128(aDS + kk * 2048, 8192, 1024), wgmma_desc_sw128(aKall + kk * 2048, 8192, 1024), kk > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(dvacc);
      wgmma_reg_fence(dkacc);
      wgmma_reg_fence(qacc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      if (i + 2 < n_q) named_bar_arrive(FB_BAR_DS_EMPTY + b, 256);
      // ---- dQ -> fp32 tile (two 32-column halves, 128B-swizzled like the tensor map) -> one bulk reduce-add into dq
      if (leader) bulk_wait_read_all();
      named_bar_sync(FB_BAR_DQ + cwg, 128);
      const int r0 = w4 * 16 + g, r1 = r0 + 8;
#pragma unroll
      for (int n8 = 0; n8 < 8; ++n8) {
        const int chunk = 2 * (n8 & 3) + (t >> 1), off = (n8 >> 2) * 8192 + (t & 1) * 8;
        *reinterpret_cast<float2*>(sDQ + off + r0 * 128 + ((chunk ^ (r0 & 7)) << 4)) = make_float2(qacc[4 * n8], qacc[4 * n8 + 1]);
        *reinterpret_cast<float2*>(sDQ + off + r1 * 128 + ((chunk ^ (r1 & 7)) << 4)) = make_float2(qacc[4 * n8 + 2], qacc[4 * n8 + 3]);
      }
      fence_proxy_async_smem();
      named_bar_sync(FB_BAR_DQ + cwg, 128);
      if (leader) {
        tma_reduce_add_2d(&tmDQ, sDQ, head * 64, qb);
        tma_reduce_add_2d(&tmDQ, sDQ + 8192, head * 64 + 32, qb);
        bulk_commit();
      }
    } else {
      wgmma_wait<0>();
      wgmma_reg_fence(dvacc);
      wgmma_reg_fence(dkacc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    if (++s == FB_STAGES) { s = 0; phase ^= 1; }
  }
  if (leader) bulk_wait_all();
  // ---- dK (fp32) and dV (bf16) of this key tile
#pragma unroll
  for (int n8 = 0; n8 < 8; ++n8) {
    if (key_a < kv_end) {
      *reinterpret_cast<float2*>(dk + (long long)key_a * H * 64 + head * 64 + n8 * 8 + 2 * t) = make_float2(dkacc[4 * n8], dkacc[4 * n8 + 1]);
      *reinterpret_cast<uint32_t*>(dv + (long long)key_a * ld_dv + head * 64 + n8 * 8 + 2 * t) = pack_bf16(dvacc[4 * n8], dvacc[4 * n8 + 1]);
    }
    if (key_b < kv_end) {
      *reinterpret_cast<float2*>(dk + (long long)key_b * H * 64 + head * 64 + n8 * 8 + 2 * t) = make_float2(dkacc[4 * n8 + 2], dkacc[4 * n8 + 3]);
      *reinterpret_cast<uint32_t*>(dv + (long long)key_b * ld_dv + head * 64 + n8 * 8 + 2 * t) = pack_bf16(dvacc[4 * n8 + 2], dvacc[4 * n8 + 3]);
    }
  }
}

// 1-D map of n 4-byte elements (fp32 or int32), box of FB_ROW_BOX elements, zero fill past the end
inline int make_tmap_rows(CUtensorMap* tm, CUtensorMapDataType type, const void* ptr, long long n) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return -1;
  cuuint64_t dims[1] = {(cuuint64_t)n};
  cuuint64_t strides[1] = {0};
  cuuint32_t box[1] = {FB_ROW_BOX}, estr[1] = {1};
  CUresult r = enc(tm, type, 1, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -(int)r - 1000;
}

// dq [M][H * 64] fp32: box of 32 columns (128 B, the swizzle span) x FB_BQ rows, 128-byte swizzle
inline int make_tmap_dq(CUtensorMap* tm, float* dq, int M, int H) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return -1;
  cuuint64_t dims[2] = {(cuuint64_t)H * 64, (cuuint64_t)M};
  cuuint64_t strides[1] = {(cuuint64_t)H * 64 * 4};
  cuuint32_t box[2] = {32, FB_BQ}, estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, dq, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -(int)r - 1000;
}

}  // namespace tfx

using namespace tfx;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int tfx_attn_fast_params(const float* q_gamma, const float* k_gamma, int dim_head, float scale, float softcap, float* params, void* stream) {
  TFX_REQUIRE(dim_head > 0 && softcap > 0.f, "attn_fast_params: bad arguments");
  attn_fast_params_k<<<1, 32, 0, ST(stream)>>>(q_gamma, k_gamma, dim_head, scale, softcap, params);
  return check_launch("attn_fast_params");
}

int tfx_attn_fwd_tc(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H,
                    const int* kv_limit, const int* tile_q0, const int* tile_qend, const int* tile_kv0, const int* tile_kvend, int n_tiles,
                    void* o, long long ld_o, float* lse, int M, int M_kv, float scale, float softcap, const float* fast_params, void* stream) {
  if (n_tiles <= 0) return 0;
  if (M_kv <= 0) M_kv = M;
  TFX_REQUIRE(fast_params != nullptr, "attn_fwd_tc: fast_params (from tfx_attn_fast_params) is required");
  TFX_REQUIRE(ld_q % 8 == 0 && ld_k % 8 == 0 && ld_v % 8 == 0 && ld_o % 8 == 0, "attn_fwd_tc: row pitches must be multiples of 8 bf16");
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_tmap_bf16(&tq, q, (long long)H * 64, M, ld_q, FA_BM)) || (rc = make_tmap_bf16(&tk, k, (long long)H * 64, M_kv, ld_k, FA_BN)) ||
      (rc = make_tmap_bf16(&tv, v, (long long)H * 64, M_kv, ld_v, FA_BN))) {
    set_error("attn_fwd_tc: cuTensorMapEncodeTiled failed (%d)", rc);
    return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(attn_fwd_tc_k, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM) != cudaSuccess) { set_error("attn_fwd_tc: cannot raise dynamic smem"); return -2; }
    attr_set = true;
  }
  attn_fwd_tc_k<<<dim3(n_tiles, H), FA_THREADS, FA_SMEM, ST(stream)>>>(tq, tk, tv, gates, H, kv_limit, tile_q0, tile_qend, tile_kv0, tile_kvend, (__nv_bfloat16*)o, ld_o, lse, M,
                                                                      scale, softcap, fast_params);
  return check_launch("attn_fwd_tc");
}

int tfx_attn_bwd_tc(const void* q, const void* k, const void* v, const void* do_pre, long long ld_q, long long ld_k, long long ld_v, long long ld_do,
                    const float* lse, const float* dsum_hm, const int* kv_limit, const int* kt_kv0, const int* kt_kvend, const int* kt_q0, const int* kt_qend,
                    const int* kt_order, int n_kv_tiles, float* dq, float* dk, void* dv, long long ld_dv, int M, int H, float scale, float softcap, const float* fast_params,
                    void* stream) {
  if (n_kv_tiles <= 0) return 0;
  TFX_REQUIRE(fast_params != nullptr, "attn_bwd_tc: fast_params (from tfx_attn_fast_params) is required");
  TFX_REQUIRE(ld_q % 8 == 0 && ld_k % 8 == 0 && ld_v % 8 == 0 && ld_do % 8 == 0 && ld_dv % 8 == 0, "attn_bwd_tc: row pitches must be multiples of 8 bf16");
  CUtensorMap tq, tk, tv, tdo, tlim, tlse, td, tdq;
  int rc;
  if ((rc = make_tmap_bf16(&tq, q, (long long)H * 64, M, ld_q, FB_BQ)) || (rc = make_tmap_bf16(&tk, k, (long long)H * 64, M, ld_k, FA_BN)) ||
      (rc = make_tmap_bf16(&tv, v, (long long)H * 64, M, ld_v, FA_BN)) || (rc = make_tmap_bf16(&tdo, do_pre, (long long)H * 64, M, ld_do, FB_BQ)) ||
      (rc = make_tmap_rows(&tlim, CU_TENSOR_MAP_DATA_TYPE_INT32, kv_limit, M)) || (rc = make_tmap_rows(&tlse, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, lse, (long long)H * M)) ||
      (rc = make_tmap_rows(&td, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, dsum_hm, (long long)H * M)) || (rc = make_tmap_dq(&tdq, dq, M, H))) {
    set_error("attn_bwd_tc: cuTensorMapEncodeTiled failed (%d): kv_limit, lse, dsum and dq must be 16-byte aligned", rc);
    return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(attn_bwd_tc_k, cudaFuncAttributeMaxDynamicSharedMemorySize, FB_SMEM) != cudaSuccess) { set_error("attn_bwd_tc: cannot raise dynamic smem"); return -2; }
    attr_set = true;
  }
  attn_bwd_tc_k<<<n_kv_tiles * H, FB_THREADS, FB_SMEM, ST(stream)>>>(tq, tk, tv, tdo, tlim, tlse, td, tdq, kt_kv0, kt_kvend, kt_q0, kt_qend, kt_order, dk,
                                                                     (__nv_bfloat16*)dv, ld_dv, M, H, scale, softcap, fast_params);
  return check_launch("attn_bwd_tc");
}

}  // extern "C"
