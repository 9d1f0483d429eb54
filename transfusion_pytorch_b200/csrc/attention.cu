// Fused span-masked, soft-capped attention for packed ragged sequences (forward + backward).
//
// Semantics (reference: transfusion_pytorch/transfusion.py:998-1027 with the mask of
// :452-470 / :315-338):   s = (q . k) * dh^-1/2 ;  s = cap * tanh(s / cap) ;  visible(i, j) <=> j <= kv_limit[i]
// (kv_limit[i] = i for text, = last token of the span for tokens inside a modality span) ;
// o = softmax_j(s) v ;  o *= sigmoid(gate[i, head]).
// The mask is evaluated from one int per query row in registers - no N x N mask or score tensor exists.
//
// Layout: token-major q/k/v/o [M_total][heads*DH] bf16 (head dim DH = 64 or 128), sequences packed back to back; 64-row tiles
// never straddle a sequence (host builds the tile tables).  The forward and the backward pre-pass are templates on DH; the backward main
// pass is attn_bwd_k at 64 and attn_bwd_dh_k (8 warps) at 128.
// Math: bf16 mma.sync m16n8k16 with fp32 accumulation, online softmax in registers (FlashAttention-2
// schedule).  The score path is MUFU-bound (tanh + exp per score), not tensor-bound, at head dim 64.
#include "common.cuh"
#include "../../include/tfx_b200.h"

namespace tfx {

constexpr int ATT_BM = 64, ATT_BN = 64, ATT_THREADS = 128;
constexpr int ATT_BWD_SMEM = 7 * 64 * 64 * 2 + 6 * 64 * 4;
// attn_fwd_k: Q and the K / V double buffers
constexpr int att_fwd_smem(int dh) { return 5 * 64 * dh * 2; }
// head dim 128 (attn_bwd_dh_k below): K, V, double-buffered Q / dO, dS^T, the dS weights of the four key groups and the per-query rows
constexpr int ATT_BWD_THREADS_D128 = 256;
constexpr int ATT_BWD_SMEM_D128 = 6 * 64 * 128 * 2 + 64 * 64 * 2 + 4 * 16 * 64 * 4 + 6 * 64 * 4;

__device__ __forceinline__ uint32_t s_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s_u32(smem)), "l"(gmem), "r"(sz) : "memory");
}
// (cp_async_commit / cp_async_wait<N>: common.cuh)

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// tile element (row, 16-byte chunk) -> swizzled bf16 offset inside a [64][DH] tile (the xor stays inside each group of 8 chunks)
template <int DH>
__device__ __forceinline__ int swz(int row, int chunk) { return row * DH + ((chunk ^ (row & 7)) << 3); }

// cooperative async load of a [64 rows][DH bf16] tile by NT threads; rows >= row_end are zero filled
template <int DH, int NT = ATT_THREADS>
__device__ __forceinline__ void load_tile(__nv_bfloat16* s, const __nv_bfloat16* g, long long ld, int row0, int row_end, int tid) {
  constexpr int SH = DH == 64 ? 3 : 4;       // log2 of the 16-byte chunks per row
#pragma unroll
  for (int it = 0; it < 64 * DH / 8 / NT; ++it) {
    const int idx = tid + it * NT;
    const int r = idx >> SH, ch = idx & ((1 << SH) - 1);
    const bool ok = row0 + r < row_end;
    const __nv_bfloat16* src = g + (long long)(ok ? row0 + r : row0) * ld + ch * 8;
    cp_async16(s + swz<DH>(r, ch), src, ok);
  }
}

// ================================================================================================ forward
// One CTA per (64-query tile, head), 4 warps of 16 query rows; K / V tiles double-buffered through cp.async.  The whole head is held in
// registers (oacc DH / 2, qf DH / 4 per thread).
template <int DH>
__global__ void __launch_bounds__(ATT_THREADS) attn_fwd_k(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v,
                                                         long long ld_q, long long ld_k, long long ld_v, const float* __restrict__ gates, int H,
                                                         const int* __restrict__ kv_limit, const int* __restrict__ tile_q0, const int* __restrict__ tile_qend,
                                                         const int* __restrict__ tile_kv0, const int* __restrict__ tile_kvend, __nv_bfloat16* __restrict__ o,
                                                         long long ld_o, float* __restrict__ lse, int M, float scale, float cap, const float* __restrict__ skip_if_fast) {
  // the bounded-logit wgmma kernel (attention_sm90.cu, head dim 64 only) handles this layer
  if (DH == 64 && skip_if_fast && skip_if_fast[0] != 0.f) return;
  constexpr int TILE = 64 * DH;
  __nv_bfloat16* sQ;
  __nv_bfloat16 (*sK)[TILE];     // [2][TILE]
  __nv_bfloat16 (*sV)[TILE];     // [2][TILE]
  if constexpr (DH == 64) {          // 40 KB fit in static shared memory; the 80 KB of DH = 128 need the dynamic opt-in
    __shared__ __align__(128) __nv_bfloat16 sQs[TILE];
    __shared__ __align__(128) __nv_bfloat16 sKs[2][TILE];
    __shared__ __align__(128) __nv_bfloat16 sVs[2][TILE];
    sQ = sQs; sK = sKs; sV = sVs;
  } else {
    extern __shared__ __align__(128) uint8_t att_smem[];
    sQ = reinterpret_cast<__nv_bfloat16*>(att_smem);
    sK = reinterpret_cast<__nv_bfloat16 (*)[TILE]>(sQ + TILE);
    sV = reinterpret_cast<__nv_bfloat16 (*)[TILE]>(sQ + 3 * TILE);
  }
  const int tile = gridDim.x - 1 - blockIdx.x;      // heavy (late) tiles first
  const int head = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int q0 = tile_q0[tile], q_end = tile_qend[tile], kv0 = tile_kv0[tile], kv_end = tile_kvend[tile];
  const __nv_bfloat16* qh = q + head * DH;
  const __nv_bfloat16* kh = k + head * DH;
  const __nv_bfloat16* vh = v + head * DH;

  load_tile<DH>(sQ, qh, ld_q, q0, q_end, tid);
  const int n_kv = (kv_end - kv0 + ATT_BN - 1) / ATT_BN;
  load_tile<DH>(sK[0], kh, ld_k, kv0, kv_end, tid);
  load_tile<DH>(sV[0], vh, ld_v, kv0, kv_end, tid);
  cp_async_commit();

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const int lim_a = row_a < q_end ? kv_limit[row_a] : -1;
  const int lim_b = row_b < q_end ? kv_limit[row_b] : -1;
  // warp-level upper bound on visible keys: lets a warp skip KV tiles that are fully masked for its 16 rows
  int wlim = max(lim_a, lim_b);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) wlim = max(wlim, __shfl_xor_sync(0xffffffffu, wlim, off));

  float oacc[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f; }
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
  uint32_t qf[DH / 16][4];
  const float inv_cap = 1.f / cap;
  const float LOG2E = 1.4426950408889634f;

  for (int j = 0; j < n_kv; ++j) {
    const int buf = j & 1;
    if (j + 1 < n_kv) {
      load_tile<DH>(sK[buf ^ 1], kh, ld_k, kv0 + (j + 1) * ATT_BN, kv_end, tid);
      load_tile<DH>(sV[buf ^ 1], vh, ld_v, kv0 + (j + 1) * ATT_BN, kv_end, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (j == 0) {
#pragma unroll
      for (int ks = 0; ks < DH / 16; ++ks) {
        const int mat = lane >> 3;
        const int row = warp * 16 + (mat & 1) * 8 + (lane & 7);
        ldsm_x4(s_u32(sQ + swz<DH>(row, ks * 2 + (mat >> 1))), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
      }
    }
    const int key0 = kv0 + j * ATT_BN;
    if (key0 <= wlim) {
      // ---- S = Q K^T
      float sacc[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) { sacc[i][0] = sacc[i][1] = sacc[i][2] = sacc[i][3] = 0.f; }
#pragma unroll
      for (int ks = 0; ks < DH / 16; ++ks) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          const int mat = lane >> 3;
          const int row = np * 16 + (mat >> 1) * 8 + (lane & 7);
          uint32_t b0, b1, b2, b3;
          ldsm_x4(s_u32(sK[buf] + swz<DH>(row, ks * 2 + (mat & 1))), b0, b1, b2, b3);
          mma_bf16(sacc[2 * np], qf[ks], b0, b1);
          mma_bf16(sacc[2 * np + 1], qf[ks], b2, b3);
        }
      }
      // ---- soft-cap, mask, online softmax
      float mx_a = m_a, mx_b = m_b;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + nt * 8 + 2 * t + (e & 1);
          const int lim = (e < 2) ? lim_a : lim_b;
          float s = cap * tanh_acc(sacc[nt][e] * scale * inv_cap);
          s = key <= lim ? s : -INFINITY;
          sacc[nt][e] = s;
          if (e < 2) mx_a = fmaxf(mx_a, s); else mx_b = fmaxf(mx_b, s);
        }
      }
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1)); mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1)); mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
      const float ma_s = mx_a == -INFINITY ? 0.f : mx_a, mb_s = mx_b == -INFINITY ? 0.f : mx_b;   // fully masked rows stay at p = 0
      const float ca = exp2f((m_a - ma_s) * LOG2E), cb = exp2f((m_b - mb_s) * LOG2E);
      m_a = mx_a; m_b = mx_b;
      float ra = 0.f, rb = 0.f;
      uint32_t pf[4][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float p0 = exp2f((sacc[nt][0] - ma_s) * LOG2E), p1 = exp2f((sacc[nt][1] - ma_s) * LOG2E);
        const float p2 = exp2f((sacc[nt][2] - mb_s) * LOG2E), p3 = exp2f((sacc[nt][3] - mb_s) * LOG2E);
        ra += p0 + p1; rb += p2 + p3;
        pf[nt >> 1][(nt & 1) * 2] = pack2_bf16(p0, p1);
        pf[nt >> 1][(nt & 1) * 2 + 1] = pack2_bf16(p2, p3);
      }
      l_a = l_a * ca + ra; l_b = l_b * cb + rb;
#pragma unroll
      for (int i = 0; i < DH / 8; ++i) { oacc[i][0] *= ca; oacc[i][1] *= ca; oacc[i][2] *= cb; oacc[i][3] *= cb; }
      // ---- O += P V
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int dp = 0; dp < DH / 16; ++dp) {
          const int mat = lane >> 3;
          const int row = kk * 16 + (mat & 1) * 8 + (lane & 7);
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(s_u32(sV[buf] + swz<DH>(row, dp * 2 + (mat >> 1))), b0, b1, b2, b3);
          mma_bf16(oacc[2 * dp], pf[kk], b0, b1);
          mma_bf16(oacc[2 * dp + 1], pf[kk], b2, b3);
        }
      }
    }
    __syncthreads();
  }
  // ---- epilogue: normalise, value gate, store
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1); l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1); l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
  const float ia = l_a > 0.f ? 1.f / l_a : 0.f, ib = l_b > 0.f ? 1.f / l_b : 0.f;
  float ga = 1.f, gb = 1.f;
  if (gates) {
    if (row_a < q_end) ga = 1.f / (1.f + __expf(-gates[(long long)row_a * H + head]));
    if (row_b < q_end) gb = 1.f / (1.f + __expf(-gates[(long long)row_b * H + head]));
  }
  if (row_a < q_end) {
    __nv_bfloat16* dst = o + (long long)row_a * ld_o + head * DH + 2 * t;
#pragma unroll
    for (int nt = 0; nt < DH / 8; ++nt) *reinterpret_cast<uint32_t*>(dst + nt * 8) = pack2_bf16(oacc[nt][0] * ia * ga, oacc[nt][1] * ia * ga);
    if (t == 0 && lse) lse[(long long)head * M + row_a] = m_a + logf(l_a);
  }
  if (row_b < q_end) {
    __nv_bfloat16* dst = o + (long long)row_b * ld_o + head * DH + 2 * t;
#pragma unroll
    for (int nt = 0; nt < DH / 8; ++nt) *reinterpret_cast<uint32_t*>(dst + nt * 8) = pack2_bf16(oacc[nt][2] * ib * gb, oacc[nt][3] * ib * gb);
    if (t == 0 && lse) lse[(long long)head * M + row_b] = m_b + logf(l_b);
  }
}

// ================================================================================================ backward
// pre-pass (one warp per token): dsum[h][row] = sum_d dO_gated*O_gated ; dO_pre = dO_gated * sigmoid(gate) ; dq accumulator cleared.
// DH / 8 lanes share a head (16-byte bf16 accesses; 8 at DH = 64, 16 at 128), 32 / (DH / 8) heads per pass, the per-head dot product is a
// log2(DH / 8)-step shuffle.
template <int DH>
__global__ void __launch_bounds__(ROW_THREADS) attn_bwd_prep_k(const __nv_bfloat16* __restrict__ dog, const __nv_bfloat16* __restrict__ og, const float* __restrict__ gates,
                                                              __nv_bfloat16* __restrict__ dop, float* __restrict__ dsum, float* __restrict__ dsum_rowmajor,
                                                              float* __restrict__ dq_zero, int M, int H) {
  constexpr int LPH = DH / 8, HPP = 32 / LPH;
  const int lane = threadIdx.x & 31, sub = lane % LPH, hq = (lane >> 3) / (LPH / 8);
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const int HI = H * DH;
  for (int row = warp0; row < M; row += nwarps) {
    for (int h0 = 0; h0 < H; h0 += HPP) {
      const int h = h0 + hq;
      const bool act = h < H;
      const long long off = (long long)row * HI + (act ? h : 0) * DH + sub * 8;
      const uint4 a4 = *reinterpret_cast<const uint4*>(dog + off), b4 = *reinterpret_cast<const uint4*>(og + off);
      const float sg = (act && gates) ? 1.f / (1.f + __expf(-gates[(long long)row * H + h])) : 1.f;
      const uint32_t aw[4] = {a4.x, a4.y, a4.z, a4.w}, bw[4] = {b4.x, b4.y, b4.z, b4.w};
      uint32_t ow[4];
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = unpack2_bf16(aw[e]), b = unpack2_bf16(bw[e]);
        s += a.x * b.x + a.y * b.y;
        ow[e] = pack2_bf16(a.x * sg, a.y * sg);
      }
#pragma unroll
      for (int o = 1; o < LPH; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (act) {
        *reinterpret_cast<uint4*>(dop + off) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        if (sub == 0) { dsum[(long long)h * M + row] = s; if (dsum_rowmajor) dsum_rowmajor[(long long)row * H + h] = s; }
        if (dq_zero) {
          *reinterpret_cast<float4*>(dq_zero + off) = make_float4(0.f, 0.f, 0.f, 0.f);
          *reinterpret_cast<float4*>(dq_zero + off + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
  }
}

// main pass: one CTA per (64-key tile, head); each warp owns 16 keys and sweeps the query tiles that can see them.
// Works on the transposed score tile S^T [keys x queries] so that dV, dK accumulate in registers per warp;
// dS^T goes through shared memory once to produce the dQ contribution, which is atomically added (fp32).
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_k(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v,
                                                         const __nv_bfloat16* __restrict__ dop, long long ld_q, long long ld_k, long long ld_v, long long ld_do,
                                                         const float* __restrict__ lse, const float* __restrict__ dsum, const int* __restrict__ kv_limit,
                                                         const int* __restrict__ kt_kv0, const int* __restrict__ kt_kvend, const int* __restrict__ kt_q0,
                                                         const int* __restrict__ kt_qend, float* __restrict__ dq, float* __restrict__ dk,
                                                         __nv_bfloat16* __restrict__ dv, long long ld_dv, int M, int H, float scale, float cap, const float* __restrict__ skip_if_fast) {
  if (skip_if_fast && skip_if_fast[0] != 0.f) return;     // the bounded-logit wgmma kernel (attention_sm90.cu) handles this layer
  extern __shared__ __align__(128) uint8_t att_smem[];
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(att_smem);
  __nv_bfloat16* sV = sK + 64 * 64;
  __nv_bfloat16* sQb = sV + 64 * 64;          // [2][64*64]
  __nv_bfloat16* sDOb = sV + 3 * 64 * 64;     // [2][64*64]
  __nv_bfloat16* sDS = sV + 5 * 64 * 64;      // dS^T [key][query]
  float* sLseb = reinterpret_cast<float*>(sDS + 64 * 64);   // [2][64]
  float* sDb = sLseb + 128;                                  // [2][64]
  int* sLimb = reinterpret_cast<int*>(sLseb + 256);          // [2][64]
#define sQ_(b) (sQb + (b) * 4096)
#define sDO_(b) (sDOb + (b) * 4096)
#define sLse_(b) (sLseb + (b) * 64)
#define sD_(b) (sDb + (b) * 64)
#define sLim_(b) (sLimb + (b) * 64)
  const int tile = blockIdx.x, head = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int kv0 = kt_kv0[tile], kv_end = kt_kvend[tile], q_begin = kt_q0[tile], q_end = kt_qend[tile];
  const int HI = H * 64;
  const __nv_bfloat16* qh = q + head * 64;
  const __nv_bfloat16* doh = dop + head * 64;
  const float* lse_h = lse + (long long)head * M;
  const float* ds_h = dsum + (long long)head * M;
  const int n_q = (q_end - q_begin + 63) / 64;

  auto load_q = [&](int buf, int i) {
    const int r0 = q_begin + i * 64;
    load_tile<64>(sQ_(buf), qh, ld_q, r0, q_end, tid);
    load_tile<64>(sDO_(buf), doh, ld_do, r0, q_end, tid);
    if (tid < 64) {
      const int r = r0 + tid;
      const bool ok = r < q_end;
      sLse_(buf)[tid] = ok ? lse_h[r] : 0.f;
      sD_(buf)[tid] = ok ? ds_h[r] : 0.f;
      sLim_(buf)[tid] = ok ? kv_limit[r] : -1;
    }
  };
  load_tile<64>(sK, k + head * 64, ld_k, kv0, kv_end, tid);
  load_tile<64>(sV, v + head * 64, ld_v, kv0, kv_end, tid);
  if (n_q > 0) load_q(0, 0);
  cp_async_commit();

  float dvacc[8][4], dkacc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { dvacc[i][0] = dvacc[i][1] = dvacc[i][2] = dvacc[i][3] = 0.f; dkacc[i][0] = dkacc[i][1] = dkacc[i][2] = dkacc[i][3] = 0.f; }
  const int key_a = kv0 + warp * 16 + g, key_b = key_a + 8;
  const float inv_cap = 1.f / cap;

  for (int i = 0; i < n_q; ++i) {
    const int buf = i & 1;
    if (i + 1 < n_q) { load_q(buf ^ 1, i + 1); cp_async_commit(); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();
    // ---- S^T = K Q^T  and  dP^T = V dO^T      (rows: this warp's 16 keys, cols: 64 queries)
    float sacc[8][4], pacc[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) { sacc[n][0] = sacc[n][1] = sacc[n][2] = sacc[n][3] = 0.f; pacc[n][0] = pacc[n][1] = pacc[n][2] = pacc[n][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t ka[4], va[4];
      {
        const int mat = lane >> 3;
        const int row = warp * 16 + (mat & 1) * 8 + (lane & 7);
        ldsm_x4(s_u32(sK + swz<64>(row, ks * 2 + (mat >> 1))), ka[0], ka[1], ka[2], ka[3]);
        ldsm_x4(s_u32(sV + swz<64>(row, ks * 2 + (mat >> 1))), va[0], va[1], va[2], va[3]);
      }
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        const int mat = lane >> 3;
        const int row = np * 16 + (mat >> 1) * 8 + (lane & 7);
        uint32_t b0, b1, b2, b3;
        ldsm_x4(s_u32(sQ_(buf) + swz<64>(row, ks * 2 + (mat & 1))), b0, b1, b2, b3);
        mma_bf16(sacc[2 * np], ka, b0, b1);
        mma_bf16(sacc[2 * np + 1], ka, b2, b3);
        ldsm_x4(s_u32(sDO_(buf) + swz<64>(row, ks * 2 + (mat & 1))), b0, b1, b2, b3);
        mma_bf16(pacc[2 * np], va, b0, b1);
        mma_bf16(pacc[2 * np + 1], va, b2, b3);
      }
    }
    // ---- P^T, dS^T (elementwise, accumulator layout: rows = keys g / g+8, cols = queries nt*8 + 2t + {0,1})
    uint32_t pf[4][4], dsf[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      float pv[4], dv_[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qc = nt * 8 + 2 * t + (e & 1);
        const int key = (e < 2) ? key_a : key_b;
        const float th = tanh_acc(sacc[nt][e] * scale * inv_cap);
        const bool vis = key <= sLim_(buf)[qc];
        const float p = vis ? __expf(cap * th - sLse_(buf)[qc]) : 0.f;
        pv[e] = p;
        dv_[e] = p * (pacc[nt][e] - sD_(buf)[qc]) * (1.f - th * th) * scale;
      }
      pf[nt >> 1][(nt & 1) * 2] = pack2_bf16(pv[0], pv[1]);
      pf[nt >> 1][(nt & 1) * 2 + 1] = pack2_bf16(pv[2], pv[3]);
      dsf[nt >> 1][(nt & 1) * 2] = pack2_bf16(dv_[0], dv_[1]);
      dsf[nt >> 1][(nt & 1) * 2 + 1] = pack2_bf16(dv_[2], dv_[3]);
      // stage dS^T [key][query] for the dQ product
      const int ch = nt;   // 8 queries per chunk
      *reinterpret_cast<uint32_t*>(sDS + swz<64>(warp * 16 + g, ch) + 2 * t) = dsf[nt >> 1][(nt & 1) * 2];
      *reinterpret_cast<uint32_t*>(sDS + swz<64>(warp * 16 + g + 8, ch) + 2 * t) = dsf[nt >> 1][(nt & 1) * 2 + 1];
    }
    // ---- dV += P^T dO ;  dK += dS^T Q       (k-dim = queries, B row-major [query][d] -> transposed ldmatrix)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int dp = 0; dp < 4; ++dp) {
        const int mat = lane >> 3;
        const int row = kk * 16 + (mat & 1) * 8 + (lane & 7);
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(s_u32(sDO_(buf) + swz<64>(row, dp * 2 + (mat >> 1))), b0, b1, b2, b3);
        mma_bf16(dvacc[2 * dp], pf[kk], b0, b1);
        mma_bf16(dvacc[2 * dp + 1], pf[kk], b2, b3);
        ldsm_x4_t(s_u32(sQ_(buf) + swz<64>(row, dp * 2 + (mat >> 1))), b0, b1, b2, b3);
        mma_bf16(dkacc[2 * dp], dsf[kk], b0, b1);
        mma_bf16(dkacc[2 * dp + 1], dsf[kk], b2, b3);
      }
    }
    __syncthreads();     // sDS complete
    // ---- dQ (this warp: 16 queries) += dS K : A = dS [query][key] = transposed read of sDS, B = K [key][d] (trans)
    {
      float qacc[8][4];
#pragma unroll
      for (int n = 0; n < 8; ++n) { qacc[n][0] = qacc[n][1] = qacc[n][2] = qacc[n][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {      // 16 keys per step
        uint32_t a[4];
        {
          // A fragment (rows = queries warp*16.., cols = keys kk*16..): matrices (q 0-7,k 0-7),(q 8-15,k 0-7),(q 0-7,k 8-15),(q 8-15,k 8-15)
          // stored transposed in sDS[key][query] -> trans load of blocks (keys, queries)
          const int mat = lane >> 3;
          const int krow = kk * 16 + (mat >> 1) * 8 + (lane & 7);
          const int qchunk = warp * 2 + (mat & 1);
          ldsm_x4_t(s_u32(sDS + swz<64>(krow, qchunk)), a[0], a[1], a[2], a[3]);
        }
#pragma unroll
        for (int dp = 0; dp < 4; ++dp) {
          const int mat = lane >> 3;
          const int row = kk * 16 + (mat & 1) * 8 + (lane & 7);
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(s_u32(sK + swz<64>(row, dp * 2 + (mat >> 1))), b0, b1, b2, b3);
          mma_bf16(qacc[2 * dp], a, b0, b1);
          mma_bf16(qacc[2 * dp + 1], a, b2, b3);
        }
      }
      const int r_a = q_begin + i * 64 + warp * 16 + g, r_b = r_a + 8;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        if (r_a < q_end) {
          float* d = dq + (long long)r_a * HI + head * 64 + nt * 8 + 2 * t;
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d), "f"(qacc[nt][0]), "f"(qacc[nt][1]) : "memory");
        }
        if (r_b < q_end) {
          float* d = dq + (long long)r_b * HI + head * 64 + nt * 8 + 2 * t;
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d), "f"(qacc[nt][2]), "f"(qacc[nt][3]) : "memory");
        }
      }
    }
    __syncthreads();     // before the next iteration overwrites sDS / the other q buffer
  }
  // ---- write dK (fp32) and dV (bf16)
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    if (key_a < kv_end) {
      *reinterpret_cast<float2*>(dk + (long long)key_a * HI + head * 64 + nt * 8 + 2 * t) = make_float2(dkacc[nt][0], dkacc[nt][1]);
      *reinterpret_cast<uint32_t*>(dv + (long long)key_a * ld_dv + head * 64 + nt * 8 + 2 * t) = pack2_bf16(dvacc[nt][0], dvacc[nt][1]);
    }
    if (key_b < kv_end) {
      *reinterpret_cast<float2*>(dk + (long long)key_b * HI + head * 64 + nt * 8 + 2 * t) = make_float2(dkacc[nt][2], dkacc[nt][3]);
      *reinterpret_cast<uint32_t*>(dv + (long long)key_b * ld_dv + head * 64 + nt * 8 + 2 * t) = pack2_bf16(dvacc[nt][2], dvacc[nt][3]);
    }
  }
}

// ================================================================================================ backward, head dim 128
// Same tile tables, span mask, soft-cap and gate as attn_bwd_k.

// main pass: one CTA per (64-key tile, head), 8 warps.  At DH = 128 a warp cannot hold both the dK and the dV accumulators of its 16 keys
// (2 x 64 fp32 per thread) next to the score fragments without spilling, so the two accumulators go to two warps: the warps of key group
// kg = warp & 3 share 16 keys; warp kg (role 0) forms S^T = K Q^T, P^T and dV += P^T dO, warp kg + 4 (role 1) forms dP^T = V dO^T, dS^T and
// dK += dS^T Q.  Role 0 hands w = p (1 - tanh^2) scale to role 1 through shared memory in fragment order (dS^T = w (dP^T - D)).  The dQ
// product is split by columns: warp w takes queries 16 (w & 3) .. + 15 and head dims 64 (w >> 2) .. + 63.
template <int DH>
__global__ void __launch_bounds__(ATT_BWD_THREADS_D128) attn_bwd_dh_k(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                                      const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ dop, long long ld_q,
                                                                      long long ld_k, long long ld_v, long long ld_do, const float* __restrict__ lse,
                                                                      const float* __restrict__ dsum, const int* __restrict__ kv_limit, const int* __restrict__ kt_kv0,
                                                                      const int* __restrict__ kt_kvend, const int* __restrict__ kt_q0, const int* __restrict__ kt_qend,
                                                                      float* __restrict__ dq, float* __restrict__ dk, __nv_bfloat16* __restrict__ dv, long long ld_dv,
                                                                      int M, int H, float scale, float cap) {
  constexpr int NT = ATT_BWD_THREADS_D128, TILE = 64 * DH;
  extern __shared__ __align__(128) uint8_t att_smem[];
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(att_smem);
  __nv_bfloat16* sV = sK + TILE;
  __nv_bfloat16* sQb = sV + TILE;             // [2][TILE]
  __nv_bfloat16* sDOb = sQb + 2 * TILE;       // [2][TILE]
  __nv_bfloat16* sDS = sDOb + 2 * TILE;       // dS^T [key][query], 64 x 64
  float* sW = reinterpret_cast<float*>(sDS + 64 * 64);      // [4 key groups][32 fragment values][32 lanes]
  float* sLseb = sW + 4 * 16 * 64;                           // [2][64]
  float* sDb = sLseb + 128;                                  // [2][64]
  int* sLimb = reinterpret_cast<int*>(sDb + 128);            // [2][64]
  const int tile = blockIdx.x, head = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int kg = warp & 3, role = warp >> 2;
  const int kv0 = kt_kv0[tile], kv_end = kt_kvend[tile], q_begin = kt_q0[tile], q_end = kt_qend[tile];
  const int HI = H * DH;
  const __nv_bfloat16* qh = q + head * DH;
  const __nv_bfloat16* doh = dop + head * DH;
  const float* lse_h = lse + (long long)head * M;
  const float* ds_h = dsum + (long long)head * M;
  const int n_q = (q_end - q_begin + 63) / 64;
  float* w_frag = sW + kg * (16 * 64);

  auto load_q = [&](int buf, int i) {
    const int r0 = q_begin + i * 64;
    load_tile<DH, NT>(sQb + buf * TILE, qh, ld_q, r0, q_end, tid);
    load_tile<DH, NT>(sDOb + buf * TILE, doh, ld_do, r0, q_end, tid);
    if (tid < 64) {
      const int r = r0 + tid;
      const bool ok = r < q_end;
      sLseb[buf * 64 + tid] = ok ? lse_h[r] : 0.f;
      sDb[buf * 64 + tid] = ok ? ds_h[r] : 0.f;
      sLimb[buf * 64 + tid] = ok ? kv_limit[r] : -1;
    }
  };
  load_tile<DH, NT>(sK, k + head * DH, ld_k, kv0, kv_end, tid);
  load_tile<DH, NT>(sV, v + head * DH, ld_v, kv0, kv_end, tid);
  if (n_q > 0) load_q(0, 0);
  cp_async_commit();

  float acc[DH / 8][4];             // role 0: dV, role 1: dK   (rows: keys g / g + 8 of the group, cols: head dims)
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
  const int key_a = kv0 + kg * 16 + g, key_b = key_a + 8;
  const float inv_cap = 1.f / cap;

  for (int i = 0; i < n_q; ++i) {
    const int buf = i & 1;
    const __nv_bfloat16* sQ = sQb + buf * TILE;
    const __nv_bfloat16* sDO = sDOb + buf * TILE;
    const float* sLse = sLseb + buf * 64;
    const float* sD = sDb + buf * 64;
    const int* sLim = sLimb + buf * 64;
    if (i + 1 < n_q) { load_q(buf ^ 1, i + 1); cp_async_commit(); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();
    // ---- role 0: S^T = K Q^T ;  role 1: dP^T = V dO^T       (rows: the group's 16 keys, cols: 64 queries)
    float sacc[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) { sacc[n][0] = sacc[n][1] = sacc[n][2] = sacc[n][3] = 0.f; }
    {
      const __nv_bfloat16* sA = role == 0 ? sK : sV;
      const __nv_bfloat16* sB = role == 0 ? sQ : sDO;
#pragma unroll
      for (int ks = 0; ks < DH / 16; ++ks) {
        uint32_t a[4];
        {
          const int mat = lane >> 3;
          const int row = kg * 16 + (mat & 1) * 8 + (lane & 7);
          ldsm_x4(s_u32(sA + swz<DH>(row, ks * 2 + (mat >> 1))), a[0], a[1], a[2], a[3]);
        }
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          const int mat = lane >> 3;
          const int row = np * 16 + (mat >> 1) * 8 + (lane & 7);
          uint32_t b0, b1, b2, b3;
          ldsm_x4(s_u32(sB + swz<DH>(row, ks * 2 + (mat & 1))), b0, b1, b2, b3);
          mma_bf16(sacc[2 * np], a, b0, b1);
          mma_bf16(sacc[2 * np + 1], a, b2, b3);
        }
      }
    }
    uint32_t af[4][4];                // role 0: P^T, role 1: dS^T   (A fragments of the dV / dK products)
    if (role == 0) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        float pv[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qc = nt * 8 + 2 * t + (e & 1);
          const int key = (e < 2) ? key_a : key_b;
          const float th = tanh_acc(sacc[nt][e] * scale * inv_cap);
          const bool vis = key <= sLim[qc];
          const float p = vis ? __expf(cap * th - sLse[qc]) : 0.f;
          pv[e] = p;
          w_frag[(nt * 4 + e) * 32 + lane] = p * (1.f - th * th) * scale;
        }
        af[nt >> 1][(nt & 1) * 2] = pack2_bf16(pv[0], pv[1]);
        af[nt >> 1][(nt & 1) * 2 + 1] = pack2_bf16(pv[2], pv[3]);
      }
    }
    __syncthreads();                  // w of every key group is in shared memory
    if (role == 1) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        float dsv[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qc = nt * 8 + 2 * t + (e & 1);
          dsv[e] = w_frag[(nt * 4 + e) * 32 + lane] * (sacc[nt][e] - sD[qc]);
        }
        af[nt >> 1][(nt & 1) * 2] = pack2_bf16(dsv[0], dsv[1]);
        af[nt >> 1][(nt & 1) * 2 + 1] = pack2_bf16(dsv[2], dsv[3]);
        // stage dS^T [key][query] for the dQ product
        *reinterpret_cast<uint32_t*>(sDS + swz<64>(kg * 16 + g, nt) + 2 * t) = af[nt >> 1][(nt & 1) * 2];
        *reinterpret_cast<uint32_t*>(sDS + swz<64>(kg * 16 + g + 8, nt) + 2 * t) = af[nt >> 1][(nt & 1) * 2 + 1];
      }
    }
    // ---- role 0: dV += P^T dO ;  role 1: dK += dS^T Q       (k-dim = queries, B row-major [query][d] -> transposed ldmatrix)
    {
      const __nv_bfloat16* sB = role == 0 ? sDO : sQ;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int dp = 0; dp < DH / 16; ++dp) {
          const int mat = lane >> 3;
          const int row = kk * 16 + (mat & 1) * 8 + (lane & 7);
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(s_u32(sB + swz<DH>(row, dp * 2 + (mat >> 1))), b0, b1, b2, b3);
          mma_bf16(acc[2 * dp], af[kk], b0, b1);
          mma_bf16(acc[2 * dp + 1], af[kk], b2, b3);
        }
      }
    }
    __syncthreads();     // sDS complete
    // ---- dQ (queries 16 (warp & 3) .., dims 64 (warp >> 2) ..) += dS K : A = transposed read of sDS, B = K [key][d] (trans)
    {
      constexpr int QC = 64;          // head dims per warp
      float qacc[QC / 8][4];
#pragma unroll
      for (int n = 0; n < QC / 8; ++n) { qacc[n][0] = qacc[n][1] = qacc[n][2] = qacc[n][3] = 0.f; }
      const int qw = warp & 3, c0 = (warp >> 2) * QC;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {      // 16 keys per step
        uint32_t a[4];
        {
          const int mat = lane >> 3;
          const int krow = kk * 16 + (mat >> 1) * 8 + (lane & 7);
          const int qchunk = qw * 2 + (mat & 1);
          ldsm_x4_t(s_u32(sDS + swz<64>(krow, qchunk)), a[0], a[1], a[2], a[3]);
        }
#pragma unroll
        for (int dp = 0; dp < QC / 16; ++dp) {
          const int mat = lane >> 3;
          const int row = kk * 16 + (mat & 1) * 8 + (lane & 7);
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(s_u32(sK + swz<DH>(row, c0 / 8 + dp * 2 + (mat >> 1))), b0, b1, b2, b3);
          mma_bf16(qacc[2 * dp], a, b0, b1);
          mma_bf16(qacc[2 * dp + 1], a, b2, b3);
        }
      }
      const int r_a = q_begin + i * 64 + qw * 16 + g, r_b = r_a + 8;
#pragma unroll
      for (int nt = 0; nt < QC / 8; ++nt) {
        if (r_a < q_end) {
          float* d = dq + (long long)r_a * HI + head * DH + c0 + nt * 8 + 2 * t;
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d), "f"(qacc[nt][0]), "f"(qacc[nt][1]) : "memory");
        }
        if (r_b < q_end) {
          float* d = dq + (long long)r_b * HI + head * DH + c0 + nt * 8 + 2 * t;
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d), "f"(qacc[nt][2]), "f"(qacc[nt][3]) : "memory");
        }
      }
    }
    __syncthreads();     // before the next iteration overwrites sDS / sW / the other q buffer
  }
  // ---- write dV (bf16, role 0) and dK (fp32, role 1)
#pragma unroll
  for (int nt = 0; nt < DH / 8; ++nt) {
    if (role == 0) {
      if (key_a < kv_end) *reinterpret_cast<uint32_t*>(dv + (long long)key_a * ld_dv + head * DH + nt * 8 + 2 * t) = pack2_bf16(acc[nt][0], acc[nt][1]);
      if (key_b < kv_end) *reinterpret_cast<uint32_t*>(dv + (long long)key_b * ld_dv + head * DH + nt * 8 + 2 * t) = pack2_bf16(acc[nt][2], acc[nt][3]);
    } else {
      if (key_a < kv_end) *reinterpret_cast<float2*>(dk + (long long)key_a * HI + head * DH + nt * 8 + 2 * t) = make_float2(acc[nt][0], acc[nt][1]);
      if (key_b < kv_end) *reinterpret_cast<float2*>(dk + (long long)key_b * HI + head * DH + nt * 8 + 2 * t) = make_float2(acc[nt][2], acc[nt][3]);
    }
  }
}

int num_sms();

}  // namespace tfx

using namespace tfx;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

// tfx_attn_bwd_prep / tfx_attn_bwd_prep_d128; `name` is the entry point's name for error messages
template <int DH>
static int attn_bwd_prep(const char* name, const void* do_gated, const void* o_gated, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero,
                         int M, int H, void* stream) {
  if (M <= 0) return 0;
  attn_bwd_prep_k<DH><<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>((const __nv_bfloat16*)do_gated, (const __nv_bfloat16*)o_gated, gates,
                                                                            (__nv_bfloat16*)do_pre, dsum_hm, dsum_mh, dq_zero, M, H);
  return check_launch(name);
}

extern "C" {

int tfx_attn_fwd(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H,
                 const int* kv_limit, const int* tile_q0, const int* tile_qend, const int* tile_kv0, const int* tile_kvend, int n_tiles,
                 void* o, long long ld_o, float* lse, int M, float scale, float softcap, const float* skip_if_fast, void* stream) {
  if (n_tiles <= 0) return 0;
  TFX_REQUIRE(softcap > 0.f, "attn_fwd: softcap must be > 0 (got %f)", softcap);
  attn_fwd_k<64><<<dim3(n_tiles, H), ATT_THREADS, 0, ST(stream)>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, ld_q, ld_k,
                                                                                 ld_v, gates, H, kv_limit, tile_q0, tile_qend, tile_kv0, tile_kvend, (__nv_bfloat16*)o,
                                                                                 ld_o, lse, M, scale, softcap, skip_if_fast);
  return check_launch("attn_fwd");
}

int tfx_attn_bwd_prep(const void* do_gated, const void* o_gated, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero, int M, int H, void* stream) {
  return attn_bwd_prep<64>("attn_bwd_prep", do_gated, o_gated, gates, do_pre, dsum_hm, dsum_mh, dq_zero, M, H, stream);
}

int tfx_attn_bwd(const void* q, const void* k, const void* v, const void* do_pre, long long ld_q, long long ld_k, long long ld_v, long long ld_do,
                 const float* lse, const float* dsum_hm, const int* kv_limit, const int* kt_kv0, const int* kt_kvend, const int* kt_q0, const int* kt_qend,
                 int n_kv_tiles, float* dq, float* dk, void* dv, long long ld_dv, int M, int H, float scale, float softcap, const float* skip_if_fast, void* stream) {
  if (n_kv_tiles <= 0) return 0;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(attn_bwd_k, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_BWD_SMEM) != cudaSuccess) { set_error("attn_bwd: cannot raise dynamic smem"); return -2; }
    attr_set = true;
  }
  attn_bwd_k<<<dim3(n_kv_tiles, H), ATT_THREADS, ATT_BWD_SMEM, ST(stream)>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (const __nv_bfloat16*)do_pre, ld_q, ld_k,
                                                                  ld_v, ld_do, lse, dsum_hm, kv_limit, kt_kv0, kt_kvend, kt_q0, kt_qend, dq, dk, (__nv_bfloat16*)dv, ld_dv, M, H,
                                                                  scale, softcap, skip_if_fast);
  return check_launch("attn_bwd");
}

int tfx_attn_fwd_d128(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H,
                      const int* kv_limit, const int* tile_q0, const int* tile_qend, const int* tile_kv0, const int* tile_kvend, int n_tiles,
                      void* o, long long ld_o, float* lse, int M, float scale, float softcap, void* stream) {
  if (n_tiles <= 0) return 0;
  TFX_REQUIRE(softcap > 0.f, "attn_fwd_d128: softcap must be > 0 (got %f)", softcap);
  TFX_REQUIRE(ld_q % 8 == 0 && ld_k % 8 == 0 && ld_v % 8 == 0 && ld_o % 2 == 0, "attn_fwd_d128: row pitches must keep 16-byte rows aligned");
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(attn_fwd_k<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, att_fwd_smem(128)) != cudaSuccess) { set_error("attn_fwd_d128: cannot raise dynamic smem"); return -2; }
    attr_set = true;
  }
  attn_fwd_k<128><<<dim3(n_tiles, H), ATT_THREADS, att_fwd_smem(128), ST(stream)>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, ld_q, ld_k, ld_v,
                                                                                 gates, H, kv_limit, tile_q0, tile_qend, tile_kv0, tile_kvend, (__nv_bfloat16*)o, ld_o, lse, M,
                                                                                 scale, softcap, nullptr);
  return check_launch("attn_fwd_d128");
}

int tfx_attn_bwd_prep_d128(const void* do_gated, const void* o_gated, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero, int M, int H, void* stream) {
  return attn_bwd_prep<128>("attn_bwd_prep_d128", do_gated, o_gated, gates, do_pre, dsum_hm, dsum_mh, dq_zero, M, H, stream);
}

int tfx_attn_bwd_d128(const void* q, const void* k, const void* v, const void* do_pre, long long ld_q, long long ld_k, long long ld_v, long long ld_do,
                      const float* lse, const float* dsum_hm, const int* kv_limit, const int* kt_kv0, const int* kt_kvend, const int* kt_q0, const int* kt_qend,
                      int n_kv_tiles, float* dq, float* dk, void* dv, long long ld_dv, int M, int H, float scale, float softcap, void* stream) {
  if (n_kv_tiles <= 0) return 0;
  TFX_REQUIRE(softcap > 0.f, "attn_bwd_d128: softcap must be > 0 (got %f)", softcap);
  TFX_REQUIRE(ld_q % 8 == 0 && ld_k % 8 == 0 && ld_v % 8 == 0 && ld_do % 8 == 0 && ld_dv % 2 == 0, "attn_bwd_d128: row pitches must keep 16-byte rows aligned");
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(attn_bwd_dh_k<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_BWD_SMEM_D128) != cudaSuccess) { set_error("attn_bwd_d128: cannot raise dynamic smem"); return -2; }
    attr_set = true;
  }
  attn_bwd_dh_k<128><<<dim3(n_kv_tiles, H), ATT_BWD_THREADS_D128, ATT_BWD_SMEM_D128, ST(stream)>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v,
                                                                                                (const __nv_bfloat16*)do_pre, ld_q, ld_k, ld_v, ld_do, lse, dsum_hm, kv_limit,
                                                                                                kt_kv0, kt_kvend, kt_q0, kt_qend, dq, dk, (__nv_bfloat16*)dv, ld_dv, M, H,
                                                                                                scale, softcap);
  return check_launch("attn_bwd_d128");
}

}  // extern "C"
