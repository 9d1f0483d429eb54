// Persistent, warp-specialised bf16 GEMM for sm_90a: TMA (128B swizzle) -> smem ring -> wgmma (two consumer warpgroups in
// ping-pong, each computing whole 128 x 128 tiles with fp32 accumulators in registers) -> accumulator tile staged through
// shared memory -> the Transfusion-specific fused epilogues.
//
//   D[m][n] = sum_k A(m,k) * B(n,k)
//   A "K-major":  stored row-major [M][K]   (activations as GEMM input, dY for dgrad)
//   A "MN-major": stored row-major [K][M]   (dY^T for wgrad: K = tokens)
//   B likewise over n.
//
// Roles (384 threads): warpgroup 0 = TMA producer (one lane, 40 registers), warpgroups 1 and 2 = wgmma consumers (232 registers)
// that also run the epilogue.  The consumers take alternate work items of the CTA's sequence (j = 0, 2, .. and j = 1, 3, ..), so
// one warpgroup's epilogue runs while the other's main loop keeps the tensor cores busy.  Per 16-deep k step a consumer issues two
// wgmma.m64n128k16 (rows 0-63, rows 64-127).  Two hand-offs order the warpgroups, both as named-barrier pairs (one warpgroup
// arrives, the other waits):
//   MMA: item j's main loop starts after item j-1's last k-block was issued.  Besides keeping the tensor cores on one tile at a
//        time, this is what makes the ring's parity waits exact: a consumer skips the other's k-blocks, and without the hand-off it
//        could wait on a full barrier two phases ahead of the one in flight and take a stale completion for its own.
//   ACC: item j's accumulators go to the 64 KB fp32 tile in shared memory after item j-1's epilogue has finished with it and with
//        the staging tiles.  GEGLU reads its whole accumulator row first and hands the tile on right then; its warpgroups stage
//        through separate tiles, so the GELU math and stores of item j-1 overlap item j's accumulator write.
// In the epilogue each thread of the warpgroup owns ONE accumulator row (warp q = 0..3: rows 32 q .. + 31, all 128 columns), the
// layout the per-row epilogue math (qk-RMSNorm, RoPE, gate select) wants.  EPI_QKVG_ROPE is EPI_QKVG without the qk-RMSNorm.
//
// Epilogue global traffic is staged through a per-warp 32 x 128 B shared-memory tile (XOR-swizzled 16 B chunks) so that every
// global load / store instruction covers whole 64 / 128-byte row segments.  Apart from GEGLU, one warpgroup runs an epilogue at a
// time, so the two share four such tiles.
//
// CL = 2: a cluster of two CTAs computes two vertically adjacent 128 x 128 tiles that share one B tile.  Each CTA loads its own A
// tile and HALF of the B tile, multicast into the same offset of both CTAs' rings, so a pair reads B from L2 once instead of twice.
// A ring slot is refilled only after the consumers of BOTH CTAs have released it (they arrive on the empty barriers of both).
#pragma once
#include "sm90_ptx.cuh"
#include "dropout.cuh"

namespace tfx {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BN = 128;
constexpr int GEMM_BK = 64;     // 64 bf16 = 128 B = one swizzle atom row
constexpr int GEMM_UK = 16;     // wgmma K for 16-bit inputs

// GEGLU_DROP: GEGLU with FFN dropout on h.  QKVG_ROPE: QKVG without the qk-RMSNorm (`qk_rmsnorm = False`): q, k = RoPE(acc), no qk_inv
// QKVG_D128 / QKVG_ROPE_D128: QKVG / QKVG_ROPE at head dim 128 (one head per 128-column tile; rope_cs is [64][rope_len])
enum : int { EPI_STORE = 0, EPI_QKVG = 1, EPI_RESID = 2, EPI_GEGLU = 3, EPI_GEGLU_DROP = 4, EPI_QKVG_ROPE = 5, EPI_QKVG_D128 = 6, EPI_QKVG_ROPE_D128 = 7 };
// the four QKVG epilogues are one body: head width (64 or 128) and whether q / k get the qk-RMSNorm
constexpr bool epi_is_qkvg(int e) { return e == EPI_QKVG || e == EPI_QKVG_ROPE || e == EPI_QKVG_D128 || e == EPI_QKVG_ROPE_D128; }
constexpr int qkvg_dh(int e) { return e == EPI_QKVG_D128 || e == EPI_QKVG_ROPE_D128 ? 128 : 64; }
constexpr bool qkvg_norm(int e) { return e == EPI_QKVG || e == EPI_QKVG_D128; }

struct GemmParams {
  int M, N, K;                 // D is M x N, reduction K
  int k_splits;                // >1: split-K, fp32 atomic accumulate (EPI_STORE only)
  // ---- EPI_STORE: out = alpha*acc + bias[n]
  float* out_f32; long long ld_f32;
  __nv_bfloat16* out_bf16; long long ld_bf16;
  const float* bias;           // [N] or null
  const long long* row_off;    // optional per-output-row element offset into out_f32 (-1 = skip row); replaces m*ld_f32
  float alpha;
  int accumulate_f32;          // 1: out_f32 += (red.add)
  int K1;                      // A is the concatenation [A | A2] along K; A2 starts at k = K1 (K1 % 64 == 0); K1 = K when unused
  // ---- EPI_QKVG* at head dim DH = 64 or 128 (N tile 128 = 128 / DH heads: H DH / 128 q tiles | as many k | as many v | 1 gate tile)
  int H;                       // heads (even at DH = 64)
  __nv_bfloat16 *q, *k, *v;    // [M][H*DH]
  float* gates;                // [M][H]   raw gate logits; null for an ungated model (columns [0, H) of the gate tile are then unused)
  float* mix_pre;              // [M][H]   optional: columns [m0, m0 + H) of the gate tile, m0 = H rounded up to even, = pre-activation of the
                               //          learned value-residual mix (T.py:956-960).  Without both there is no gate tile (N = 3 H DH)
  float* qk_inv;               // [M][2H]  1/max(|x|,eps) for q heads then k heads
  const float *q_gamma, *k_gamma;   // [DH]
  const int* rope_pos;         // [M]
  const float2* rope_cs;       // [DH/2][rope_len] (cos, sin): transposed table, consecutive positions are contiguous
  int rope_len;
  const int* kv_rows;          // optional [M]: destination ROW of token m inside k / v (in-place kv-cache append: k, v then point at a
                               // layer's cache slabs and q stays dense); null = row m
  // ---- EPI_RESID: y = acc + bias; y_bf16 = y; x_out = x_res + y * scale(row, col)
  const float* x_res; float* x_out; __nv_bfloat16* x_out_bf16;     // [M][N]
  __nv_bfloat16* y_bf16;       // [M][N] optional (pre-scale branch output, saved for backward)
  const int* cond_row;         // [M]  >=0: modality token -> row of zgate; <0: text token
  const float* zgate;          // [n_cond][zgate_ld]  sigmoid(to_ada_ln_zero(cond))
  long long zgate_ld;
  const float* ls;             // [N] layerscale (scale = ls + 1 for text rows); null => scale = 1
  // ---- EPI_GEGLU (N tile 128 = [64 value cols | 64 gate cols], N = 2*inner_pad)
  __nv_bfloat16* vg;           // [M][N] pre-activation (value|gate interleaved per tile), saved for backward
  __nv_bfloat16* h;            // [M][N/2] gelu(gate)*value (EPI_GEGLU_DROP: times mask / (1 - p); vg stays undropped)
  DropParams drop;             // EPI_GEGLU_DROP only (dropout.cuh, site FFN: i = row, j = column of h)
};

template <int EPI> struct GemmCfg {
  static constexpr int BM = GEMM_BM;
  static constexpr int THREADS = 384;
  static constexpr int STAGES = 4;
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
  static constexpr int B_BYTES = GEMM_BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_BYTES = GEMM_BM * GEMM_BN * 4;          // fp32 accumulator tile, rows of 512 B
  // per-warp staging: 32 rows x 128 B; RESID adds a 64-byte-pitch bf16 tile (2 KB).  Four warps (one epilogue warpgroup at a
  // time), except GEGLU: its warpgroups hand the accumulator tile over before their epilogues end, so each has its own four.
  static constexpr int STG_WARP = EPI == 2 ? 4096 + 2048 : 4096;
  static constexpr int STAGING = (EPI == EPI_GEGLU || EPI == EPI_GEGLU_DROP ? 8 : 4) * STG_WARP;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + STAGING + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one block");
};

// accumulator tile in shared memory: 16-byte chunk c of row r at r * 512 + ((c ^ (r & 7)) << 4)
__device__ __forceinline__ uint32_t acc_off(int r, int col) { return r * 512 + ((((col >> 2) ^ (r & 7))) << 4) + (col & 3) * 4; }
// 32 consecutive fp32 accumulators of row r starting at column col (col % 32 == 0)
__device__ __forceinline__ void acc_ld32(const uint8_t* acc, int r, int col, uint32_t (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const uint4 t = *reinterpret_cast<const uint4*>(acc + r * 512 + ((((col >> 2) + q) ^ (r & 7)) << 4));
    v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
  }
}

// Phi(g) and phi(g) of the exact-erf GELU (T.py:831-834, F.gelu default) from ONE exponential: Abramowitz-Stegun 7.1.26,
// erf(x) = 1 - (a1 t + .. + a5 t^5) e^{-x^2}, t = 1/(1 + p x), |err| <= 1.5e-7 - far below the bf16 rounding of the outputs.
// ~14 FMA-pipe instructions + 2 MUFU instead of the ~50 of erff + expf: the GEGLU epilogues are instruction-bound.
__device__ __forceinline__ void gelu_parts(float g, float& cdf, float& pdf) {
  const float ax = fabsf(g) * 0.70710678118654752f;
  const float t = __fdividef(1.f, fmaf(0.3275911f, ax, 1.f));
  const float E = __expf(-ax * ax);
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float h = 0.5f * poly * t * E;          // 0.5 * (1 - erf(|g|/sqrt 2))
  cdf = g >= 0.f ? 1.f - h : h;
  pdf = 0.3989422804014327f * E;
}
__device__ __forceinline__ float gelu_erf(float x) { float c, d; gelu_parts(x, c, d); return x * c; }
// value * gelu(gate) for two adjacent columns
__device__ __forceinline__ float2 geglu_pair(float2 g, float2 v) {
  return make_float2(gelu_erf(g.x) * v.x, gelu_erf(g.y) * v.y);
}

__device__ __forceinline__ void cp_async16_zfill(void* smem, const void* gmem, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz) : "memory");
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack2_bf16_(uint32_t w) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&w);
  return __bfloat1622float2(t);
}

// ---- per-warp staging tile: 32 rows x 128 B, 16-byte chunk c of row r lives at r*128 + ((c ^ (r & 7)) << 4)
// lane == row when writing/reading "own row"; (row, chunk) = f(iteration, lane) when touching global memory.
template <int CH>   // chunks (16 B) per row actually used: 8 (32 fp32 / 64 bf16) or 4 (32 bf16)
__device__ __forceinline__ void stg_put(uint8_t* sw, int lane, const uint32_t* w) {
#pragma unroll
  for (int c = 0; c < CH; ++c)
    *reinterpret_cast<uint4*>(sw + lane * 128 + ((c ^ (lane & 7)) << 4)) = make_uint4(w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3]);
}
template <int CH>
__device__ __forceinline__ void stg_get(const uint8_t* sw, int lane, uint32_t* w) {
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const uint4 t = *reinterpret_cast<const uint4*>(sw + lane * 128 + ((c ^ (lane & 7)) << 4));
    w[4 * c] = t.x; w[4 * c + 1] = t.y; w[4 * c + 2] = t.z; w[4 * c + 3] = t.w;
  }
}
// coalesced global store of the staged tile: g points at (tile row 0, first column); pitch in bytes
template <int CH>
__device__ __forceinline__ void stg_store(const uint8_t* sw, int lane, uint8_t* g, long long pitch, int rows_valid) {
  constexpr int RPI = 32 / CH;
#pragma unroll
  for (int it = 0; it < 32 / RPI; ++it) {
    const int row = it * RPI + lane / CH, ch = lane % CH;
    if (row < rows_valid)
      *reinterpret_cast<uint4*>(g + row * pitch + ch * 16) = *reinterpret_cast<const uint4*>(sw + row * 128 + ((ch ^ (row & 7)) << 4));
  }
}
// coalesced global load of a 32 x 128 B tile into registers (4 rows per instruction; rows >= rows_valid read as zero), and those
// registers into the staging tile: split so that the loads of several tiles can be in flight at once
__device__ __forceinline__ void stg_fetch(int lane, const uint8_t* g, long long pitch, int rows_valid, uint4 (&t)[8]) {
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int row = it * 4 + lane / 8, ch = lane % 8;
    t[it] = row < rows_valid ? *reinterpret_cast<const uint4*>(g + row * pitch + ch * 16) : make_uint4(0, 0, 0, 0);
  }
}
__device__ __forceinline__ void stg_fill(uint8_t* sw, int lane, const uint4 (&t)[8]) {
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int row = it * 4 + lane / 8, ch = lane % 8;
    *reinterpret_cast<uint4*>(sw + row * 128 + ((ch ^ (row & 7)) << 4)) = t[it];
  }
}

// 32 fp32 values of the lane's row -> bf16 -> staging tile (128 B pitch, 4 chunks), packed chunk by chunk
__device__ __forceinline__ void stg_put_pack(uint8_t* sw, int lane, const float* y) {
#pragma unroll
  for (int c = 0; c < 4; ++c)
    *reinterpret_cast<uint4*>(sw + lane * 128 + ((c ^ (lane & 7)) << 4)) =
        make_uint4(pack_bf16(y[8 * c], y[8 * c + 1]), pack_bf16(y[8 * c + 2], y[8 * c + 3]), pack_bf16(y[8 * c + 4], y[8 * c + 5]), pack_bf16(y[8 * c + 6], y[8 * c + 7]));
}
// compact variant for 32 bf16 per row: 32 rows x 64 B, chunk c of row r at r*64 + ((c ^ ((r >> 1) & 3)) << 4)  (conflict-free both ways)
__device__ __forceinline__ void stg64_put(uint8_t* sw, int lane, const uint32_t* w) {
#pragma unroll
  for (int c = 0; c < 4; ++c)
    *reinterpret_cast<uint4*>(sw + lane * 64 + ((c ^ ((lane >> 1) & 3)) << 4)) = make_uint4(w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3]);
}
__device__ __forceinline__ void stg64_put_pack(uint8_t* sw, int lane, const float* y) {
#pragma unroll
  for (int c = 0; c < 4; ++c)
    *reinterpret_cast<uint4*>(sw + lane * 64 + ((c ^ ((lane >> 1) & 3)) << 4)) =
        make_uint4(pack_bf16(y[8 * c], y[8 * c + 1]), pack_bf16(y[8 * c + 2], y[8 * c + 3]), pack_bf16(y[8 * c + 4], y[8 * c + 5]), pack_bf16(y[8 * c + 6], y[8 * c + 7]));
}
__device__ __forceinline__ void stg64_store(const uint8_t* sw, int lane, uint8_t* g, long long pitch, int rows_valid) {
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int row = it * 8 + (lane >> 2), ch = lane & 3;
    if (row < rows_valid)
      *reinterpret_cast<uint4*>(g + row * pitch + ch * 16) = *reinterpret_cast<const uint4*>(sw + row * 64 + ((ch ^ ((row >> 1) & 3)) << 4));
  }
}

// row-mapped variants: slab row r of the warp goes to global row rows[r] (rows already offset to the warp's first row)
__device__ __forceinline__ void stg64_store_rows(const uint8_t* sw, int lane, uint8_t* g, long long pitch, int rows_valid, const int* __restrict__ rows) {
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int row = it * 8 + (lane >> 2), ch = lane & 3;
    if (row < rows_valid)
      *reinterpret_cast<uint4*>(g + (long long)rows[row] * pitch + ch * 16) = *reinterpret_cast<const uint4*>(sw + row * 64 + ((ch ^ ((row >> 1) & 3)) << 4));
  }
}
template <int CH>
__device__ __forceinline__ void stg_store_rows(const uint8_t* sw, int lane, uint8_t* g, long long pitch, int rows_valid, const int* __restrict__ rows) {
  constexpr int RPI = 32 / CH;
#pragma unroll
  for (int it = 0; it < 32 / RPI; ++it) {
    const int row = it * RPI + lane / CH, ch = lane % CH;
    if (row < rows_valid)
      *reinterpret_cast<uint4*>(g + (long long)rows[row] * pitch + ch * 16) = *reinterpret_cast<const uint4*>(sw + row * 128 + ((ch ^ (row & 7)) << 4));
  }
}

// EPI_STORE epilogue of one 32-column slice [cbase, cbase + 32) of a warp's 32 rows: out = alpha * acc + bias.  Thread `lane` holds the
// raw accumulators of slice row `lane` in r; slice row i is output row row_of(i).  sw is the warp's staging tile (free on entry and exit).
// Both GEMM schedules end in this function, so their outputs agree bit for bit wherever their accumulators do.
template <class RowOf>
__device__ __forceinline__ void store_slice(const GemmParams& p, uint8_t* sw, int lane, uint32_t (&r)[32], int cbase, RowOf row_of) {
  const bool f32_staged = p.out_f32 && (p.row_off || (p.ld_f32 & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.out_f32) & 15) == 0);
  const bool bf16_staged = p.out_bf16 && (p.ld_bf16 & 7) == 0 && ((reinterpret_cast<uintptr_t>(p.out_bf16) & 15) == 0);
  const int row = row_of(lane);
  const bool row_ok = row < p.M;
  const bool full = cbase + 32 <= p.N;
  float v[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
  if (p.alpha != 1.f) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] *= p.alpha;
  }
  if (p.bias) {
    if (full) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) { const float4 b = *reinterpret_cast<const float4*>(p.bias + cbase + j); v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w; }
    } else {
      for (int j = 0; j < 32; ++j) if (cbase + j < p.N) v[j] += p.bias[cbase + j];
    }
  }
  if (p.out_f32) {
    if (full && f32_staged) {
#pragma unroll
      for (int j = 0; j < 32; ++j) r[j] = __float_as_uint(v[j]);
      stg_put<8>(sw, lane, r);
      __syncwarp();
      auto put = [&](float* dst, float x) { if (p.accumulate_f32) atomicAdd(dst, x); else *dst = x; };
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + (lane >> 3), ch = lane & 7;
        const int grow = row_of(rr);
        if (grow < p.M) {
          const long long off = p.row_off ? p.row_off[grow] : (long long)grow * p.ld_f32;
          if (off >= 0) {
            float* drow = p.out_f32 + off + cbase;                  // 4-byte aligned; 16-byte aligned iff off % 4 == 0
            const uint8_t* srow = sw + rr * 128;
            const int a = (int)(reinterpret_cast<uintptr_t>(drow) >> 2) & 3;
            if (a == 0) {
              float* dst = drow + ch * 4;
              const float4 t = *reinterpret_cast<const float4*>(srow + ((ch ^ (rr & 7)) << 4));
              if (p.accumulate_f32) asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(t.x), "f"(t.y), "f"(t.z), "f"(t.w) : "memory");
              else *reinterpret_cast<float4*>(dst) = t;
            } else {
              // a row offset that is not a multiple of 4 (the [512 x 1365] W2 gradient in the flat buffer): the first pe columns reach the next
              // 16-byte boundary, lanes 0-6 then cover 28 columns in aligned groups of 4, and lane 7 takes the pe leading and a trailing columns
              const int pe = 4 - a;
              auto col = [&](int j) { return *reinterpret_cast<const float*>(srow + (((j >> 2) ^ (rr & 7)) << 4) + (j & 3) * 4); };
              if (ch < 7) {
                const int j = pe + 4 * ch;
                float* dst = drow + j;
                const float4 t = make_float4(col(j), col(j + 1), col(j + 2), col(j + 3));
                if (p.accumulate_f32) asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(t.x), "f"(t.y), "f"(t.z), "f"(t.w) : "memory");
                else *reinterpret_cast<float4*>(dst) = t;
              } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) { const int j = i < pe ? i : 28 + i; put(drow + j, col(j)); }
              }
            }
          }
        }
      }
      __syncwarp();
    } else if (row_ok) {
      const long long off = p.row_off ? p.row_off[row] : (long long)row * p.ld_f32;
      if (off >= 0) {
        float* dst = p.out_f32 + off + cbase;
        for (int j = 0; j < 32; ++j)
          if (cbase + j < p.N) { if (p.accumulate_f32) atomicAdd(dst + j, v[j]); else dst[j] = v[j]; }
      }
    }
  }
  if (p.out_bf16) {
    if (full && bf16_staged) {
      uint32_t w[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) w[j] = pack_bf16(v[2 * j], v[2 * j + 1]);
      stg_put<4>(sw, lane, w);
      __syncwarp();
#pragma unroll
      for (int it = 0; it < 4; ++it) {                           // 8 rows x 64 B per instruction
        const int rr = it * 8 + (lane >> 2), ch = lane & 3;
        const int grow = row_of(rr);
        if (grow < p.M)
          *reinterpret_cast<uint4*>(p.out_bf16 + (long long)grow * p.ld_bf16 + cbase + ch * 8) = *reinterpret_cast<const uint4*>(sw + rr * 128 + ((ch ^ (rr & 7)) << 4));
      }
      __syncwarp();
    } else if (row_ok) {
      __nv_bfloat16* dst = p.out_bf16 + (long long)row * p.ld_bf16 + cbase;
      for (int j = 0; j < 32; ++j) if (cbase + j < p.N) dst[j] = __float2bfloat16(v[j]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ pipeline of both kernels
// Persistent schedule: work items run over (k split, m unit, n tile), n fastest; an m unit is CL vertically adjacent BM-row tiles, one per
// CTA of the cluster.
template <int BM, int CL>
struct GemmSched {
  struct Work { int m_blk, n_blk, kb0, kb1; };
  int n_tiles, unit_items, kb_total, kb_per_split, num_items;
  __device__ __forceinline__ explicit GemmSched(const GemmParams& p) {
    const int m_tiles = (p.M + BM - 1) / BM;
    n_tiles = (p.N + GEMM_BN - 1) / GEMM_BN;
    kb_total = (p.K + GEMM_BK - 1) / GEMM_BK;
    kb_per_split = (kb_total + p.k_splits - 1) / p.k_splits;
    unit_items = (m_tiles + CL - 1) / CL * n_tiles;
    num_items = unit_items * p.k_splits;
  }
  // the tile of work item `item` that CTA `cta_rank` computes, and its k-blocks [kb0, kb1).  With CL = 2 and an odd tile count the last
  // unit's second tile is past the end: TMA zero-fills it and every store is row-guarded.
  __device__ __forceinline__ Work work(int item, int cta_rank) const {
    const int split = item / unit_items;
    const int rem = item - split * unit_items;
    const int m_unit = rem / n_tiles;
    const int kb0 = split * kb_per_split;
    return {m_unit * CL + cta_rank, rem - m_unit * n_tiles, kb0, min(kb0 + kb_per_split, kb_total)};
  }
};

// a slot of the STAGES-deep shared-memory ring and the parity of its current fill
template <int STAGES>
struct GemmRing {
  int stage = 0; uint32_t phase = 0;
  __device__ __forceinline__ void step() { if (++stage == STAGES) { stage = 0; phase ^= 1; } }
};

// Producer: once the ring slot is free, load k-block kb of the Cfg::BM-row A tile m_blk and the 128-row B tile n_blk into it, and step on.
// TWO_A: a K-major A is the concatenation [A | A2] along K, with A2 (tmA2) from k = p.K1.  CL = 2: this CTA's half of the B tile (64 rows,
// or one 64-wide MN block) goes to the same offset of both CTAs' rings.
template <class Cfg, bool A_MN, bool B_MN, int CL, bool TWO_A>
__device__ __forceinline__ void gemm_fill(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, GemmRing<Cfg::STAGES>& ring,
                                          const CUtensorMap* tmA, const CUtensorMap* tmA2, const CUtensorMap* tmB, const GemmParams& p,
                                          int kb, int m_blk, int n_blk, int cta_rank) {
  constexpr int BM = Cfg::BM, BN = GEMM_BN;
  mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1);
  uint8_t* sA = smem + ring.stage * Cfg::STAGE_BYTES;
  uint8_t* sB = sA + Cfg::A_BYTES;
  uint64_t* bar = &full_bar[ring.stage];
  mbar_expect_tx(bar, Cfg::STAGE_BYTES);
  if (!A_MN) {
    if (!TWO_A || kb * GEMM_BK < p.K1) tma_load_2d(tmA, bar, sA, kb * GEMM_BK, m_blk * BM);     // one 64 x BM box
    else tma_load_2d(tmA2, bar, sA, kb * GEMM_BK - p.K1, m_blk * BM);
  } else {
#pragma unroll
    for (int a = 0; a < BM / 64; ++a)
      tma_load_2d(tmA, bar, sA + a * (GEMM_BK * 128), m_blk * BM + a * 64, kb * GEMM_BK);
  }
  if constexpr (CL > 1) {
    if (!B_MN) tma_load_2d_multicast(tmB, bar, sB + cta_rank * (64 * 128), kb * GEMM_BK, n_blk * BN + cta_rank * 64, (uint16_t)3);
    else tma_load_2d_multicast(tmB, bar, sB + cta_rank * (GEMM_BK * 128), n_blk * BN + cta_rank * 64, kb * GEMM_BK, (uint16_t)3);
  } else if (!B_MN) {
    tma_load_2d(tmB, bar, sB, kb * GEMM_BK, n_blk * BN);
  } else {
#pragma unroll
    for (int a = 0; a < BN / 64; ++a)
      tma_load_2d(tmB, bar, sB + a * (GEMM_BK * 128), n_blk * BN + a * 64, kb * GEMM_BK);
  }
  ring.step();
}

// Consumer main loop of one work item: k-blocks [kb0, kb1) into the accumulators of 128 tile rows (d0: rows 0-63, d1: rows 64-127), whose
// A rows start a_off bytes into the slot's A tile.  Two wgmma.m64n128k16 per 16-deep k step.  A slot is released one k-block behind, once
// wgmma.wait_group 1 shows its MMAs retired; the slot of the last k-block (-1 if none) is returned for gemm_drain.
template <class Cfg, bool A_MN, bool B_MN, class Release>
__device__ __forceinline__ int gemm_mainloop(uint8_t* smem, uint64_t* full_bar, GemmRing<Cfg::STAGES>& ring, uint32_t a_off, int kb0, int kb1,
                                             float (&d0)[64], float (&d1)[64], Release& release) {
#pragma unroll
  for (int i = 0; i < 64; ++i) { d0[i] = 0.f; d1[i] = 0.f; }
  int prev_stage = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full_bar[ring.stage], ring.phase);
    const uint32_t sA = smem_u32(smem + ring.stage * Cfg::STAGE_BYTES) + a_off;
    const uint32_t sB = smem_u32(smem + ring.stage * Cfg::STAGE_BYTES) + Cfg::A_BYTES;
    wgmma_reg_fence(d0);
    wgmma_reg_fence(d1);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < GEMM_BK / GEMM_UK; ++k) {
      const uint64_t db = B_MN ? wgmma_desc_sw128(sB + k * (GEMM_UK * 128), GEMM_BK * 128, 1024)
                               : wgmma_desc_sw128(sB + k * (GEMM_UK * 2), 16, 1024);
      // A rows 64-127: the second 64-wide MN block (MN-major) or 64 rows further down (K-major)
      const uint64_t da0 = A_MN ? wgmma_desc_sw128(sA + k * (GEMM_UK * 128), GEMM_BK * 128, 1024)
                                : wgmma_desc_sw128(sA + k * (GEMM_UK * 2), 16, 1024);
      const uint64_t da1 = A_MN ? wgmma_desc_sw128(sA + GEMM_BK * 128 + k * (GEMM_UK * 128), GEMM_BK * 128, 1024)
                                : wgmma_desc_sw128(sA + 64 * 128 + k * (GEMM_UK * 2), 16, 1024);
      const uint32_t acc_flag = (kb > kb0 || k > 0) ? 1u : 0u;
      wgmma_m64n128_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(d0, da0, db, acc_flag);
      wgmma_m64n128_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(d1, da1, db, acc_flag);
    }
    wgmma_commit();
    wgmma_wait<1>();                        // the previous k-block's MMAs have retired: its smem slot is free
    if (prev_stage >= 0) release(prev_stage);
    prev_stage = ring.stage;
    ring.step();
  }
  return prev_stage;
}

// after the main loop: every MMA retired, the accumulators fenced, the last slot released
template <class Release>
__device__ __forceinline__ void gemm_drain(float (&d0)[64], float (&d1)[64], int last_stage, Release& release) {
  wgmma_wait<0>();
  wgmma_reg_fence(d0);
  wgmma_reg_fence(d1);
  if (last_stage >= 0) release(last_stage);
}

template <bool A_MN, bool B_MN, int EPI, int CL>
__global__ void __launch_bounds__(384, 1)
gemm_sm90_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using Cfg = GemmCfg<EPI>;
  constexpr bool GEGLU = EPI == EPI_GEGLU || EPI == EPI_GEGLU_DROP;
  constexpr bool QKVG = epi_is_qkvg(EPI);
  constexpr int BN = GEMM_BN;
  constexpr int STAGES = Cfg::STAGES;
  static_assert(Cfg::STAGE_BYTES % 1024 == 0 && 2 * STAGES <= 32, "stage alignment / barrier area");
  // declared 1024-byte aligned (SWIZZLE_128B tiles) and used directly: rounding the pointer up through an integer loses the shared address space
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();      // SWIZZLE_128B tiles need 1024-byte alignment (no printf: see TFX_DEBUG_SPIN)
  uint8_t* acc = smem + STAGES * Cfg::STAGE_BYTES;
  uint8_t* staging = acc + Cfg::ACC_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + Cfg::STAGING);
  uint64_t* full_bar = bars;                  // [STAGES]
  uint64_t* empty_bar = bars + STAGES;        // [STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const GemmSched<GEMM_BM, CL> sched(p);
  const int num_items = sched.num_items;
  const int cta_rank = CL > 1 ? (int)cluster_ctarank() : 0;
  const int first_item = blockIdx.x / CL, item_stride = gridDim.x / CL;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    // empty: one arrival per warp of the consuming warpgroup, in every CTA of the cluster
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4 * CL); }
    mbar_fence_init();
  }
  __syncthreads();
  if constexpr (CL > 1) cluster_sync_all();               // the peer's barriers are initialised before anything is signalled at them

  if (warp < 4) {
    // ===================================================== TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      GemmRing<STAGES> ring;
      for (int item = first_item; item < num_items; item += item_stride) {
        const auto w = sched.work(item, cta_rank);
        for (int kb = w.kb0; kb < w.kb1; ++kb)
          gemm_fill<Cfg, A_MN, B_MN, CL, true>(smem, full_bar, empty_bar, ring, &tmA, &tmA2, &tmB, p, kb, w.m_blk, w.n_blk, cta_rank);
      }
    }
  } else {
    // ===================================================== consumers (ping-pong): wgmma main loop, then the epilogue
    setmaxnreg_inc<232>();
    // named barriers: 1 + cw accumulator tile written (this warpgroup), 3 + cw MMA turn of warpgroup cw, 5 + cw ACC turn of warpgroup cw
    constexpr int BAR_TILE = 1, BAR_MMA = 3, BAR_ACC = 5;
    const int cw = (warp >> 2) - 1;            // consumer warpgroup 0 / 1: items j = cw, cw + 2, .. of this CTA
    const int quad = warp & 3;                 // epilogue rows 32 quad .. + 31; fragment rows 16 quad .. of each 64-row half
    uint8_t* sw = staging + ((GEGLU ? 4 * cw : 0) + quad) * Cfg::STG_WARP;
    const int erow = quad * 32 + lane;         // this thread's accumulator row in the epilogue
    GemmRing<STAGES> ring;
    // a consumed ring slot is released in every CTA that wrote into it
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) {
        if constexpr (CL > 1) { mbar_arrive_cluster(&empty_bar[s], 0); mbar_arrive_cluster(&empty_bar[s], 1); }
        else mbar_arrive(&empty_bar[s]);
      }
    };
    int nth = 0;                               // position of `item` in this CTA's sequence
    for (int item = first_item; item < num_items; item += item_stride, ++nth) {
      const auto [m_blk, n_blk, kb0, kb1] = sched.work(item, cta_rank);
      if ((nth & 1) != cw) {                                 // the other warpgroup's item: step over its k-blocks in the ring
        const int s = ring.stage + (kb1 - kb0);
        ring.stage = s % STAGES;
        ring.phase ^= (uint32_t)(s / STAGES) & 1u;
        continue;
      }
      // hand-offs pair up exactly: item nth waits for nth - 1's signal iff nth > 0, and signals iff there is an item nth + 1
      const bool has_next = item + item_stride < num_items;
      if (nth > 0) named_bar_sync(BAR_MMA + cw, 256);
      float d0[64], d1[64];                                   // accumulator rows 0-63 / 64-127
      const int last_stage = gemm_mainloop<Cfg, A_MN, B_MN>(smem, full_bar, ring, 0, kb0, kb1, d0, d1, release);
      if (has_next) named_bar_arrive(BAR_MMA + (cw ^ 1), 256);     // every k-block of this item is issued: the other main loop may start
      gemm_drain(d0, d1, last_stage, release);

      // ---- accumulator fragments -> shared fp32 tile, once the previous item's epilogue has finished reading it
      if (nth > 0) named_bar_sync(BAR_ACC + cw, 256);
      {
        const int r0 = quad * 16 + (lane >> 2);
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          const int c = 8 * q + 2 * (lane & 3);
          *reinterpret_cast<float2*>(acc + acc_off(r0, c)) = make_float2(d0[4 * q], d0[4 * q + 1]);
          *reinterpret_cast<float2*>(acc + acc_off(r0 + 8, c)) = make_float2(d0[4 * q + 2], d0[4 * q + 3]);
          *reinterpret_cast<float2*>(acc + acc_off(r0 + 64, c)) = make_float2(d1[4 * q], d1[4 * q + 1]);
          *reinterpret_cast<float2*>(acc + acc_off(r0 + 72, c)) = make_float2(d1[4 * q + 2], d1[4 * q + 3]);
        }
      }
      named_bar_sync(BAR_TILE + cw, 128);

      const int wrow0 = m_blk * GEMM_BM + quad * 32;          // first row of this warp's 32-row slab
      const int row = wrow0 + lane;
      const bool row_ok = row < p.M;
      const int rows_valid = min(32, p.M - wrow0);            // may be <= 0
      const int col0 = n_blk * BN;
      int qk_pos = 0;
      if constexpr (QKVG) { qk_pos = row_ok ? p.rope_pos[row] : 0; }
      if constexpr (EPI == EPI_RESID) { qk_pos = (row_ok && p.cond_row) ? p.cond_row[row] : -1; }      // (reused as the condition row)

      if constexpr (EPI == EPI_STORE) {
#pragma unroll 1
        for (int c = 0; c < BN / 32; ++c) {
          const int cbase = col0 + c * 32;
          if (cbase >= p.N) break;
          uint32_t r[32];
          acc_ld32(acc, erow, c * 32, r);
          store_slice(p, sw, lane, r, cbase, [&](int i) { return wrow0 + i; });
        }
      } else if constexpr (QKVG) {
        // N tiles: H DH / 128 q tiles | as many k tiles | as many v tiles | 1 gate tile; a tile holds 128 / DH heads
        constexpr int DH = qkvg_dh(EPI), HPT = BN / DH;
        constexpr float SQRT_DH = DH == 64 ? 8.f : 11.313708498984761f;
        const int tps = (p.H * DH) >> 7;      // tiles per section, H DH / 128 (H > 0: a shift, where a signed divide costs instructions)
        const int kind = n_blk / tps;         // 0 q, 1 k, 2 v, 3 gates
        const int tis = n_blk - kind * tps;   // tile in section
        const long long HI = (long long)p.H * DH;
        if (kind <= 1) {
          const float* gamma = kind == 0 ? p.q_gamma : p.k_gamma;
          __nv_bfloat16* dstm = kind == 0 ? p.q : p.k;
          const float2* cs = p.rope_cs + qk_pos;        // entry i of this row's position: cs[i * rope_len]
          // qk-RMSNorm of the head that starts in the tile's 64-column half hh, from its sum of squares: 1/|x| goes to qk_inv, and the
          // columns are scaled by sqrt(DH) / |x| (times gamma + 1 per column below).  The sum is taken where each width has its head:
          // at 128 the whole tile row, re-read from shared memory before the halves so that 128 accumulators are not held in registers;
          // at 64 the two slices of the half just loaded.
          float sc = 1.f;
          auto norm = [&](float ss, int hh) {
            const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
            if (row_ok) p.qk_inv[(long long)row * 2 * p.H + kind * p.H + tis * HPT + hh * 64 / DH] = inv;
            sc = inv * SQRT_DH;
          };
          if constexpr (qkvg_norm(EPI) && DH == 128) {
            float ss = 0.f;
#pragma unroll 1
            for (int c = 0; c < 4; ++c) {
              uint32_t r[32];
              acc_ld32(acc, erow, c * 32, r);
#pragma unroll
              for (int j = 0; j < 32; ++j) { const float a = __uint_as_float(r[j]); ss += a * a; }
            }
            norm(ss, 0);
          }
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {              // the tile's two 64-column halves
            const int c0 = hh * 64 % DH;                  // the half's first column within its head
            uint32_t r0[32], r1[32];
            acc_ld32(acc, erow, hh * 64, r0);
            acc_ld32(acc, erow, hh * 64 + 32, r1);
            if constexpr (qkvg_norm(EPI) && DH == 64) {
              float ss = 0.f;
#pragma unroll
              for (int j = 0; j < 32; ++j) { float a = __uint_as_float(r0[j]), b = __uint_as_float(r1[j]); ss += a * a + b * b; }
              norm(ss, hh);
            }
            const int head = tis * HPT + hh * 64 / DH;
            uint32_t outw[32];
#pragma unroll
            for (int dh = 0; dh < 2; ++dh) {              // the half's two 32-column slices
              uint32_t* rr = dh == 0 ? r0 : r1;
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                const int d0 = c0 + dh * 32 + 2 * i;     // column within the head
                float y0 = __uint_as_float(rr[2 * i]), y1 = __uint_as_float(rr[2 * i + 1]);
                if constexpr (qkvg_norm(EPI)) {
                  const float2 gm = *reinterpret_cast<const float2*>(gamma + d0);
                  y0 = y0 * sc * (gm.x + 1.f);
                  y1 = y1 * sc * (gm.y + 1.f);
                }
                const float2 cc = cs[(long long)(d0 >> 1) * p.rope_len];
                outw[dh * 16 + i] = pack_bf16(y0 * cc.x - y1 * cc.y, y1 * cc.x + y0 * cc.y);
              }
            }
            stg_put<8>(sw, lane, outw);
            __syncwarp();
            if (kind == 1 && p.kv_rows) stg_store_rows<8>(sw, lane, reinterpret_cast<uint8_t*>(dstm + head * DH + c0), HI * 2, rows_valid, p.kv_rows + wrow0);
            else stg_store<8>(sw, lane, reinterpret_cast<uint8_t*>(dstm + (long long)wrow0 * HI + head * DH + c0), HI * 2, rows_valid);
            __syncwarp();
          }
        } else if (kind == 2) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            uint32_t r0[32], r1[32], w[32];
            acc_ld32(acc, erow, c * 64, r0);
            acc_ld32(acc, erow, c * 64 + 32, r1);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              w[j] = pack_bf16(__uint_as_float(r0[2 * j]), __uint_as_float(r0[2 * j + 1]));
              w[16 + j] = pack_bf16(__uint_as_float(r1[2 * j]), __uint_as_float(r1[2 * j + 1]));
            }
            stg_put<8>(sw, lane, w);
            __syncwarp();
            if (p.kv_rows) stg_store_rows<8>(sw, lane, reinterpret_cast<uint8_t*>(p.v + tis * 128 + c * 64), HI * 2, rows_valid, p.kv_rows + wrow0);
            else stg_store<8>(sw, lane, reinterpret_cast<uint8_t*>(p.v + (long long)wrow0 * HI + tis * 128 + c * 64), HI * 2, rows_valid);
            __syncwarp();
          }
        } else {
          uint32_t r[32];
          acc_ld32(acc, erow, 0, r);
          if (row_ok) {
            constexpr int H_MAX = DH == 64 ? 32 : 16;   // the largest head count the entry points accept at this width
            if (p.gates) {                              // null for an ungated model (`gate_values = False`), whose tile carries the mix only
              float* dst = p.gates + (long long)row * p.H;
#pragma unroll
              for (int j = 0; j < H_MAX; ++j) if (j < p.H) dst[j] = __uint_as_float(r[j]);
            }
            if (p.mix_pre) {                            // mix columns start at an even column (bf16 pairs of their gradient stay 4-byte aligned)
              const int m0 = (p.H + 1) & ~1;
              float* dm = p.mix_pre + (long long)row * p.H;
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                // H is even at width 64, so the start is H.  Spelled per width so that each keeps its generated code: p.H read per
                // column at 64, the rounded start computed once at 128.
                const int mj = DH == 64 ? p.H : m0;
                if (j >= mj && j < mj + p.H) dm[j - mj] = __uint_as_float(r[j]);
              }
              // above 16 heads of 64 the mix runs past the first slice, into columns [32, 2 H): loaded into the same words once the
              // first slice is stored, so no more accumulators are live than at H <= 16 (at 128, H <= 16 keeps it in the first slice)
              if constexpr (DH == 64) {
                if (p.H > 16) {
                  acc_ld32(acc, erow, 32, r);
#pragma unroll
                  for (int j = 0; j < 32; ++j) if (32 + j < 2 * p.H) dm[32 + j - p.H] = __uint_as_float(r[j]);
                }
              }
            }
          }
        }
      } else if constexpr (EPI == EPI_RESID) {
        const int crow = qk_pos;
        const float* zrow = (p.zgate && crow >= 0) ? p.zgate + (long long)crow * p.zgate_ld : nullptr;
        uint8_t* swb = sw + 4096;                       // 64-byte-pitch tile for the bf16 outputs
        // the residual rows are requested one slice ahead: the global loads of slice sl + 1 are in flight while slice sl is computed
        uint4 xres[8];
        auto fetch = [&](int sl) {
          stg_fetch(lane, reinterpret_cast<const uint8_t*>(p.x_res + (long long)wrow0 * p.N + col0 + sl * 32), (long long)p.N * 4,
                    col0 + sl * 32 < p.N ? rows_valid : 0, xres);
        };
        fetch(0);
#pragma unroll 1
        for (int sl = 0; sl < BN / 32; ++sl) {          // 32-column slices of the tile
          const int cbase = col0 + sl * 32;
          if (cbase >= p.N) break;                      // N is a multiple of 32 for every RESID use
          __syncwarp();
          stg_fill(sw, lane, xres);
          if (sl + 1 < BN / 32) fetch(sl + 1);
          uint32_t r[32];
          acc_ld32(acc, erow, sl * 32, r);
          float y[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) y[j] = __uint_as_float(r[j]);
          if (p.bias) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) { const float4 b = *reinterpret_cast<const float4*>(p.bias + cbase + j); y[j] += b.x; y[j + 1] += b.y; y[j + 2] += b.z; y[j + 3] += b.w; }
          }
          if (p.y_bf16) {
            stg64_put_pack(swb, lane, y);
            __syncwarp();
            stg64_store(swb, lane, reinterpret_cast<uint8_t*>(p.y_bf16 + (long long)wrow0 * p.N + cbase), (long long)p.N * 2, rows_valid);
            __syncwarp();
          }
          {
            uint32_t xrv[32];
            __syncwarp();
            stg_get<8>(sw, lane, xrv);                  // residual row
            if (zrow) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                const float4 s4 = *reinterpret_cast<const float4*>(zrow + cbase + j);
                y[j] = __uint_as_float(xrv[j]) + y[j] * s4.x; y[j + 1] = __uint_as_float(xrv[j + 1]) + y[j + 1] * s4.y;
                y[j + 2] = __uint_as_float(xrv[j + 2]) + y[j + 2] * s4.z; y[j + 3] = __uint_as_float(xrv[j + 3]) + y[j + 3] * s4.w;
              }
            } else if (p.ls) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                const float4 s4 = *reinterpret_cast<const float4*>(p.ls + cbase + j);
                y[j] = __uint_as_float(xrv[j]) + y[j] * (s4.x + 1.f); y[j + 1] = __uint_as_float(xrv[j + 1]) + y[j + 1] * (s4.y + 1.f);
                y[j + 2] = __uint_as_float(xrv[j + 2]) + y[j + 2] * (s4.z + 1.f); y[j + 3] = __uint_as_float(xrv[j + 3]) + y[j + 3] * (s4.w + 1.f);
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j) y[j] += __uint_as_float(xrv[j]);
            }
          }
          // x_out (fp32, optional when only the bf16 copy is kept) leaves in two 16-column passes through the 64-byte-pitch tile
          if (p.x_out)
#pragma unroll
          for (int hfc = 0; hfc < 2; ++hfc) {
            uint32_t w16[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) w16[j] = __float_as_uint(y[hfc * 16 + j]);
            __syncwarp();
            stg64_put(swb, lane, w16);
            __syncwarp();
            stg64_store(swb, lane, reinterpret_cast<uint8_t*>(p.x_out + (long long)wrow0 * p.N + cbase + hfc * 16), (long long)p.N * 4, rows_valid);
          }
          if (p.x_out_bf16) {
            __syncwarp();
            stg64_put_pack(swb, lane, y);
            __syncwarp();
            stg64_store(swb, lane, reinterpret_cast<uint8_t*>(p.x_out_bf16 + (long long)wrow0 * p.N + cbase), (long long)p.N * 2, rows_valid);
          }
          __syncwarp();
        }
      } else if constexpr (GEGLU) {
        // the 128-wide tile is [64 value | 64 gate]; column slice c handles 32 value and the matching 32 gate columns.  The whole
        // accumulator row is read first and the tile handed on at once, so the GELU math and the stores overlap the next item's
        // accumulator write (this warpgroup stages through its own four tiles).
        // dropout: the keep bits of the row's 64 h columns (one Philox call per 8), computed before the accumulator row is loaded,
        // where few registers are live (drawn later, next to the 128 accumulator words, they spill)
        uint32_t keep[2] = {0u, 0u};
        if constexpr (EPI == EPI_GEGLU_DROP) {
          const uint32_t k0 = __ldg(p.drop.key), k1 = __ldg(p.drop.key + 1);
#pragma unroll
          for (int q = 0; q < 8; ++q) keep[q >> 2] |= drop_keep8(p.drop, k0, k1, DROP_SITE_FFN, 0, (uint32_t)row, (uint32_t)(n_blk * 8 + q)) << (8 * (q & 3));
        }
        uint32_t ra[4][32];
#pragma unroll
        for (int q = 0; q < 4; ++q) acc_ld32(acc, erow, q * 32, ra[q]);
        if (has_next) named_bar_arrive(BAR_ACC + (cw ^ 1), 256);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int cv = col0 + c * 32, cg = cv + 64;
          if (cv >= p.N) break;                         // N is a multiple of 128: a tile is either complete or absent
          float v[32], g[32];                           // value and gate pre-activations stay in registers for the product
#pragma unroll
          for (int j = 0; j < 32; ++j) { v[j] = __uint_as_float(ra[c][j]) + p.bias[cv + j]; g[j] = __uint_as_float(ra[2 + c][j]) + p.bias[cg + j]; }
          __syncwarp();
          stg64_put_pack(sw, lane, v);
          __syncwarp();
          stg64_store(sw, lane, reinterpret_cast<uint8_t*>(p.vg + (long long)wrow0 * p.N + cv), (long long)p.N * 2, rows_valid);
          __syncwarp();
          stg64_put_pack(sw, lane, g);
          __syncwarp();
          stg64_store(sw, lane, reinterpret_cast<uint8_t*>(p.vg + (long long)wrow0 * p.N + cg), (long long)p.N * 2, rows_valid);
#pragma unroll
          for (int j = 0; j < 32; j += 2) {
            const float2 o = geglu_pair(make_float2(g[j], g[j + 1]), make_float2(v[j], v[j + 1]));
            g[j] = o.x; g[j + 1] = o.y;
          }
          if constexpr (EPI == EPI_GEGLU_DROP) {
#pragma unroll
            for (int j = 0; j < 32; ++j) g[j] = (keep[c] >> j) & 1u ? g[j] * p.drop.scale : 0.f;
          }
          __syncwarp();
          stg64_put_pack(sw, lane, g);
          __syncwarp();
          stg64_store(sw, lane, reinterpret_cast<uint8_t*>(p.h + (long long)wrow0 * (p.N / 2) + n_blk * 64 + c * 32), (long long)p.N, rows_valid);
          __syncwarp();
        }
      }
      if (!GEGLU && has_next) named_bar_arrive(BAR_ACC + (cw ^ 1), 256);   // accumulator and staging tiles are free for item nth + 1
    }
  }
  if constexpr (CL > 1) {
    __syncthreads();
    cluster_sync_all();                                   // no CTA leaves while its peer can still multicast into it or arrive on its barriers
  }
}

// ------------------------------------------------------------------------------------------------ EPI_STORE, 256 x 128 cooperative tile
// For plain-store launches with long work items (the dgrad / wgrad products), where the main loop is the whole cost and the ping-pong
// epilogue overlap buys little.  Both consumer warpgroups work on ONE 256 x 128 tile: warpgroup cw owns rows 128 cw .. + 127 and issues
// exactly the two wgmma.m64n128k16 per 16-deep k step of the ping-pong kernel, from its half of the 256-row A tile and the shared B tile,
// so its accumulators are bit-identical to those of the 128 x 128 tile 2 m + cw there.  Per byte fetched from L2 a stage carries 4/3 of the
// MMA work, and the same ring depth covers twice the MMA time.  A ring slot is released when all 8 consumer warps have arrived; the
// warpgroups may drift apart by less than STAGES k-blocks, which keeps the parity waits exact.
// No fp32 accumulator tile: after the main loop each warp moves its fragments 32 columns at a time through its own 4 KB staging tile into
// the per-row layout of store_slice (warp q of warpgroup cw: slice rows 0-15 = tile rows 128 cw + 16 q + i, 16-31 = those + 64).
struct GemmWideCfg {
  static constexpr int BM = 256;
  static constexpr int THREADS = 384;
  static constexpr int STAGES = 4;
  static constexpr int A_BYTES = BM * GEMM_BK * 2;
  static constexpr int B_BYTES = GEMM_BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;             // 48 KB
  static constexpr int STAGING = 8 * 4096;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one block");
};

template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(384, 1)
gemm_sm90_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using Cfg = GemmWideCfg;
  constexpr int BM = Cfg::BM, BN = GEMM_BN, STAGES = Cfg::STAGES;
  static_assert(Cfg::STAGE_BYTES % 1024 == 0, "stage alignment");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* staging = smem + STAGES * Cfg::STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + Cfg::STAGING);    // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                     // [STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const GemmSched<BM, 1> sched(p);
  const int num_items = sched.num_items;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }    // empty: one arrival per consumer warp
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================================================== TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      GemmRing<STAGES> ring;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const auto w = sched.work(item, 0);
        for (int kb = w.kb0; kb < w.kb1; ++kb)
          gemm_fill<Cfg, A_MN, B_MN, 1, false>(smem, full_bar, empty_bar, ring, &tmA, nullptr, &tmB, p, kb, w.m_blk, w.n_blk, 0);
      }
    }
  } else {
    // ===================================================== consumers: both warpgroups on every item
    setmaxnreg_inc<232>();
    const int cw = (warp >> 2) - 1;            // rows 128 cw .. + 127 of the tile
    const int quad = warp & 3;                 // fragment rows 16 quad .. + 15 of each 64-row half
    uint8_t* sw = staging + (4 * cw + quad) * 4096;
    // this warpgroup's 128 rows of A: 128 rows further down (K-major) or the third and fourth 64-wide MN blocks; 16 KB either way
    const uint32_t a_half = (uint32_t)cw * (A_MN ? 2 * GEMM_BK * 128 : 128 * 128);
    GemmRing<STAGES> ring;
    auto release = [&](int s) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[s]); };
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      const auto [m_blk, n_blk, kb0, kb1] = sched.work(item, 0);
      float d0[64], d1[64];                                   // accumulator rows 0-63 / 64-127 of this warpgroup's half
      const int last_stage = gemm_mainloop<Cfg, A_MN, B_MN>(smem, full_bar, ring, a_half, kb0, kb1, d0, d1, release);
      gemm_drain(d0, d1, last_stage, release);

      // ---- epilogue: 32-column slices, fragments -> staging tile -> one row per thread -> store_slice
      const int wrow0 = m_blk * BM + 128 * cw + 16 * quad;
      const int r0 = lane >> 2;
#pragma unroll
      for (int c = 0; c < BN / 32; ++c) {
        const int cbase = n_blk * BN + c * 32;
        if (cbase >= p.N) break;
#pragma unroll
        for (int q4 = 0; q4 < 4; ++q4) {
          const int q = 4 * c + q4, col = 8 * q4 + 2 * (lane & 3);
          auto put2 = [&](int rr, float x, float y) {
            *reinterpret_cast<float2*>(sw + rr * 128 + ((((col >> 2) ^ (rr & 7))) << 4) + (col & 3) * 4) = make_float2(x, y);
          };
          put2(r0, d0[4 * q], d0[4 * q + 1]);
          put2(r0 + 8, d0[4 * q + 2], d0[4 * q + 3]);
          put2(r0 + 16, d1[4 * q], d1[4 * q + 1]);
          put2(r0 + 24, d1[4 * q + 2], d1[4 * q + 3]);
        }
        __syncwarp();
        uint32_t r[32];
        stg_get<8>(sw, lane, r);
        __syncwarp();
        store_slice(p, sw, lane, r, cbase, [&](int i) { return wrow0 + (i & 15) + ((i >> 4) << 6); });
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) != cudaSuccess || !f) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(f);
  }
  return fn;
}

// bf16 2-D tensor map: `inner` contiguous elements per row, `outer` rows, row pitch `ld` elements,
// box = 64 x box_rows, 128-byte swizzle, zero OOB fill.
inline int make_tmap_bf16(CUtensorMap* tm, const void* ptr, long long inner, long long outer, long long ld, int box_rows) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return -1;
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -(int)r - 1000;
}

struct GemmOperand {
  const void* ptr;
  long long ld;      // row pitch in elements of the stored matrix
  bool mn_major;     // false: stored [MN][K];  true: stored [K][MN]
  const void* ptr2 = nullptr;   // optional second K segment of A (K-major only), starting at k = GemmParams::K1
  long long ld2 = 0;
};

// tensor map of operand X (mn rows of depth k): K-major boxes are 64 deep x box_rows, MN-major ones one 64-wide MN block x 64 deep
inline int make_operand_tmap(CUtensorMap* tm, const GemmOperand& X, long long mn, long long k, int box_rows) {
  return X.mn_major ? make_tmap_bf16(tm, X.ptr, mn, k, X.ld, GEMM_BK) : make_tmap_bf16(tm, X.ptr, k, mn, X.ld, box_rows);
}

// launch of a persistent kernel without clusters: one CTA per SM, at most one per work item.  The dynamic shared-memory limit is
// raised on the kernel's first launch.
template <class Cfg, auto kern, class... Args>
int launch_persistent(int items, int num_sms, cudaStream_t stream, const Args&... args) {
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES) != cudaSuccess) return -2;
    attr_set = true;
  }
  const int grid = items < num_sms ? items : num_sms;
  kern<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(args...);
  return cudaGetLastError() == cudaSuccess ? 0 : -3;
}

// CTA pairing (CL = 2): mode 1 (default) never, 2 every launch, 3 launches with at least 16 k-blocks per work item and two tiles per SM.  Set by
// tfx_gemm_set_cluster_mode, or once from the environment (TFX_GEMM_CLUSTER).  Off by default: on an H100 (400 W limit) the config-2 step's GEMM
// time doubled with mode 3 (64 -> 129 ms per step, same machine, alternated runs).
inline int& gemm_cluster_mode_ref() {
  static int mode = -1;
  if (mode < 0) { const char* e = getenv("TFX_GEMM_CLUSTER"); mode = e ? atoi(e) : 1; }
  return mode;
}

// split-K factor a launch really uses: clamped to [1, k-blocks], then lowered until no split is empty
inline int gemm_effective_splits(int K, int k_splits) {
  const int kbt = (K + GEMM_BK - 1) / GEMM_BK;
  int s = k_splits < 1 ? 1 : k_splits > kbt ? kbt : k_splits;
  const int per = (kbt + s - 1) / s;
  return (kbt + per - 1) / per;
}
inline int gemm_kb_per_item(int K, int k_splits) { return ((K + GEMM_BK - 1) / GEMM_BK + k_splits - 1) / k_splits; }

// Tile of the plain-store launches (tfx_gemm_store): mode 1 (default) the 256 x 128 cooperative tile for work items of at least
// GEMM_WIDE_MIN_KB k-blocks when CTA pairing is off, else the 128 x 128 ping-pong tile; 2 always the wide tile; 3 never.  Set by
// tfx_gemm_set_wide_mode (tests and tools/bench_gemm.py compare the two paths with it).
constexpr int GEMM_WIDE_MIN_KB = 16;
inline int& gemm_wide_mode_ref() { static int mode = 1; return mode; }
inline bool gemm_store_wide(int K, int k_splits) {
  const int mode = gemm_wide_mode_ref();
  if (mode != 1) return mode == 2;
  return gemm_cluster_mode_ref() == 1 && gemm_kb_per_item(K, gemm_effective_splits(K, k_splits)) >= GEMM_WIDE_MIN_KB;
}

template <bool A_MN, bool B_MN>
int launch_gemm_wide_t(const GemmOperand& A, const GemmOperand& B, const GemmParams& p_in, int num_sms, cudaStream_t stream) {
  using Cfg = GemmWideCfg;
  GemmParams p = p_in;
  p.K1 = p.K;
  p.k_splits = gemm_effective_splits(p.K, p.k_splits);
  const int items = ((p.M + Cfg::BM - 1) / Cfg::BM) * ((p.N + GEMM_BN - 1) / GEMM_BN) * p.k_splits;
  if (items <= 0) return 0;
  CUtensorMap tmA, tmB;
  int rc = make_operand_tmap(&tmA, A, p.M, p.K, Cfg::BM);
  if (rc) return rc;
  rc = make_operand_tmap(&tmB, B, p.N, p.K, GEMM_BN);
  if (rc) return rc;
  return launch_persistent<Cfg, gemm_sm90_wide_kernel<A_MN, B_MN>>(items, num_sms, stream, tmA, tmB, p);
}

template <bool A_MN, bool B_MN, int EPI>
int launch_gemm_t(const GemmOperand& A, const GemmOperand& B, const GemmParams& p_in, int num_sms, cudaStream_t stream) {
  using Cfg = GemmCfg<EPI>;
  GemmParams p = p_in;
  CUtensorMap tmA, tmA2, tmB;
  const bool two = (!A_MN) && A.ptr2 != nullptr;
  if (!two) p.K1 = p.K;
  int rc = make_operand_tmap(&tmA, A, p.M, p.K1, GEMM_BM);         // the first K segment (all of K unless A is split)
  if (rc) return rc;
  if (two) { rc = make_tmap_bf16(&tmA2, A.ptr2, p.K - p.K1, p.M, A.ld2, GEMM_BM); if (rc) return rc; } else tmA2 = tmA;
  p.k_splits = gemm_effective_splits(p.K, p.k_splits);
  const int m_tiles = (p.M + GEMM_BM - 1) / GEMM_BM, n_tiles = (p.N + GEMM_BN - 1) / GEMM_BN;
  const int items = m_tiles * n_tiles * p.k_splits;
  if (items <= 0) return 0;
  const int mode = gemm_cluster_mode_ref();
  const int kb_item = gemm_kb_per_item(p.K, p.k_splits);      // k-blocks per work item
  const bool paired = mode == 2 || (mode == 3 && m_tiles >= 2 && kb_item >= 16 && items >= 2 * num_sms);
  // paired CTAs each fetch half of the B tile: the K-major box is 64 rows (the MN-major box is one 64-wide block either way)
  rc = make_operand_tmap(&tmB, B, p.N, p.K, paired ? GEMM_BN / 2 : GEMM_BN);
  if (rc) return rc;
  if (paired) {
    auto kern = gemm_sm90_kernel<A_MN, B_MN, EPI, 2>;
    static int max_clusters = 0;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.blockDim = dim3(Cfg::THREADS); cfg.dynamicSmemBytes = Cfg::SMEM_BYTES; cfg.stream = stream; cfg.attrs = at; cfg.numAttrs = 1;
    if (!max_clusters) {
      if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES) != cudaSuccess) return -2;
      cfg.gridDim = dim3(2 * (num_sms / 2));
      int nc = 0;
      if (cudaOccupancyMaxActiveClusters(&nc, kern, &cfg) != cudaSuccess || nc < 1) { cudaGetLastError(); nc = num_sms / 2; }
      max_clusters = nc < num_sms / 2 ? nc : num_sms / 2;
    }
    const int pair_items = ((m_tiles + 1) / 2) * n_tiles * p.k_splits;
    const int clusters = pair_items < max_clusters ? pair_items : max_clusters;
    cfg.gridDim = dim3(2 * clusters);
    return cudaLaunchKernelEx(&cfg, kern, tmA, tmA2, tmB, p) == cudaSuccess ? 0 : -3;
  }
  return launch_persistent<Cfg, gemm_sm90_kernel<A_MN, B_MN, EPI, 1>>(items, num_sms, stream, tmA, tmA2, tmB, p);
}

}  // namespace tfx
