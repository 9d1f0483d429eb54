// Warp-per-token ("row") kernels of the Transfusion hot path: adaptive LayerNorm (FiLM / text select),
// branch-output gating backward, depth-wise AttentionResidual, final RMSNorm, token assemble,
// qk-RMSNorm+RoPE backward.  All HBM-bound: one contiguous 512 B run per warp access, fp32 math,
// warp-shuffle reductions, no shared memory.  Reference math: transfusion_pytorch/
// transfusion.py:640-775 (AdaptiveWrapper), 779-829 (RMSNorm, AttentionResidual), 946-965 (qk norm, RoPE),
// 3173-3184 (token select).
#include "common.cuh"
#include <string.h>
#include "../../include/tfx_b200.h"

namespace tfx {

constexpr int MAX_HIDDENS = TFX_MAX_DEPTH + 1;    // x0 and every layer output: 65 pointers, 520 B of kernel parameters
struct HiddenList { const __nv_bfloat16* p[MAX_HIDDENS]; };

// Wide rows (D = 1536, 2048: NCH 12, 16).  The lane layout stays the same, but a whole row per lane (48 / 64 floats per array) no longer fits
// in registers next to the other rows a kernel holds.  The kernels that would spill take such rows in groups of WIDE_GROUP chunks
// (512 columns, 16 floats per lane) instead: a row reduction is one pass over the groups, and the apply pass reads each group again - from
// the row's cp.async ring slot where the kernel has one, else from global memory, where the row was just read and is still cached.
// Per-column accumulators that outlive a row live in per-warp shared-memory rows; a lane only touches its own columns there, so no barrier
// is needed.  Every kernel with NCH <= 8 keeps its register-row form.
constexpr int WIDE_GROUP = 4;

// ------------------------------------------------------------------------------------ adaLN forward
// u = isM ? LN(x)*(gamma_c+1)+beta_c : LN(x)*(g+1)      (T.py:747-755; text-only 677-679)
// The fp32 token rows stream through a per-warp ring of shared-memory slots filled by lane-private cp.async pieces (ADALN_FWD_RING - 1 rows per
// warp in flight, no registers spent) - with one row per warp in flight the loads are latency-bound.
// The FiLM rows (L2-resident, address depends on the token's condition row) are plain loads; the condition row is fetched one row ahead.
// Wide rows (NCH > 8, see WIDE_GROUP) are not copied to registers: the mean, variance and apply passes each read the row's ring slot in
// 512-column groups, and the slot is refilled after the apply pass.  Three 8 KB slots per warp keep the ring within 227 KB at D = 2048.
template <int NCH> constexpr int ADALN_FWD_RING = NCH > 8 ? 3 : 4;
template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) adaln_fwd_k(const float* __restrict__ x, const int* __restrict__ cond_row,
                                                          const float* __restrict__ film, long long film_ld,
                                                          const float* __restrict__ g, __nv_bfloat16* __restrict__ u,
                                                          float* __restrict__ stats, int M) {
  constexpr int D = NCH * 128;
  constexpr int RING = ADALN_FWD_RING<NCH>;
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  extern __shared__ __align__(16) float adaln_ring[];
  const float* ring = adaln_ring + (threadIdx.x >> 5) * (RING * D);
  const uint32_t ring_u32 = (uint32_t)__cvta_generic_to_shared(ring);
  int iss_row = warp0, iss_slot = 0;
  auto issue = [&]() {
    if (iss_row < M) {
      const float* f = x + (long long)iss_row * D + lane * 4;
#pragma unroll
      for (int c = 0; c < NCH; ++c) cp_async_16(ring_u32 + (iss_slot * D + c * 128 + lane * 4) * 4, f + c * 128);
      iss_row += nwarps;
    }
    cp_async_commit();
    iss_slot = iss_slot + 1 == RING ? 0 : iss_slot + 1;
  };
#pragma unroll
  for (int i = 0; i < RING; ++i) issue();
  int cons_slot = 0;
  if constexpr (NCH > 8) {
    constexpr int W = WIDE_GROUP;
    int cr_next = (cond_row && warp0 < M) ? cond_row[warp0] : -1;
    for (int row = warp0; row < M; row += nwarps) {
      const int cr = cr_next;
      cr_next = (cond_row && row + nwarps < M) ? cond_row[row + nwarps] : -1;
      cp_async_wait<RING - 1>();
      const float* xs = ring + cons_slot * D;
      float v[W * 4], s = 0.f, q = 0.f;
#pragma unroll 1
      for (int c0 = 0; c0 < NCH; c0 += W) {
        load_row_f32<W>(xs + c0 * 128, lane, v);
#pragma unroll
        for (int i = 0; i < W * 4; ++i) s += v[i];
      }
      const float mean = warp_sum(s) * (1.f / D);
#pragma unroll 1
      for (int c0 = 0; c0 < NCH; c0 += W) {
        load_row_f32<W>(xs + c0 * 128, lane, v);
#pragma unroll
        for (int i = 0; i < W * 4; ++i) { v[i] -= mean; q += v[i] * v[i]; }
      }
      const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + 1e-5f);
#pragma unroll 1
      for (int c0 = 0; c0 < NCH; c0 += W) {
        float sc[W * 4], bt[W * 4];
        load_row_f32<W>(xs + c0 * 128, lane, v);
        if (cr >= 0) {
          load_row_f32<W>(film + cr * film_ld + c0 * 128, lane, sc);
          load_row_f32<W>(film + cr * film_ld + D + c0 * 128, lane, bt);
#pragma unroll
          for (int i = 0; i < W * 4; ++i) v[i] = (v[i] - mean) * rstd * (sc[i] + 1.f) + bt[i];
        } else {
          load_row_f32<W>(g + c0 * 128, lane, sc);
#pragma unroll
          for (int i = 0; i < W * 4; ++i) v[i] = (v[i] - mean) * rstd * (sc[i] + 1.f);
        }
        store_row_bf16<W>(u + (long long)row * D + c0 * 128, lane, v);
      }
      cons_slot = cons_slot + 1 == RING ? 0 : cons_slot + 1;
      issue();
      if (lane == 0) { stats[2 * row] = mean; stats[2 * row + 1] = rstd; }
    }
    cp_async_wait<0>();
    return;
  }
  float gv[NCH * 4];
  load_row_f32<NCH>(g, lane, gv);
  int cr_next = (cond_row && warp0 < M) ? cond_row[warp0] : -1;
  for (int row = warp0; row < M; row += nwarps) {
    const int cr = cr_next;
    float v[NCH * 4], gm[NCH * 4], bt[NCH * 4];
    if (cr >= 0) {
      load_row_f32<NCH>(film + cr * film_ld, lane, gm);
      load_row_f32<NCH>(film + cr * film_ld + D, lane, bt);
    }
    cr_next = (cond_row && row + nwarps < M) ? cond_row[row + nwarps] : -1;
    cp_async_wait<RING - 1>();
    load_row_f32<NCH>(ring + cons_slot * D, lane, v);
    cons_slot = cons_slot + 1 == RING ? 0 : cons_slot + 1;
    issue();
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) s += v[i];
    const float mean = warp_sum(s) * (1.f / D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) { v[i] -= mean; q += v[i] * v[i]; }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + 1e-5f);
    if (cr >= 0) {
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) v[i] = v[i] * rstd * (gm[i] + 1.f) + bt[i];
    } else {
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) v[i] = v[i] * rstd * (gv[i] + 1.f);
    }
    store_row_bf16<NCH>(u + (long long)row * D, lane, v);
    if (lane == 0) { stats[2 * row] = mean; stats[2 * row + 1] = rstd; }
  }
  cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------ adaLN backward
// dx += LN'(du * scale);  d(gamma_c) += du*xhat, d(beta_c) += du   (per cond row)   d(g) += du*xhat (text)
template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS, 2) adaln_bwd_k(const float* __restrict__ du, const float* __restrict__ x,
                                                          const float* __restrict__ stats, const int* __restrict__ cond_row,
                                                          const float* __restrict__ film, long long film_ld, const float* __restrict__ g,
                                                          float* __restrict__ dx, float* __restrict__ dfilm, long long dfilm_ld,
                                                          float* __restrict__ dg, int M, int tpw) {
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int r0 = min(M, warp * tpw), r1 = min(M, r0 + tpw);      // (no early return: block-wide barrier below)
  // text rows all update the same [D] vector: per-warp smem rows + one block-level reduction instead of one global atomic per warp
  // (thousands of same-address atomics serialise in the L2 atomic units).  Condition rows are shared by only a few warps: direct red.
  if constexpr (NCH > 8) {
    // wide: one pass for m1, m2 and a second that reads du / x / the scale again and applies; the per-warp accumulators are shared-memory
    // rows [d(gamma_c) | d(beta_c) of the current condition row | d(g) of the text rows], 3 x D floats per warp (dynamic, 192 KB at 2048)
    constexpr int W = WIDE_GROUP;
    extern __shared__ __align__(16) float adaln_bwd_acc[];
    float* accA = adaln_bwd_acc + (threadIdx.x >> 5) * 3 * D;
    float* accB = accA + D;
    float* my_g = accB + D;
    float z[W * 4];
#pragma unroll
    for (int i = 0; i < W * 4; ++i) z[i] = 0.f;
#pragma unroll 1
    for (int c0 = 0; c0 < NCH; c0 += W) store_row_f32<W>(my_g + c0 * 128, lane, z);
    int cur = -1;
    for (int row = r0; row < r1; ++row) {
      const int cr = cond_row ? cond_row[row] : -1;
      if (cr != cur) {
#pragma unroll 1
        for (int c0 = 0; c0 < NCH; c0 += W) {
          float a[W * 4];
          if (cur >= 0) {
            load_row_f32<W>(accA + c0 * 128, lane, a); red_row_f32<W>(dfilm + cur * dfilm_ld + c0 * 128, lane, a);
            load_row_f32<W>(accB + c0 * 128, lane, a); red_row_f32<W>(dfilm + cur * dfilm_ld + D + c0 * 128, lane, a);
          }
          store_row_f32<W>(accA + c0 * 128, lane, z); store_row_f32<W>(accB + c0 * 128, lane, z);
        }
        cur = cr;
      }
      const float mean = stats[2 * row], rstd = stats[2 * row + 1];
      const float* scale = cr >= 0 ? film + cr * film_ld : g;
      const float* dur = du + (long long)row * D;
      const float* xr = x + (long long)row * D;
      float m1 = 0.f, m2 = 0.f;
#pragma unroll 1
      for (int c0 = 0; c0 < NCH; c0 += W) {
        float d[W * 4], xh[W * 4], sc[W * 4];
        load_row_f32<W>(dur + c0 * 128, lane, d);
        load_row_f32<W>(xr + c0 * 128, lane, xh);
        load_row_f32<W>(scale + c0 * 128, lane, sc);
#pragma unroll
        for (int i = 0; i < W * 4; ++i) {
          xh[i] = (xh[i] - mean) * rstd;
          d[i] *= sc[i] + 1.f;
          m1 += d[i]; m2 += d[i] * xh[i];
        }
      }
      m1 = warp_sum(m1) * (1.f / D); m2 = warp_sum(m2) * (1.f / D);
      float* acc = cr >= 0 ? accA : my_g;
#pragma unroll 1
      for (int c0 = 0; c0 < NCH; c0 += W) {
        float d[W * 4], xh[W * 4], sc[W * 4], a[W * 4];
        load_row_f32<W>(dur + c0 * 128, lane, d);
        load_row_f32<W>(xr + c0 * 128, lane, xh);
        load_row_f32<W>(scale + c0 * 128, lane, sc);
        load_row_f32<W>(acc + c0 * 128, lane, a);
#pragma unroll
        for (int i = 0; i < W * 4; ++i) { xh[i] = (xh[i] - mean) * rstd; a[i] += d[i] * xh[i]; }
        store_row_f32<W>(acc + c0 * 128, lane, a);
        if (cr >= 0) {
          load_row_f32<W>(accB + c0 * 128, lane, a);
#pragma unroll
          for (int i = 0; i < W * 4; ++i) a[i] += d[i];
          store_row_f32<W>(accB + c0 * 128, lane, a);
        }
        load_row_f32<W>(dx + (long long)row * D + c0 * 128, lane, a);
#pragma unroll
        for (int i = 0; i < W * 4; ++i) a[i] += rstd * (d[i] * (sc[i] + 1.f) - m1 - xh[i] * m2);
        store_row_f32<W>(dx + (long long)row * D + c0 * 128, lane, a);
      }
    }
    if (cur >= 0) {
#pragma unroll 1
      for (int c0 = 0; c0 < NCH; c0 += W) {
        float a[W * 4];
        load_row_f32<W>(accA + c0 * 128, lane, a); red_row_f32<W>(dfilm + cur * dfilm_ld + c0 * 128, lane, a);
        load_row_f32<W>(accB + c0 * 128, lane, a); red_row_f32<W>(dfilm + cur * dfilm_ld + D + c0 * 128, lane, a);
      }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < D; c += ROW_THREADS) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < WARPS_PER_BLOCK; ++w) t += adaln_bwd_acc[w * 3 * D + 2 * D + c];
      if (t != 0.f) atomicAdd(dg + c, t);
    }
    return;
  }
  __shared__ __align__(16) float red_g[WARPS_PER_BLOCK][D];
  float* my_g = red_g[threadIdx.x >> 5];
  {
    float z[NCH * 4];
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) z[i] = 0.f;
    store_row_f32<NCH>(my_g, lane, z);
  }
  float gv[NCH * 4];
  load_row_f32<NCH>(g, lane, gv);
  float accA[NCH * 4], accB[NCH * 4];
  int cur = -2;
  auto flush = [&]() {
    if (cur == -2) return;
    if (cur >= 0) { red_row_f32<NCH>(dfilm + cur * dfilm_ld, lane, accA); red_row_f32<NCH>(dfilm + cur * dfilm_ld + D, lane, accB); }
    else {
      float t[NCH * 4];
      load_row_f32<NCH>(my_g, lane, t);
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) t[i] += accA[i];
      store_row_f32<NCH>(my_g, lane, t);
    }
  };
  for (int row = r0; row < r1; ++row) {
    const int cr = cond_row ? cond_row[row] : -1;
    if (cr != cur) {
      flush(); cur = cr;
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) { accA[i] = 0.f; accB[i] = 0.f; }
    }
    float d[NCH * 4], xh[NCH * 4], sc[NCH * 4];
    load_row_f32<NCH>(du + (long long)row * D, lane, d);
    load_row_f32<NCH>(x + (long long)row * D, lane, xh);
    const float mean = stats[2 * row], rstd = stats[2 * row + 1];
    if (cr >= 0) {
      load_row_f32<NCH>(film + cr * film_ld, lane, sc);
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) sc[i] += 1.f;
    } else {
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) sc[i] = gv[i] + 1.f;
    }
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) {
      xh[i] = (xh[i] - mean) * rstd;
      accA[i] += d[i] * xh[i];
      accB[i] += d[i];
      d[i] *= sc[i];
      m1 += d[i]; m2 += d[i] * xh[i];
    }
    m1 = warp_sum(m1) * (1.f / D); m2 = warp_sum(m2) * (1.f / D);
    float o[NCH * 4];
    load_row_f32<NCH>(dx + (long long)row * D, lane, o);
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) o[i] += rstd * (d[i] - m1 - xh[i] * m2);
    store_row_f32<NCH>(dx + (long long)row * D, lane, o);
  }
  flush();
  __syncthreads();
  for (int c = threadIdx.x; c < D; c += ROW_THREADS) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS_PER_BLOCK; ++w) t += red_g[w][c];
    if (t != 0.f) atomicAdd(dg + c, t);
  }
}

// ------------------------------------------------------------------------------------ branch-output gate backward
// forward was x_out = x_res + y * s,  s = isM ? sigmoid(z_c) : (layerscale+1)       (T.py:765-769)
// dy = dx*s (bf16, feeds the dgrad / wgrad GEMMs);  d s accumulated per cond row / for layerscale.
// block-level column reduction of per-warp register rows, then one atomicAdd per column per block
template <int NCH>
__device__ __forceinline__ void block_red_cols(float* smem /*[WARPS_PER_BLOCK][NCH*128]*/, const float (&acc)[NCH * 4], float* __restrict__ dst) {
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  store_row_f32<NCH>(smem + warp * D, lane, acc);
  __syncthreads();
  for (int c = threadIdx.x; c < D; c += ROW_THREADS) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS_PER_BLOCK; ++w) t += smem[w * D + c];
    atomicAdd(dst + c, t);
  }
}

template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) resid_bwd_k(const float* __restrict__ dx, const __nv_bfloat16* __restrict__ y,
                                                          const int* __restrict__ cond_row, const float* __restrict__ zgate, long long zgate_ld,
                                                          const float* __restrict__ ls, __nv_bfloat16* __restrict__ dy,
                                                          float* __restrict__ dzgate, long long dzgate_ld, float* __restrict__ dls,
                                                          float* __restrict__ dbias, int M, int tpw) {
  constexpr int D = NCH * 128;
  // every column is independent here, so a wide row is taken one 512-column group at a time, each group over all of the warp's rows
  // (one group of NCH chunks up to NCH = 8)
  constexpr int W = NCH > 8 ? WIDE_GROUP : NCH;
  extern __shared__ float red_smem[];
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int r0 = min(M, warp * tpw), r1 = min(M, r0 + tpw);
  const bool has_scale = ls != nullptr;
#pragma unroll 1
  for (int c0 = 0; c0 < NCH; c0 += W) {
    float lsv[W * 4];
    if (has_scale) load_row_f32<W>(ls + c0 * 128, lane, lsv);
    float acc[W * 4], accb[W * 4], accl[W * 4];      // per cond row / bias / layerscale (text rows) accumulators
#pragma unroll
    for (int i = 0; i < W * 4; ++i) { accb[i] = 0.f; accl[i] = 0.f; }
    int cur = -2;
    auto flush = [&]() {
      if (cur == -2 || !has_scale) return;
      if (cur >= 0) red_row_f32<W>(dzgate + cur * dzgate_ld + c0 * 128, lane, acc);
      else {
#pragma unroll
        for (int i = 0; i < W * 4; ++i) accl[i] += acc[i];
      }
    };
    for (int row = r0; row < r1; ++row) {
      const int cr = (cond_row && zgate) ? cond_row[row] : -1;
      if (cr != cur) {
        flush(); cur = cr;
#pragma unroll
        for (int i = 0; i < W * 4; ++i) acc[i] = 0.f;
      }
      float d[W * 4];
      load_row_f32<W>(dx + (long long)row * D + c0 * 128, lane, d);
      if (has_scale) {
        float yv[W * 4], sc[W * 4];
        load_row_bf16<W>(y + (long long)row * D + c0 * 128, lane, yv);
        if (cr >= 0) load_row_f32<W>(zgate + cr * zgate_ld + c0 * 128, lane, sc);
#pragma unroll
        for (int i = 0; i < W * 4; ++i) {
          const float s = cr >= 0 ? sc[i] : lsv[i] + 1.f;
          acc[i] += d[i] * yv[i];
          d[i] *= s;
        }
      }
#pragma unroll
      for (int i = 0; i < W * 4; ++i) accb[i] += d[i];
      store_row_bf16<W>(dy + (long long)row * D + c0 * 128, lane, d);
    }
    flush();
    if (dbias) block_red_cols<W>(red_smem, accb, dbias + c0 * 128);     // uniform branch: every thread of the block reaches the barrier
    if (has_scale) { __syncthreads(); block_red_cols<W>(red_smem, accl, dls + c0 * 128); }   // layerscale gradient: one atomic per column per block
    if (NCH > W) __syncthreads();                     // the next group reuses red_smem
  }
}

// ------------------------------------------------------------------------------------ AttentionResidual forward
// sim_l = <h_l, (gamma+1)*pq> / max(|h_l|, eps)   (sqrt(D) of the RMSNorm cancels the D^-1/2 scale)
// x = sum_l softmax_l(sim) h_l           (T.py:803-829)   single pass, online softmax over depth.
// The depth loop is a serial chain (online softmax), so the hiddens of a warp's rows stream through a per-warp ring of shared-memory slots
// filled by lane-private cp.async pieces: RING - 1 row loads per warp stay in flight without spending registers (a register double buffer
// would need twice the registers per row and halve the resident warps).
constexpr int ARES_FWD_RING = 4;
template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) attn_res_fwd_k(HiddenList hid, int L1, const float* __restrict__ gamma, const float* __restrict__ pq,
                                                             float* __restrict__ xo, __nv_bfloat16* __restrict__ xb, float* __restrict__ lse_out, int M) {
  constexpr int D = NCH * 128;
  constexpr int RING = ARES_FWD_RING;
  constexpr int SLOT = D * 2;                                   // bytes: one bf16 row
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  extern __shared__ __align__(16) uint8_t ares_ring[];
  const uint8_t* ring = ares_ring + (threadIdx.x >> 5) * (RING * SLOT);
  const uint32_t ring_u32 = (uint32_t)__cvta_generic_to_shared(ring);
  int iss_row = warp0, iss_k = 0, iss_slot = 0;
  auto issue = [&]() {
    if (iss_row < M) {
      const uint32_t dst = ring_u32 + iss_slot * SLOT;
      const __nv_bfloat16* b = hid.p[iss_k] + (long long)iss_row * D + lane * 4;
#pragma unroll
      for (int c = 0; c < NCH; ++c) cp_async_8(dst + (c * 128 + lane * 4) * 2, b + c * 128);
      if (++iss_k == L1) { iss_k = 0; iss_row += nwarps; }
    }
    cp_async_commit();
    iss_slot = iss_slot + 1 == RING ? 0 : iss_slot + 1;
  };
#pragma unroll
  for (int i = 0; i < RING; ++i) issue();
  int cons_slot = 0;
  float w[NCH * 4], t[NCH * 4];
  load_row_f32<NCH>(gamma, lane, w);
  load_row_f32<NCH>(pq, lane, t);
#pragma unroll
  for (int i = 0; i < NCH * 4; ++i) w[i] = (w[i] + 1.f) * t[i];
  for (int row = warp0; row < M; row += nwarps) {
    float acc[NCH * 4];
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) acc[i] = 0.f;
    float m = -INFINITY, l = 0.f;
    for (int k = 0; k < L1; ++k) {
      float h[NCH * 4];
      cp_async_wait<RING - 1>();
      load_row_bf16<NCH>(reinterpret_cast<const __nv_bfloat16*>(ring + cons_slot * SLOT), lane, h);
      cons_slot = cons_slot + 1 == RING ? 0 : cons_slot + 1;
      issue();
      float ss = 0.f, dot = 0.f;
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) { ss += h[i] * h[i]; dot += h[i] * w[i]; }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { ss += __shfl_xor_sync(0xffffffffu, ss, o); dot += __shfl_xor_sync(0xffffffffu, dot, o); }
      const float sim = dot / fmaxf(sqrtf(ss), 1e-12f);
      const float mn = fmaxf(m, sim);
      const float a = __expf(m - mn), b = __expf(sim - mn);
      l = l * a + b; m = mn;
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) acc[i] = acc[i] * a + h[i] * b;
    }
    const float inv = 1.f / l;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) acc[i] *= inv;
    store_row_f32<NCH>(xo + (long long)row * D, lane, acc);
    if (xb) store_row_bf16<NCH>(xb + (long long)row * D, lane, acc);
    if (lse_out && lane == 0) lse_out[row] = m + __logf(l);
  }
  cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------ AttentionResidual backward, deferred assembly
// Layer i' adds to the gradient of every hidden k it mixes  a_k dx + c1_k w - c2_k h_k,  and to dw (-> d gamma, d pq)  c1_k h_k, where
//     a_k = exp(sim_k - lse)  (the log-sum-exp saved by the forward),   ds_k = a_k (<h_k, dx> - <x_out, dx>),   c1_k = ds_k / |h_k|,   c2_k = ds_k <h_k, w> / |h_k|^3
// (the softmax-backward mean  sum_k a_k <h_k, dx>  equals <x_out, dx>, x_out being the saved forward output, so every h_k is read once per layer).
// |h_k| stands for max(|h_k|, 1e-12) as F.normalize clamps it; below the clamp the norm is a constant for the gradient, so c2_k = 0 there.
// Adding these terms into dH_k at every layer would read-modify-write (i + 2) fp32 rows per token and layer.  Each term is (per-token scalars) x (a vector
// that already exists: the incoming gradient dx_i', the layer's w_i', the hidden itself), so this kernel stores the three scalars per (token, layer, hidden) -
// 12 bytes instead of 2 KB - and assembles the COMPLETE gradient of one hidden, once, when the backward pass needs it:
//     G_k = sum_{i' >= k-1} [ a_{i',k} dx_{i'} + c1_{i',k} w_{i'} ] - (sum_{i'} c2_{i',k}) h_k
// Layer i (own = 1): scalar pass over h_0 .. h_{i+1} (parameter gradients, scalars out), then G_{i+1} from its own term and the stored scalars / incoming
// gradients of the later layers.  own = 0: only the assembly (G_0, after the first layer).  Bytes per token over 8 layers: 167 KB instead of the 234 KB of
// accumulating into dH_k at every layer.
// One launch assembles at most BWD2_CHUNK later layers (their w rows in shared memory, one lane each for their scalars).  The sum is linear in the
// later layers, so deeper models add the rest chunk by chunk: ACC launches (own = 0) add their chunk's terms, c2 part included, into G.
constexpr int BWD2_CHUNK = 10;
struct ResBwd2Args {
  const __nv_bfloat16* hid[MAX_HIDDENS];   // bf16 hiddens h_0 .. h_{L1-1}
  const float* dx_later[BWD2_CHUNK];        // incoming gradients of the later AttentionResiduals (layers i+1 ..)
  const float* sc_later[BWD2_CHUNK];        // their scalars for THIS hidden: points at element [token 0][k = L1-1][0]; row stride = sc_stride floats
  const float* gam[BWD2_CHUNK + 1];         // norm_keys.gamma: own layer first (unused when own = 0), then the later layers
  const float* pq[BWD2_CHUNK + 1];
  int L1, n_later, own;
};

// Every global read of the kernel goes through a per-warp ring of row-sized shared-memory slots filled by cp.async (lane-private 16 / 8 / 4 byte
// pieces: a lane only ever reads back what it copied itself, so cp.async.wait_group is the only synchronisation).  The item order of a row is
// fixed - [scalars of the later layers + lse] [dx_out] [x_out] [h_0 .. h_{L1-1}] [dx_later ..] - so RING - 1 row loads per warp are always in
// flight (a register prefetch keeps only one).
// Wide rows (NCH > 8) take RING = 2: the shared memory at D = 2048 is 8 KB (w of the own layer) + 64 KB (accumulators, below) + 128 KB (rings).
template <int NCH> struct ResBwd2Cfg { static constexpr int RING = NCH <= 4 ? 5 : (NCH <= 8 ? 3 : 2); };

template <int NCH, bool ACC>
__global__ void __launch_bounds__(ROW_THREADS, NCH > 8 ? 1 : 2) attn_res_bwd2_k(ResBwd2Args A, const float* __restrict__ dxo, const float* __restrict__ xo, const float* __restrict__ lse,
                                                                 float* __restrict__ G, float* __restrict__ sc_out, int sc_stride, float* __restrict__ partials, int M, int tpw) {
  constexpr int D = NCH * 128;
  constexpr int RING = ResBwd2Cfg<NCH>::RING;
  constexpr int SLOT = D * 4;                                   // bytes: one fp32 row
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int r0 = min(M, warp * tpw), r1 = min(M, r0 + tpw);    // (no early return: block-wide barriers below)
  extern __shared__ __align__(16) float w_s[];                  // [max(1 + n_later, warps)][D]: w = (gamma + 1) * pq of the own layer (slot 0) and of the later ones; then the rings
  // (wide rows: [w of the own layer][accw: warps][rings], see below)
  const int w_slots = NCH > 8 ? 1 + WARPS_PER_BLOCK : ((1 + A.n_later) > WARPS_PER_BLOCK ? (1 + A.n_later) : WARPS_PER_BLOCK);
  const uint8_t* ring = reinterpret_cast<const uint8_t*>(w_s + w_slots * D) + (threadIdx.x >> 5) * (RING * SLOT);
  const uint32_t ring_u32 = (uint32_t)__cvta_generic_to_shared(ring);

  // ---- producer side of the ring
  const int n_items = A.own ? 3 + A.L1 + A.n_later : 2 + A.n_later;
  int iss_row = r0, iss_it = 0, iss_slot = 0;
  auto issue = [&]() {
    if (iss_row < r1) {
      const uint32_t dst = ring_u32 + iss_slot * SLOT;
      const int it = iss_it;
      if (it == 0) {                                            // lane j: (a, c1, c2) of later layer j for this hidden; lane 31: lse of the row
        if (lane < A.n_later) {
          const float* sp = A.sc_later[lane] + (long long)iss_row * sc_stride;
          cp_async_4(dst + lane * 16, sp); cp_async_4(dst + lane * 16 + 4, sp + 1); cp_async_4(dst + lane * 16 + 8, sp + 2);
        }
        if (A.own && lane == 31) cp_async_4(dst + 31 * 16, lse + iss_row);
      } else {
        const float* f = nullptr;
        const __nv_bfloat16* b = nullptr;
        if (A.own) {
          if (it == 1) f = dxo; else if (it == 2) f = xo; else if (it < 3 + A.L1) b = A.hid[it - 3]; else f = A.dx_later[it - 3 - A.L1];
        } else {
          if (it == 1) b = A.hid[A.L1 - 1]; else f = A.dx_later[it - 2];
        }
        if (f) {
          f += (long long)iss_row * D + lane * 4;
#pragma unroll
          for (int c = 0; c < NCH; ++c) cp_async_16(dst + (c * 128 + lane * 4) * 4, f + c * 128);
        } else {
          b += (long long)iss_row * D + lane * 4;
#pragma unroll
          for (int c = 0; c < NCH; ++c) cp_async_8(dst + (c * 128 + lane * 4) * 2, b + c * 128);
        }
      }
      if (++iss_it == n_items) { iss_it = 0; ++iss_row; }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");         // (an empty group past the last row keeps the group count uniform)
    iss_slot = iss_slot + 1 == RING ? 0 : iss_slot + 1;
  };
  // ---- consumer side: the oldest outstanding row -> registers, then its slot is refilled
  int cons_slot = 0;
  auto take_f32 = [&](float (&v)[NCH * 4]) {
    cp_async_wait<RING - 1>();
    const float* sp = reinterpret_cast<const float*>(ring + cons_slot * SLOT);
    load_row_f32<NCH>(sp, lane, v);
    cons_slot = cons_slot + 1 == RING ? 0 : cons_slot + 1;
    issue();
  };
  auto take_bf16 = [&](float (&v)[NCH * 4]) {
    cp_async_wait<RING - 1>();
    const __nv_bfloat16* sp = reinterpret_cast<const __nv_bfloat16*>(ring + cons_slot * SLOT);
    load_row_bf16<NCH>(sp, lane, v);
    cons_slot = cons_slot + 1 == RING ? 0 : cons_slot + 1;
    issue();
  };

  if constexpr (NCH > 8) {
    // Wide rows: only dx_out stays in registers next to the assembled gradient g.  Every other item is read in place from its ring slot,
    // once per pass (a hidden: the reductions, then c1 * h into accw); accw is a per-warp shared-memory row, the later layers' w are
    // recomputed from gamma / pq per column group (L2-resident), and the c2 term of the newest hidden is applied with its own term, as its
    // slot is refilled before the later layers' gradients arrive.
    float* accw_s = w_s + D + (threadIdx.x >> 5) * D;
    auto slot = [&]() { cp_async_wait<RING - 1>(); return ring + cons_slot * SLOT; };
    auto release = [&]() { cons_slot = cons_slot + 1 == RING ? 0 : cons_slot + 1; issue(); };
    if (A.own)
      for (int c = threadIdx.x; c < D; c += ROW_THREADS) w_s[c] = (A.gam[0][c] + 1.f) * A.pq[0][c];
#pragma unroll
    for (int c = 0; c < NCH; ++c) *reinterpret_cast<float4*>(accw_s + c * 128 + lane * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < RING; ++i) issue();
    __syncthreads();
    for (int row = r0; row < r1; ++row) {
      float g[NCH * 4];
      const float4 scl = *reinterpret_cast<const float4*>(slot() + lane * 16);
      release();
      float c2sum = 0.f;
      if (A.own) {
        const float lse_r = __shfl_sync(0xffffffffu, scl.x, 31);
        float dxv[NCH * 4];
        take_f32(dxv);
        float mean_da = 0.f;
        {
          const float* xs = reinterpret_cast<const float*>(slot());
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            const float4 x4 = *reinterpret_cast<const float4*>(xs + c * 128 + lane * 4);
            mean_da += x4.x * dxv[4 * c] + x4.y * dxv[4 * c + 1] + x4.z * dxv[4 * c + 2] + x4.w * dxv[4 * c + 3];
          }
          release();
        }
        mean_da = warp_sum(mean_da);
        for (int k = 0; k < A.L1; ++k) {
          const __nv_bfloat16* hs = reinterpret_cast<const __nv_bfloat16*>(slot()) + lane * 4;
          float ss = 0.f, dot = 0.f, da = 0.f;
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            const uint2 t = *reinterpret_cast<const uint2*>(hs + c * 128);
            const float2 h01 = unpack2_bf16(t.x), h23 = unpack2_bf16(t.y);
            const float4 w4 = *reinterpret_cast<const float4*>(w_s + c * 128 + lane * 4);
            ss += h01.x * h01.x + h01.y * h01.y + h23.x * h23.x + h23.y * h23.y;
            dot += h01.x * w4.x + h01.y * w4.y + h23.x * w4.z + h23.y * w4.w;
            da += h01.x * dxv[4 * c] + h01.y * dxv[4 * c + 1] + h23.x * dxv[4 * c + 2] + h23.y * dxv[4 * c + 3];
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            ss += __shfl_xor_sync(0xffffffffu, ss, o); dot += __shfl_xor_sync(0xffffffffu, dot, o); da += __shfl_xor_sync(0xffffffffu, da, o);
          }
          const float nrm = fmaxf(sqrtf(ss), 1e-12f), rn = 1.f / nrm;
          const float a = __expf(dot * rn - lse_r);
          const float ds = a * (da - mean_da);
          const float c1 = ds * rn, c2 = sqrtf(ss) < 1e-12f ? 0.f : ds * dot * rn * rn * rn;   // clamped norm: a constant for the gradient
          const bool newest = k + 1 == A.L1;
          if (newest) {
            c2sum = c2;
            for (int j = 0; j < A.n_later; ++j) c2sum += __shfl_sync(0xffffffffu, scl.z, j);
          } else if (lane < 3) {
            sc_out[(long long)row * sc_stride + k * 3 + lane] = lane == 0 ? a : (lane == 1 ? c1 : c2);
          }
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            const uint2 t = *reinterpret_cast<const uint2*>(hs + c * 128);
            const float2 h01 = unpack2_bf16(t.x), h23 = unpack2_bf16(t.y);
            float4* aw = reinterpret_cast<float4*>(accw_s + c * 128 + lane * 4);
            float4 v = *aw;
            v.x += c1 * h01.x; v.y += c1 * h01.y; v.z += c1 * h23.x; v.w += c1 * h23.y;
            *aw = v;
            if (newest) {                             // the newest hidden: its own term and the c2 term of every layer
              const float4 w4 = *reinterpret_cast<const float4*>(w_s + c * 128 + lane * 4);
              g[4 * c] = a * dxv[4 * c] + c1 * w4.x - c2sum * h01.x; g[4 * c + 1] = a * dxv[4 * c + 1] + c1 * w4.y - c2sum * h01.y;
              g[4 * c + 2] = a * dxv[4 * c + 2] + c1 * w4.z - c2sum * h23.x; g[4 * c + 3] = a * dxv[4 * c + 3] + c1 * w4.w - c2sum * h23.y;
            }
          }
          release();
        }
      } else {
        for (int j = 0; j < A.n_later; ++j) c2sum += __shfl_sync(0xffffffffu, scl.z, j);
        const __nv_bfloat16* hs = reinterpret_cast<const __nv_bfloat16*>(slot()) + lane * 4;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          const uint2 t = *reinterpret_cast<const uint2*>(hs + c * 128);
          const float2 h01 = unpack2_bf16(t.x), h23 = unpack2_bf16(t.y);
          g[4 * c] = -c2sum * h01.x; g[4 * c + 1] = -c2sum * h01.y; g[4 * c + 2] = -c2sum * h23.x; g[4 * c + 3] = -c2sum * h23.y;
        }
        release();
      }
      for (int j = 0; j < A.n_later; ++j) {
        const float* ds = reinterpret_cast<const float*>(slot()) + lane * 4;
        const float a = __shfl_sync(0xffffffffu, scl.x, j), c1 = __shfl_sync(0xffffffffu, scl.y, j);
        const float* gj = A.gam[j + 1] + lane * 4;
        const float* pj = A.pq[j + 1] + lane * 4;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          const float4 d4 = *reinterpret_cast<const float4*>(ds + c * 128);
          const float4 ga = *reinterpret_cast<const float4*>(gj + c * 128), pa = *reinterpret_cast<const float4*>(pj + c * 128);
          g[4 * c] += a * d4.x + c1 * ((ga.x + 1.f) * pa.x); g[4 * c + 1] += a * d4.y + c1 * ((ga.y + 1.f) * pa.y);
          g[4 * c + 2] += a * d4.z + c1 * ((ga.z + 1.f) * pa.z); g[4 * c + 3] += a * d4.w + c1 * ((ga.w + 1.f) * pa.w);
        }
        release();
      }
      if (ACC) {
        float o[NCH * 4];
        load_row_f32<NCH>(G + (long long)row * D, lane, o);
#pragma unroll
        for (int i = 0; i < NCH * 4; ++i) g[i] += o[i];
      }
      store_row_f32<NCH>(G + (long long)row * D, lane, g);
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    if (A.own) {
      __syncthreads();
      for (int c = threadIdx.x; c < D; c += ROW_THREADS) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < WARPS_PER_BLOCK; ++w) t += w_s[D + w * D + c];
        partials[(long long)blockIdx.x * D + c] = t;
      }
    }
    return;
  }
  for (int j = A.own ? 0 : 1; j <= A.n_later; ++j)
    for (int c = threadIdx.x; c < D; c += ROW_THREADS) w_s[j * D + c] = (A.gam[j][c] + 1.f) * A.pq[j][c];
#pragma unroll
  for (int i = 0; i < RING; ++i) issue();
  __syncthreads();
  float accw[NCH * 4];
#pragma unroll
  for (int i = 0; i < NCH * 4; ++i) accw[i] = 0.f;
  for (int row = r0; row < r1; ++row) {
    float g[NCH * 4], h[NCH * 4];
    float c2sum = 0.f;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) g[i] = 0.f;
    // item 0: this lane's later-layer scalars, lse broadcast from lane 31
    cp_async_wait<RING - 1>();
    const float4 scl = *reinterpret_cast<const float4*>(ring + cons_slot * SLOT + lane * 16);
    cons_slot = cons_slot + 1 == RING ? 0 : cons_slot + 1;
    issue();
    if (A.own) {
      const float lse_r = __shfl_sync(0xffffffffu, scl.x, 31);
      float dxv[NCH * 4];
      take_f32(dxv);
      take_f32(h);
      float mean_da = 0.f;
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) mean_da += h[i] * dxv[i];
      mean_da = warp_sum(mean_da);
      for (int k = 0; k < A.L1; ++k) {
        take_bf16(h);
        float ss = 0.f, dot = 0.f, da = 0.f;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          const float4 w4 = *reinterpret_cast<const float4*>(w_s + c * 128 + lane * 4);       // w of the own layer straight from shared memory (register budget)
          ss += h[4 * c] * h[4 * c] + h[4 * c + 1] * h[4 * c + 1] + h[4 * c + 2] * h[4 * c + 2] + h[4 * c + 3] * h[4 * c + 3];
          dot += h[4 * c] * w4.x + h[4 * c + 1] * w4.y + h[4 * c + 2] * w4.z + h[4 * c + 3] * w4.w;
          da += h[4 * c] * dxv[4 * c] + h[4 * c + 1] * dxv[4 * c + 1] + h[4 * c + 2] * dxv[4 * c + 2] + h[4 * c + 3] * dxv[4 * c + 3];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          ss += __shfl_xor_sync(0xffffffffu, ss, o); dot += __shfl_xor_sync(0xffffffffu, dot, o); da += __shfl_xor_sync(0xffffffffu, da, o);
        }
        const float nrm = fmaxf(sqrtf(ss), 1e-12f), rn = 1.f / nrm;
        const float a = __expf(dot * rn - lse_r);
        const float ds = a * (da - mean_da);
        const float c1 = ds * rn, c2 = sqrtf(ss) < 1e-12f ? 0.f : ds * dot * rn * rn * rn;   // clamped norm: a constant for the gradient
#pragma unroll
        for (int i = 0; i < NCH * 4; ++i) accw[i] += c1 * h[i];
        if (k + 1 < A.L1) {
          if (lane < 3) sc_out[(long long)row * sc_stride + k * 3 + lane] = lane == 0 ? a : (lane == 1 ? c1 : c2);
        } else {                                    // the newest hidden: its gradient is assembled right here
          c2sum = c2;
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            const float4 w4 = *reinterpret_cast<const float4*>(w_s + c * 128 + lane * 4);
            g[4 * c] = a * dxv[4 * c] + c1 * w4.x; g[4 * c + 1] = a * dxv[4 * c + 1] + c1 * w4.y;
            g[4 * c + 2] = a * dxv[4 * c + 2] + c1 * w4.z; g[4 * c + 3] = a * dxv[4 * c + 3] + c1 * w4.w;
          }
        }
      }
    } else {
      take_bf16(h);
    }
    // h now holds the hidden whose gradient is being assembled (index L1 - 1); add what the later layers sent to it
    for (int j = 0; j < A.n_later; ++j) {
      float d[NCH * 4];
      take_f32(d);
      const float a = __shfl_sync(0xffffffffu, scl.x, j), c1 = __shfl_sync(0xffffffffu, scl.y, j);
      c2sum += __shfl_sync(0xffffffffu, scl.z, j);
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const float4 w4 = *reinterpret_cast<const float4*>(w_s + (j + 1) * D + c * 128 + lane * 4);
        g[4 * c] += a * d[4 * c] + c1 * w4.x; g[4 * c + 1] += a * d[4 * c + 1] + c1 * w4.y;
        g[4 * c + 2] += a * d[4 * c + 2] + c1 * w4.z; g[4 * c + 3] += a * d[4 * c + 3] + c1 * w4.w;
      }
    }
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) g[i] -= c2sum * h[i];
    if (ACC) {                                      // a further chunk of later layers: add to what the earlier launches stored
      load_row_f32<NCH>(G + (long long)row * D, lane, h);
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) g[i] += h[i];
    }
    store_row_f32<NCH>(G + (long long)row * D, lane, g);
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  if (A.own) {
    // d w = sum over tokens of c1 * h: block-level reduction, then ONE row of partial sums per block (folded by attn_res_bwd_finish_k)
    __syncthreads();
    float* red = w_s;                               // [warps][D]: the caller sizes the w area for max(1 + n_later, warps) rows
    store_row_f32<NCH>(red + (threadIdx.x >> 5) * D, lane, accw);
    __syncthreads();
    for (int c = threadIdx.x; c < D; c += ROW_THREADS) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < WARPS_PER_BLOCK; ++w) t += red[w * D + c];
      partials[(long long)blockIdx.x * D + c] = t;
    }
  }
}

// dgamma[c] += pq[c] * sum_b partials[b][c];  dpq[c] += (gamma[c] + 1) * sum_b partials[b][c]
__global__ void attn_res_bwd_finish_k(const float* __restrict__ partials, int n_blocks, int D, const float* __restrict__ gamma, const float* __restrict__ pq,
                                      float* __restrict__ dgamma, float* __restrict__ dpq, int rows_per_block) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= D) return;
  const int b0 = blockIdx.y * rows_per_block, b1 = min(n_blocks, b0 + rows_per_block);
  float a = 0.f;
  for (int b = b0; b < b1; ++b) a += partials[(long long)b * D + c];
  atomicAdd(dgamma + c, a * pq[c]);
  atomicAdd(dpq + c, a * (gamma[c] + 1.f));
}

// ------------------------------------------------------------------------------------ final RMSNorm
// out = x / max(|x|,eps) * sqrt(D) * (gamma+1)      (T.py:779-786, 1250); optional compaction of modality rows
template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) rmsnorm_fwd_k(const float* __restrict__ x, const float* __restrict__ gamma, float* __restrict__ of,
                                                            __nv_bfloat16* __restrict__ ob, const int* __restrict__ slot, __nv_bfloat16* __restrict__ omod, int M) {
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  float gv[NCH * 4];
  load_row_f32<NCH>(gamma, lane, gv);
  const float c = sqrtf((float)D);
  for (int row = warp0; row < M; row += nwarps) {
    float v[NCH * 4];
    load_row_f32<NCH>(x + (long long)row * D, lane, v);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) ss += v[i] * v[i];
    const float r = c / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) v[i] = v[i] * r * (gv[i] + 1.f);
    if (of) store_row_f32<NCH>(of + (long long)row * D, lane, v);
    if (ob) store_row_bf16<NCH>(ob + (long long)row * D, lane, v);
    if (slot && omod) { const int s = slot[row]; if (s >= 0) store_row_bf16<NCH>(omod + (long long)s * D, lane, v); }
  }
}

template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) rmsnorm_bwd_k(const float* __restrict__ dout, const float* __restrict__ x, const float* __restrict__ gamma,
                                                            float* __restrict__ dx, float* __restrict__ dgamma, int M, int tpw) {
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int r0 = warp * tpw, r1 = min(M, r0 + tpw);
  if (r0 >= M) return;
  if constexpr (NCH > 8) {
    // wide: passes for |x|, for <d xhat, xhat> and for the apply; d gamma accumulates in a per-warp shared-memory row (dynamic, 64 KB at 2048)
    constexpr int W = WIDE_GROUP;
    extern __shared__ __align__(16) float rms_acc[];
    float* acc = rms_acc + (threadIdx.x >> 5) * D;
    float t[W * 4];
#pragma unroll
    for (int i = 0; i < W * 4; ++i) t[i] = 0.f;
#pragma unroll 1
    for (int c0 = 0; c0 < NCH; c0 += W) store_row_f32<W>(acc + c0 * 128, lane, t);
    const float c = sqrtf((float)D);
    for (int row = r0; row < r1; ++row) {
      const float* xr = x + (long long)row * D;
      const float* dr = dout + (long long)row * D;
      float ss = 0.f, dot = 0.f;
#pragma unroll 1
      for (int c0 = 0; c0 < NCH; c0 += W) {
        load_row_f32<W>(xr + c0 * 128, lane, t);
#pragma unroll
        for (int i = 0; i < W * 4; ++i) ss += t[i] * t[i];
      }
      const float nrm = sqrtf(warp_sum(ss));
      const float rn = 1.f / fmaxf(nrm, 1e-12f);
#pragma unroll 1
      for (int c0 = 0; c0 < NCH; c0 += W) {
        float d[W * 4], gv[W * 4];
        load_row_f32<W>(xr + c0 * 128, lane, t);
        load_row_f32<W>(dr + c0 * 128, lane, d);
        load_row_f32<W>(gamma + c0 * 128, lane, gv);
#pragma unroll
        for (int i = 0; i < W * 4; ++i) dot += d[i] * (c * (gv[i] + 1.f)) * (t[i] * rn);
      }
      dot = warp_sum(dot);
      if (nrm < 1e-12f) dot = 0.f;
#pragma unroll 1
      for (int c0 = 0; c0 < NCH; c0 += W) {
        float d[W * 4], gv[W * 4], a[W * 4];
        load_row_f32<W>(xr + c0 * 128, lane, t);
        load_row_f32<W>(dr + c0 * 128, lane, d);
        load_row_f32<W>(gamma + c0 * 128, lane, gv);
        load_row_f32<W>(acc + c0 * 128, lane, a);
#pragma unroll
        for (int i = 0; i < W * 4; ++i) {
          t[i] *= rn;
          a[i] += d[i] * t[i] * c;
          d[i] = rn * (d[i] * (c * (gv[i] + 1.f)) - t[i] * dot);
        }
        store_row_f32<W>(acc + c0 * 128, lane, a);
        store_row_f32<W>(dx + (long long)row * D + c0 * 128, lane, d);
      }
    }
#pragma unroll 1
    for (int c0 = 0; c0 < NCH; c0 += W) {
      load_row_f32<W>(acc + c0 * 128, lane, t);
      red_row_f32<W>(dgamma + c0 * 128, lane, t);
    }
    return;
  }
  float gv[NCH * 4], acc[NCH * 4];
  load_row_f32<NCH>(gamma, lane, gv);
#pragma unroll
  for (int i = 0; i < NCH * 4; ++i) acc[i] = 0.f;
  const float c = sqrtf((float)D);
  for (int row = r0; row < r1; ++row) {
    float v[NCH * 4], d[NCH * 4];
    load_row_f32<NCH>(x + (long long)row * D, lane, v);
    load_row_f32<NCH>(dout + (long long)row * D, lane, d);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) ss += v[i] * v[i];
    const float nrm = sqrtf(warp_sum(ss));
    const float rn = 1.f / fmaxf(nrm, 1e-12f);
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) {
      v[i] *= rn;                              // xhat
      acc[i] += d[i] * v[i] * c;
      d[i] *= c * (gv[i] + 1.f);               // d xhat
      dot += d[i] * v[i];
    }
    dot = warp_sum(dot);
    if (nrm < 1e-12f) dot = 0.f;               // clamped norm: a constant for the gradient (F.normalize), dx = d xhat / eps
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) d[i] = rn * (d[i] - v[i] * dot);
    store_row_f32<NCH>(dx + (long long)row * D, lane, d);
  }
  red_row_f32<NCH>(dgamma, lane, acc);
}

// ------------------------------------------------------------------------------------ Self-Flow representation loss
// loss = 1 - mean_r cos(a_r, b_r) (T.py:3458-3460) with the eps of torch.nn.functional.cosine_similarity: each norm is clamped to 1e-8 on its own,
// and the clamp is a constant for the gradient.  One pass reads a and b once and writes
//   da_r = -(g / n) (b_r / (na nb) - cos_r a_r / (na |a_r|)),   na = max(|a_r|, eps), nb = max(|b_r|, eps)   (second term 0 for a zero row),
// g a device scalar.  The cosine sum is deterministic: per-block partials in fixed row order, summed in block order by the last block.
template <int NCH, bool BB16>
__global__ void __launch_bounds__(ROW_THREADS) rep_cos_fwd_bwd_k(const float* __restrict__ a, const void* __restrict__ b, const float* __restrict__ g, int n_mean,
                                                                __nv_bfloat16* __restrict__ da, double* __restrict__ partials, unsigned int* __restrict__ ticket,
                                                                float* __restrict__ loss, int M) {
  constexpr int D = NCH * 128;
  __shared__ double red[WARPS_PER_BLOCK];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const float gs = -__ldg(g) / (float)n_mean;
  double local = 0.0;
  for (int row = warp0; row < M; row += nwarps) {
    float x[NCH * 4], y[NCH * 4];
    load_row_f32<NCH>(a + (long long)row * D, lane, x);
    if constexpr (BB16) load_row_bf16<NCH>(reinterpret_cast<const __nv_bfloat16*>(b) + (long long)row * D, lane, y);
    else load_row_f32<NCH>(reinterpret_cast<const float*>(b) + (long long)row * D, lane, y);
    float saa = 0.f, sbb = 0.f, sab = 0.f;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) { saa += x[i] * x[i]; sbb += y[i] * y[i]; sab += x[i] * y[i]; }
    const float la = sqrtf(warp_sum(saa)), lb = sqrtf(warp_sum(sbb));
    const float na = fmaxf(la, 1e-8f), nb = fmaxf(lb, 1e-8f);
    const float cs = warp_sum(sab) / (na * nb);
    const float cb = gs / (na * nb), ca = la > 0.f ? -gs * cs / (na * la) : 0.f;
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) x[i] = cb * y[i] + ca * x[i];
    store_row_bf16<NCH>(da + (long long)row * D, lane, x);
    local += (double)cs;
  }
  if (lane == 0) red[wib] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < WARPS_PER_BLOCK; ++w) s += red[w];
    partials[blockIdx.x] = s;
    __threadfence();
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
      __threadfence();
      double t = 0.0;
      for (int k = 0; k < (int)gridDim.x; ++k) t += reinterpret_cast<volatile double*>(partials)[k];
      *loss = (float)(1.0 - t / (double)n_mean);
      *ticket = 0u;                                // ready for the next launch
    }
  }
}

// ------------------------------------------------------------------------------------ token assemble (+ backward)
// x0 = isM ? modality_token[slot] : text_embed[max(id,0)]         (T.py:3173-3184)
template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) embed_assemble_k(const int* __restrict__ text_id, const float* __restrict__ emb, const float* __restrict__ modtok,
                                                               const int* __restrict__ slot, float* __restrict__ x0, __nv_bfloat16* __restrict__ x0b, int M) {
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp0; row < M; row += nwarps) {
    const int s = slot ? slot[row] : -1;
    float v[NCH * 4];
    if (s >= 0) load_row_f32<NCH>(modtok + (long long)s * D, lane, v);
    else { int id = text_id[row]; if (id < 0) id = 0; load_row_f32<NCH>(emb + (long long)id * D, lane, v); }
    store_row_f32<NCH>(x0 + (long long)row * D, lane, v);
    if (x0b) store_row_bf16<NCH>(x0b + (long long)row * D, lane, v);
  }
}
template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) embed_bwd_k(const float* __restrict__ dx0, const int* __restrict__ text_id, const int* __restrict__ slot,
                                                          float* __restrict__ demb, __nv_bfloat16* __restrict__ dmodtok, int M) {
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int row = warp0; row < M; row += nwarps) {
    const int s = slot ? slot[row] : -1;
    float v[NCH * 4];
    load_row_f32<NCH>(dx0 + (long long)row * D, lane, v);
    if (s >= 0) { if (dmodtok) store_row_bf16<NCH>(dmodtok + (long long)s * D, lane, v); }
    else { int id = text_id[row]; if (id < 0) id = 0; red_row_f32<NCH>(demb + (long long)id * D, lane, v); }
  }
}

// dst[row_map[s]] += src[s]   (modality rows of d(final-norm output) receive the flow-head gradient)
template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) scatter_add_rows_k(float* __restrict__ dst, const float* __restrict__ src, const int* __restrict__ row_map, int S) {
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int s = warp0; s < S; s += nwarps) {
    const int r = row_map[s];
    if (r < 0) continue;
    float a[NCH * 4], b[NCH * 4];
    load_row_f32<NCH>(src + (long long)s * D, lane, a);
    load_row_f32<NCH>(dst + (long long)r * D, lane, b);
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) b[i] += a[i];
    store_row_f32<NCH>(dst + (long long)r * D, lane, b);
  }
}

// model_output_clean (MP.py:100-126, 790-793; T.py:2454-2455): the transformer predicts the clean modality in MODEL space, the flow is
//   (embed - noised_model_tokens) / max(1 - t, eps)   before model_to_latent.  Compact modality rows: omod[s] = (out[row_token[s]] - modtok[s]) * inv(t).
// t of a row = cond_times[cond_row[token]] (device-resident: the ODE loop rewrites cond_times in place).
template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) clean_flow_fwd_k(const float* __restrict__ out, const int* __restrict__ row_token, const float* __restrict__ modtok,
                                                               const float* __restrict__ cond_times, const int* __restrict__ cond_row, float eps, __nv_bfloat16* __restrict__ omod, int S) {
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int s = warp0; s < S; s += nwarps) {
    const int r = row_token[s];
    float a[NCH * 4], b[NCH * 4];
    if (r < 0) {
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) a[i] = 0.f;
    } else {
      const float inv = 1.f / fmaxf(1.f - cond_times[cond_row[r]], eps);
      load_row_f32<NCH>(out + (long long)r * D, lane, a);
      load_row_f32<NCH>(modtok + (long long)s * D, lane, b);
#pragma unroll
      for (int i = 0; i < NCH * 4; ++i) a[i] = (a[i] - b[i]) * inv;
    }
    store_row_bf16<NCH>(omod + (long long)s * D, lane, a);
  }
}
// backward: d(out rows) = dmod * inv (in place, scattered by the caller), d(modtok) = -dmod * inv
template <int NCH>
__global__ void __launch_bounds__(ROW_THREADS) clean_flow_bwd_k(float* __restrict__ dmod, float* __restrict__ dneg, const int* __restrict__ row_token, const float* __restrict__ cond_times,
                                                               const int* __restrict__ cond_row, float eps, int S) {
  constexpr int D = NCH * 128;
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int s = warp0; s < S; s += nwarps) {
    const int r = row_token[s];
    float a[NCH * 4], b[NCH * 4];
    const float inv = r < 0 ? 0.f : 1.f / fmaxf(1.f - cond_times[cond_row[r]], eps);
    load_row_f32<NCH>(dmod + (long long)s * D, lane, a);
#pragma unroll
    for (int i = 0; i < NCH * 4; ++i) { a[i] *= inv; b[i] = -a[i]; }
    store_row_f32<NCH>(dmod + (long long)s * D, lane, a);
    store_row_f32<NCH>(dneg + (long long)s * D, lane, b);
  }
}

// ------------------------------------------------------------------------------------ qk RMSNorm + RoPE backward, packs d[q|k|.|gates]
// NORM (qk_rmsnorm = True), forward in the GEMM epilogue: xhat = x*inv;  y = xhat*sqrt(DH)*(gamma+1);  q = R(pos) y (interleaved pairs)
// (T.py:950-965).  !NORM (EPI_QKVG_ROPE): q = R(pos) x, so d x = R(pos)^T d q per interleaved pair; no saved values and no gammas are needed.
// One warp per token; DH / 8 lanes share a head (8 at DH = 64, 16 at 128) and a lane owns 8 consecutive dims = 4 rope pairs (32 B fp32 /
// 16 B bf16 accesses), so a warp covers 32 / (DH / 8) heads per pass and the per-head dot product is a log2(DH / 8)-step shuffle.
// rope_cs is [pos][DH / 2] (cos, sin).  Without NORM, q, k, qk_inv, the gammas and their gradients are not read and may be null.  Without
// gates (`gate_values = False`) neither is dsum, and no gate column is written.
// xhat is rebuilt from the bf16 output as R^T q / (sqrt(DH) (gamma + 1)): where gamma_j = -1 the forward wrote y_j = 0 and xhat_j is lost, so
// dx_j and dgamma_j come out 0 instead of -inv xhat_j (xhat . dxhat) and sum sqrt(DH) dy_j xhat_j; near -1 the bf16 error of the rope partner
// is amplified by |gamma_partner + 1| / |gamma_j + 1|.
template <int DH, bool NORM>
__global__ void __launch_bounds__(ROW_THREADS) qk_bwd_pack_k(const float* __restrict__ dq, const float* __restrict__ dk, const __nv_bfloat16* __restrict__ q,
                                                            const __nv_bfloat16* __restrict__ k, const float* __restrict__ qk_inv, const float* __restrict__ gq,
                                                            const float* __restrict__ gk, const int* __restrict__ rope_pos, const float2* __restrict__ rope_cs,
                                                            const float* __restrict__ gates, const float* __restrict__ dsum, __nv_bfloat16* __restrict__ out,
                                                            long long out_ld, float* __restrict__ dgq, float* __restrict__ dgk, int M, int H, int tpw) {
  constexpr int LPH = DH / 8, HPP = 32 / LPH;
  static_assert(2 * DH <= ROW_THREADS, "one thread per gamma column in the block reduction");
  const float RS = sqrtf((float)DH);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int sub = lane % LPH, hq = lane / LPH;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int r0 = min(M, warp * tpw), r1 = min(M, r0 + tpw);
  const int HI = H * DH;
  // NORM only: the gamma-gradient sums, gamma + 1 and 1 / (sqrt(DH) (gamma + 1)) of the lane's 8 columns, for q and k
  float acc[2][8];
  float g1[2][8], rg[2][8];
  if constexpr (NORM) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc[0][j] = acc[1][j] = 0.f;
      g1[0][j] = gq[sub * 8 + j] + 1.f; g1[1][j] = gk[sub * 8 + j] + 1.f;
      rg[0][j] = fabsf(g1[0][j]) > 1e-12f ? 1.f / (RS * g1[0][j]) : 0.f;
      rg[1][j] = fabsf(g1[1][j]) > 1e-12f ? 1.f / (RS * g1[1][j]) : 0.f;
    }
  }
  for (int row = r0; row < r1; ++row) {
    float cs[8];   // (cos, sin) of the lane's 4 rope pairs
    {
      const float4* cp = reinterpret_cast<const float4*>(rope_cs + (long long)rope_pos[row] * (DH / 2) + sub * 4);
      const float4 c0 = cp[0], c1 = cp[1];
      cs[0] = c0.x; cs[1] = c0.y; cs[2] = c0.z; cs[3] = c0.w; cs[4] = c1.x; cs[5] = c1.y; cs[6] = c1.z; cs[7] = c1.w;
    }
    for (int h0 = 0; h0 < H; h0 += HPP) {
      const int h = h0 + hq;
      // NORM: lanes past H join the shuffle on head 0's data and store nothing.  !NORM has no shuffle, so those lanes skip the head.
      if constexpr (!NORM) { if (h >= H) continue; }
      const bool act = !NORM || h < H;
      const long long off = (long long)row * HI + (act ? h : 0) * DH + sub * 8;
      // all loads of this head group (q and k, gradient and value) are issued before any arithmetic
      const float4 da[2] = {*reinterpret_cast<const float4*>(dq + off), *reinterpret_cast<const float4*>(dk + off)};
      const float4 db[2] = {*reinterpret_cast<const float4*>(dq + off + 4), *reinterpret_cast<const float4*>(dk + off + 4)};
      uint4 tv[2];
      float invs[2];
      if constexpr (NORM) {
        tv[0] = *reinterpret_cast<const uint4*>(q + off); tv[1] = *reinterpret_cast<const uint4*>(k + off);
        invs[0] = act ? qk_inv[(long long)row * 2 * H + h] : 0.f; invs[1] = act ? qk_inv[(long long)row * 2 * H + H + h] : 0.f;
      }
#pragma unroll
      for (int which = 0; which < 2; ++which) {
        const float dr[8] = {da[which].x, da[which].y, da[which].z, da[which].w, db[which].x, db[which].y, db[which].z, db[which].w};
        uint32_t w[4];
        if constexpr (NORM) {
          const float2 p0 = unpack2_bf16(tv[which].x), p1 = unpack2_bf16(tv[which].y), p2 = unpack2_bf16(tv[which].z), p3 = unpack2_bf16(tv[which].w);
          const float r[8] = {p0.x, p0.y, p1.x, p1.y, p2.x, p2.y, p3.x, p3.y};
          const float inv = invs[which];
          float xh[8], dxh[8], dot = 0.f;
#pragma unroll
          for (int pr = 0; pr < 4; ++pr) {
            const float c = cs[2 * pr], sn = cs[2 * pr + 1];
            // un-rotate (R^T)
            const float y0 = r[2 * pr] * c + r[2 * pr + 1] * sn, y1 = r[2 * pr + 1] * c - r[2 * pr] * sn;
            const float dy0 = dr[2 * pr] * c + dr[2 * pr + 1] * sn, dy1 = dr[2 * pr + 1] * c - dr[2 * pr] * sn;
            xh[2 * pr] = y0 * rg[which][2 * pr]; xh[2 * pr + 1] = y1 * rg[which][2 * pr + 1];
            dxh[2 * pr] = dy0 * RS * g1[which][2 * pr]; dxh[2 * pr + 1] = dy1 * RS * g1[which][2 * pr + 1];
            if (act) { acc[which][2 * pr] += dy0 * xh[2 * pr] * RS; acc[which][2 * pr + 1] += dy1 * xh[2 * pr + 1] * RS; }
            dot += xh[2 * pr] * dxh[2 * pr] + xh[2 * pr + 1] * dxh[2 * pr + 1];
          }
#pragma unroll
          for (int o = 1; o < LPH; o <<= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
          if (act) {
#pragma unroll
            for (int pr = 0; pr < 4; ++pr) w[pr] = pack2_bf16(inv * (dxh[2 * pr] - xh[2 * pr] * dot), inv * (dxh[2 * pr + 1] - xh[2 * pr + 1] * dot));
          }
        } else {
#pragma unroll
          for (int pr = 0; pr < 4; ++pr) {
            const float c = cs[2 * pr], sn = cs[2 * pr + 1];
            w[pr] = pack2_bf16(dr[2 * pr] * c + dr[2 * pr + 1] * sn, dr[2 * pr + 1] * c - dr[2 * pr] * sn);     // un-rotate (R^T)
          }
        }
        if (act) *reinterpret_cast<uint4*>(out + (long long)row * out_ld + which * HI + h * DH + sub * 8) = make_uint4(w[0], w[1], w[2], w[3]);
      }
    }
    // gate logits: d g = (1 - sigmoid(g)) * sum_d dO_gated * O_gated; an ungated model (gates null) has no gate column
    if (gates && lane < H) {
      const float gl = gates[(long long)row * H + lane];
      const float sg = 1.f / (1.f + __expf(-gl));
      out[(long long)row * out_ld + 3 * HI + lane] = __float2bfloat16((1.f - sg) * dsum[(long long)row * H + lane]);
    }
  }
  if constexpr (NORM) {
    // gamma gradients: reduce the head groups of the warp, then the 8 warps of the block, then one atomic per column per block
    __shared__ float red[WARPS_PER_BLOCK][2 * DH];
#pragma unroll
    for (int which = 0; which < 2; ++which)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float v = acc[which][j];
#pragma unroll
        for (int o = LPH; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (hq == 0) red[wib][which * DH + sub * 8 + j] = v;
      }
    __syncthreads();
    if (threadIdx.x < 2 * DH) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < WARPS_PER_BLOCK; ++w) t += red[w][threadIdx.x];
      atomicAdd((threadIdx.x < DH ? dgq : dgk) + (threadIdx.x % DH), t);
    }
  }
}

// rows per warp such that the grid is (just under) one full wave of `blocks_per_sm` resident blocks on every SM
static inline int balanced_tpw(int M, int sms, int blocks_per_sm, int min_tpw) {
  const long long warps = (long long)sms * blocks_per_sm * WARPS_PER_BLOCK;
  const int tpw = (int)((M + warps - 1) / warps);
  return tpw < min_tpw ? min_tpw : tpw;
}
static inline int chunk_grid(int M, int tpw) {
  long long warps = ((long long)M + tpw - 1) / tpw;
  return (int)((warps + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK);
}
int num_sms();

}  // namespace tfx

using namespace tfx;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

// tfx_qk_bwd_pack(_rope)(_d128); `name` is the entry point's name for error messages.  Without NORM the norm pointers are null.
template <int DH, bool NORM>
static int qk_bwd_pack(const char* name, const float* dq, const float* dk, const void* q_bf16, const void* k_bf16, const float* qk_inv, const float* q_gamma,
                       const float* k_gamma, const int* rope_pos, const float* rope_cs, const float* gates, const float* dsum, void* dqkvg_bf16, long long out_ld,
                       float* dq_gamma, float* dk_gamma, int M, int H, void* stream) {
  if (M <= 0) return 0;
  constexpr int max_heads = 2048 / DH;     // inner width up to 2048; at 64 also one gate column per lane
  TFX_REQUIRE(H >= 1 && H <= max_heads, "%s: heads %d out of range [1, %d]", name, H, max_heads);
  const int tpw = 8;
  qk_bwd_pack_k<DH, NORM><<<chunk_grid(M, tpw), ROW_THREADS, 0, ST(stream)>>>(dq, dk, (const __nv_bfloat16*)q_bf16, (const __nv_bfloat16*)k_bf16, qk_inv, q_gamma,
                                                                            k_gamma, rope_pos, (const float2*)rope_cs, gates, dsum, (__nv_bfloat16*)dqkvg_bf16, out_ld,
                                                                            dq_gamma, dk_gamma, M, H, tpw);
  return check_launch(name);
}

extern "C" {

int tfx_adaln_fwd(const float* x, const int* cond_row, const float* film, long long film_ld, const float* ln_gamma,
                  void* u_bf16, float* stats, int M, int D, void* stream) {
  if (M <= 0) return 0;
  TFX_DISPATCH_NCH(D, {
    auto kern = adaln_fwd_k<NCH>;
    const int smem = WARPS_PER_BLOCK * ADALN_FWD_RING<NCH> * D * 4;
    static int per_sm = 0;                            // persistent grid = the resident blocks (ring shared memory / registers decide)
    if (!per_sm) {
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, ROW_THREADS, smem);
      if (per_sm < 1) per_sm = 1;
    }
    const long long want = ((long long)M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, cap = (long long)num_sms() * per_sm;
    kern<<<(int)(want < cap ? want : cap), ROW_THREADS, smem, ST(stream)>>>(x, cond_row, film, film_ld, ln_gamma, (__nv_bfloat16*)u_bf16, stats, M);
  });
  return check_launch("adaln_fwd");
}

int tfx_adaln_bwd(const float* du, const float* x, const float* stats, const int* cond_row, const float* film, long long film_ld,
                  const float* ln_gamma, float* dx_accum, float* dfilm, long long dfilm_ld, float* dln_gamma, int M, int D, void* stream) {
  if (M <= 0) return 0;
  TFX_DISPATCH_NCH(D, {
    // wide rows keep their accumulators in dynamic shared memory (3 rows per warp): one resident block per SM
    const int smem = NCH > 8 ? WARPS_PER_BLOCK * 3 * D * 4 : 0;
    if (NCH > 8) {
      static bool attr_set = false;
      if (!attr_set) { cudaFuncSetAttribute(adaln_bwd_k<NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); attr_set = true; }
    }
    const int tpw = balanced_tpw(M, num_sms(), NCH > 8 ? 1 : 2, 4);
    adaln_bwd_k<NCH><<<chunk_grid(M, tpw), ROW_THREADS, smem, ST(stream)>>>(du, x, stats, cond_row, film, film_ld, ln_gamma, dx_accum, dfilm, dfilm_ld, dln_gamma, M, tpw);
  });
  return check_launch("adaln_bwd");
}

int tfx_resid_bwd(const float* dx, const void* y_bf16, const int* cond_row, const float* zgate, long long zgate_ld, const float* layerscale,
                  void* dy_bf16, float* dzgate, long long dzgate_ld, float* dlayerscale, float* dbias, int M, int D, void* stream) {
  if (M <= 0) return 0;
  const int tpw = balanced_tpw(M, num_sms(), 2, 4);
  const size_t smem = (dbias || layerscale) ? (size_t)WARPS_PER_BLOCK * (D > 1024 ? WIDE_GROUP * 128 : D) * sizeof(float) : 0;   // one column group
  TFX_DISPATCH_NCH(D, (resid_bwd_k<NCH><<<chunk_grid(M, tpw), ROW_THREADS, smem, ST(stream)>>>(dx, (const __nv_bfloat16*)y_bf16, cond_row, zgate, zgate_ld, layerscale,
                                                                                                 (__nv_bfloat16*)dy_bf16, dzgate, dzgate_ld, dlayerscale, dbias, M, tpw)));
  return check_launch("resid_bwd");
}

int tfx_attn_residual_fwd_h16(const void* const* hiddens_bf16, int n_hiddens, const float* gamma, const float* pseudo_query,
                              float* x_out, void* x_out_bf16, float* lse_out, int M, int D, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(n_hiddens >= 1 && n_hiddens <= MAX_HIDDENS, "attn_residual: n_hiddens %d out of range [1,%d]", n_hiddens, MAX_HIDDENS);
  HiddenList hl;
  for (int i = 0; i < n_hiddens; ++i) hl.p[i] = reinterpret_cast<const __nv_bfloat16*>(hiddens_bf16[i]);
  // persistent grid: exactly the resident blocks (registers / ring shared memory decide), rows strided over all warps
  TFX_DISPATCH_NCH(D, {
    auto kern = attn_res_fwd_k<NCH>;
    const int smem = WARPS_PER_BLOCK * ARES_FWD_RING * D * 2;
    static int per_sm = 0;
    if (!per_sm) {
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, ROW_THREADS, smem);
      if (per_sm < 1) per_sm = 1;
    }
    const long long want = ((long long)M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, cap = (long long)num_sms() * per_sm;
    kern<<<(int)(want < cap ? want : cap), ROW_THREADS, smem, ST(stream)>>>(hl, n_hiddens, gamma, pseudo_query, x_out, (__nv_bfloat16*)x_out_bf16, lse_out, M);
  });
  return check_launch("attn_residual_fwd");
}

static const int ATTN_RES_BWD2_TPW = 8;      // the ring start-up bubble is paid once per warp: more rows per warp
long long tfx_attn_residual_bwd_workspace_floats(int M, int D) { return (long long)chunk_grid(M, ATTN_RES_BWD2_TPW) * D; }

int tfx_attn_residual_bwd2(const void* const* hiddens_bf16, int n_hiddens, int own, const float* const* gammas, const float* const* pseudo_queries,
                           const float* const* dx_later, const float* const* scalars_later, int n_later, const float* dx_out, const float* x_out, const float* lse,
                           float* grad_hidden, float* scalars_out, int scalar_stride, float* dgamma, float* dpseudo_query, float* workspace, int M, int D, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(n_hiddens >= 1 && n_hiddens <= MAX_HIDDENS && n_later >= 0 && n_later <= TFX_MAX_DEPTH, "attn_residual_bwd2: %d hiddens / %d later layers out of range [1,%d] / [0,%d]",
              n_hiddens, n_later, MAX_HIDDENS, TFX_MAX_DEPTH);
  TFX_REQUIRE(!own || workspace != nullptr, "attn_residual_bwd2: workspace of tfx_attn_residual_bwd_workspace_floats(M, D) floats is required");
  const int tpw = ATTN_RES_BWD2_TPW;
  const int blocks = chunk_grid(M, tpw);
  // launch c covers later layers [j0, j0 + n): c = 0 is the full kernel (own term, scalars, parameter gradients when own = 1) and stores G; every
  // further chunk is an own = 0 assembly whose gammas / pseudo-queries start one slot early (slot 0 unused), so the kernel sees them as 1 .. n
  for (int j0 = 0; j0 == 0 || j0 < n_later; j0 += BWD2_CHUNK) {
    const int n = n_later - j0 < BWD2_CHUNK ? n_later - j0 : BWD2_CHUNK;
    const bool acc = j0 > 0;
    ResBwd2Args A;
    memset(&A, 0, sizeof(A));
    A.L1 = n_hiddens; A.n_later = n; A.own = (own && !acc) ? 1 : 0;
    for (int i = 0; i < n_hiddens; ++i) A.hid[i] = reinterpret_cast<const __nv_bfloat16*>(hiddens_bf16[i]);
    for (int j = 0; j <= n; ++j) { A.gam[j] = gammas[j0 + j]; A.pq[j] = pseudo_queries[j0 + j]; }
    for (int j = 0; j < n; ++j) { A.dx_later[j] = dx_later[j0 + j]; A.sc_later[j] = scalars_later[j0 + j]; }
    TFX_DISPATCH_NCH(D, {
      // w rows (wide: the own layer's w and the accw rows), then the rings
      const int slots = NCH > 8 ? 1 + WARPS_PER_BLOCK : ((1 + n) > WARPS_PER_BLOCK ? (1 + n) : WARPS_PER_BLOCK);
      const size_t smem = (size_t)(slots + WARPS_PER_BLOCK * ResBwd2Cfg<NCH>::RING) * D * sizeof(float);
      const int smem_max = (int)(((NCH > 8 ? 1 + WARPS_PER_BLOCK : BWD2_CHUNK + 1) + WARPS_PER_BLOCK * ResBwd2Cfg<NCH>::RING) * D * sizeof(float));
      static bool attr_set = false;               // (one flag per NCH instantiation; the size above is the maximum any call can ask for)
      if (!attr_set) {
        cudaFuncSetAttribute(attn_res_bwd2_k<NCH, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
        cudaFuncSetAttribute(attn_res_bwd2_k<NCH, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
        attr_set = true;
      }
      if (acc) attn_res_bwd2_k<NCH, true><<<blocks, ROW_THREADS, smem, ST(stream)>>>(A, dx_out, x_out, lse, grad_hidden, scalars_out, scalar_stride, workspace, M, tpw);
      else attn_res_bwd2_k<NCH, false><<<blocks, ROW_THREADS, smem, ST(stream)>>>(A, dx_out, x_out, lse, grad_hidden, scalars_out, scalar_stride, workspace, M, tpw);
    });
    if (int rc = check_launch("attn_residual_bwd2")) return rc;
  }
  if (own) {
    const int rpb = 16;
    attn_res_bwd_finish_k<<<dim3((D + 127) / 128, (blocks + rpb - 1) / rpb), 128, 0, ST(stream)>>>(workspace, blocks, D, gammas[0], pseudo_queries[0], dgamma, dpseudo_query, rpb);
    return check_launch("attn_residual_bwd_finish");
  }
  return 0;
}

int tfx_rmsnorm_fwd(const float* x, const float* gamma, float* out_f32, void* out_bf16, const int* slot, void* out_mod_bf16, int M, int D, void* stream) {
  if (M <= 0) return 0;
  TFX_DISPATCH_NCH(D, (rmsnorm_fwd_k<NCH><<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>(x, gamma, out_f32, (__nv_bfloat16*)out_bf16, slot, (__nv_bfloat16*)out_mod_bf16, M)));
  return check_launch("rmsnorm_fwd");
}

int tfx_rmsnorm_bwd(const float* dout, const float* x, const float* gamma, float* dx, float* dgamma, int M, int D, void* stream) {
  if (M <= 0) return 0;
  const int tpw = 16;
  TFX_DISPATCH_NCH(D, {
    const int smem = NCH > 8 ? WARPS_PER_BLOCK * D * 4 : 0;      // wide rows: the d gamma accumulator rows
    if (NCH > 8) {
      static bool attr_set = false;
      if (!attr_set) { cudaFuncSetAttribute(rmsnorm_bwd_k<NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); attr_set = true; }
    }
    rmsnorm_bwd_k<NCH><<<chunk_grid(M, tpw), ROW_THREADS, smem, ST(stream)>>>(dout, x, gamma, dx, dgamma, M, tpw);
  });
  return check_launch("rmsnorm_bwd");
}

int tfx_rep_cos_blocks(int M) { return row_grid(M, num_sms()); }

int tfx_rep_cos_fwd_bwd(const float* a, const void* b, int b_bf16, const float* g, int n_mean, void* da_bf16, double* partials, unsigned int* ticket, float* loss,
                        int M, int D, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(n_mean > 0, "rep_cos_fwd_bwd: n_mean must be positive (got %d)", n_mean);
  const int blocks = row_grid(M, num_sms());
  if (b_bf16) TFX_DISPATCH_NCH(D, (rep_cos_fwd_bwd_k<NCH, true><<<blocks, ROW_THREADS, 0, ST(stream)>>>(a, b, g, n_mean, (__nv_bfloat16*)da_bf16, partials, ticket, loss, M)));
  else TFX_DISPATCH_NCH(D, (rep_cos_fwd_bwd_k<NCH, false><<<blocks, ROW_THREADS, 0, ST(stream)>>>(a, b, g, n_mean, (__nv_bfloat16*)da_bf16, partials, ticket, loss, M)));
  return check_launch("rep_cos_fwd_bwd");
}

int tfx_embed_assemble(const int* text_id, const float* emb, const float* modtok, const int* slot, float* x0, void* x0_bf16, int M, int D, void* stream) {
  if (M <= 0) return 0;
  TFX_DISPATCH_NCH(D, (embed_assemble_k<NCH><<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>(text_id, emb, modtok, slot, x0, (__nv_bfloat16*)x0_bf16, M)));
  return check_launch("embed_assemble");
}

int tfx_embed_bwd(const float* dx0, const int* text_id, const int* slot, float* demb, void* dmodtok_bf16, int M, int D, void* stream) {
  if (M <= 0) return 0;
  TFX_DISPATCH_NCH(D, (embed_bwd_k<NCH><<<row_grid(M, num_sms()), ROW_THREADS, 0, ST(stream)>>>(dx0, text_id, slot, demb, (__nv_bfloat16*)dmodtok_bf16, M)));
  return check_launch("embed_bwd");
}

int tfx_scatter_add_rows(float* dst, const float* src, const int* row_map, int S, int D, void* stream) {
  if (S <= 0) return 0;
  TFX_DISPATCH_NCH(D, (scatter_add_rows_k<NCH><<<row_grid(S, num_sms()), ROW_THREADS, 0, ST(stream)>>>(dst, src, row_map, S)));
  return check_launch("scatter_add_rows");
}

int tfx_clean_flow_fwd(const float* out, const int* row_token, const float* modtok, const float* cond_times, const int* cond_row, float eps, void* omod_bf16, int S, int D, void* stream) {
  if (S <= 0) return 0;
  TFX_DISPATCH_NCH(D, (clean_flow_fwd_k<NCH><<<row_grid(S, num_sms()), ROW_THREADS, 0, ST(stream)>>>(out, row_token, modtok, cond_times, cond_row, eps, (__nv_bfloat16*)omod_bf16, S)));
  return check_launch("clean_flow_fwd");
}

int tfx_clean_flow_bwd(float* dmod_inout, float* dmodtok_neg, const int* row_token, const float* cond_times, const int* cond_row, float eps, int S, int D, void* stream) {
  if (S <= 0) return 0;
  TFX_DISPATCH_NCH(D, (clean_flow_bwd_k<NCH><<<row_grid(S, num_sms()), ROW_THREADS, 0, ST(stream)>>>(dmod_inout, dmodtok_neg, row_token, cond_times, cond_row, eps, S)));
  return check_launch("clean_flow_bwd");
}

int tfx_qk_bwd_pack(const float* dq, const float* dk, const void* q_bf16, const void* k_bf16, const float* qk_inv, const float* q_gamma, const float* k_gamma,
                    const int* rope_pos, const float* rope_cs, const float* gates, const float* dsum, void* dqkvg_bf16, long long out_ld,
                    float* dq_gamma, float* dk_gamma, int M, int H, void* stream) {
  return qk_bwd_pack<64, true>("qk_bwd_pack", dq, dk, q_bf16, k_bf16, qk_inv, q_gamma, k_gamma, rope_pos, rope_cs, gates, dsum, dqkvg_bf16, out_ld,
                               dq_gamma, dk_gamma, M, H, stream);
}

int tfx_qk_bwd_pack_rope(const float* dq, const float* dk, const int* rope_pos, const float* rope_cs, const float* gates, const float* dsum_mh, void* dqkvg_bf16,
                         long long out_ld, int M, int H, void* stream) {
  return qk_bwd_pack<64, false>("qk_bwd_pack_rope", dq, dk, nullptr, nullptr, nullptr, nullptr, nullptr, rope_pos, rope_cs, gates, dsum_mh, dqkvg_bf16, out_ld,
                                nullptr, nullptr, M, H, stream);
}

int tfx_qk_bwd_pack_d128(const float* dq, const float* dk, const void* q_bf16, const void* k_bf16, const float* qk_inv, const float* q_gamma, const float* k_gamma,
                         const int* rope_pos, const float* rope_cs, const float* gates, const float* dsum, void* dqkvg_bf16, long long out_ld,
                         float* dq_gamma, float* dk_gamma, int M, int H, void* stream) {
  return qk_bwd_pack<128, true>("qk_bwd_pack_d128", dq, dk, q_bf16, k_bf16, qk_inv, q_gamma, k_gamma, rope_pos, rope_cs, gates, dsum, dqkvg_bf16, out_ld,
                                dq_gamma, dk_gamma, M, H, stream);
}

int tfx_qk_bwd_pack_rope_d128(const float* dq, const float* dk, const int* rope_pos, const float* rope_cs, const float* gates, const float* dsum_mh, void* dqkvg_bf16,
                              long long out_ld, int M, int H, void* stream) {
  return qk_bwd_pack<128, false>("qk_bwd_pack_rope_d128", dq, dk, nullptr, nullptr, nullptr, nullptr, nullptr, rope_pos, rope_cs, gates, dsum_mh, dqkvg_bf16,
                                 out_ld, nullptr, nullptr, M, H, stream);
}

}  // extern "C"
