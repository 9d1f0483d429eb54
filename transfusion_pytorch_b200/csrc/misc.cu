// Elementwise / reduction kernels around the block stack: flow-match noise inject, time features,
// GEGLU backward, fused text cross-entropy (fwd+bwd), fused flow MSE (fwd+bwd), column sums (bias
// grads), fp32 -> bf16 weight packing, small table ops for the conditioning path, fused Adam.
// Reference math: modality_processing.py:645-656 (noise), transfusion.py:617-635 (fourier), 831-834
// (GEGLU), 3320-3376 (loss heads).
#include "common.cuh"
#include "dropout.cuh"
#include "../../include/tfx_b200.h"
#include <math.h>

namespace tfx {

int num_sms();

// Phi(g), phi(g) of the exact-erf GELU from one exponential (Abramowitz-Stegun 7.1.26, |err| <= 1.5e-7); same routine as the
// forward GEGLU epilogue (gemm_sm90.cuh).
__device__ __forceinline__ void gelu_parts(float g, float& cdf, float& pdf) {
  const float ax = fabsf(g) * 0.70710678118654752f;
  const float t = __fdividef(1.f, fmaf(0.3275911f, ax, 1.f));
  const float E = __expf(-ax * ax);
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float h = 0.5f * poly * t * E;
  cdf = g >= 0.f ? 1.f - h : h;
  pdf = 0.3989422804014327f * E;
}

static inline int ew_grid(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  long long cap = (long long)num_sms() * 16;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

// noised = x*t + eps*(1-t) (bf16, GEMM operand) ; flow = x - eps (fp32 target)
__global__ void flow_noise_k(const float* __restrict__ x, const float* __restrict__ eps, const float* __restrict__ t_row, __nv_bfloat16* __restrict__ noised,
                             long long ld_noised, float* __restrict__ noised_f32, float* __restrict__ flow, long long S, int dl) {
  const long long n = S * dl;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / dl; const int c = (int)(i - r * dl);
    const float xv = x[i];
    if (eps) {
      const float e = eps[i], t = t_row[r];
      const float nz = xv * t + e * (1.f - t);
      noised[r * ld_noised + c] = __float2bfloat16(nz);
      if (noised_f32) noised_f32[i] = nz;
      if (flow) flow[i] = xv - e;
    } else {
      noised[r * ld_noised + c] = __float2bfloat16(xv);
    }
  }
}

// feats[r] = [t, sin(2 pi t w_j), cos(2 pi t w_j)], zero padded to ld   (T.py:633-634)
__global__ void time_features_k(const float* __restrict__ times, const float* __restrict__ w, __nv_bfloat16* __restrict__ feats, int n, int half, int ld) {
  const int total = n * ld;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int r = i / ld, c = i - r * ld;
    const float t = times[r];
    float v = 0.f;
    if (c == 0) v = t;
    else if (c <= half) v = sinf(t * w[c - 1] * 2.f * 3.14159265358979323846f);
    else if (c <= 2 * half) v = cosf(t * w[c - 1 - half] * 2.f * 3.14159265358979323846f);
    feats[i] = __float2bfloat16(v);
  }
}

// table ops: op 0 sigmoid, 1 silu, 2 dsigmoid (out = g * s * (1-s), s = in2), 3 dsilu (out = g * silu'(in2))
__global__ void table_op_k(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ of, __nv_bfloat16* __restrict__ ob, long long rows, int cols,
                           long long ld_a, long long ld_b, long long ld_of, long long ld_ob, int op) {
  const long long n = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols; const int c = (int)(i - r * cols);
    const float x = a[r * ld_a + c];
    float y;
    if (op == 0) y = 1.f / (1.f + expf(-x));
    else if (op == 1) y = x / (1.f + expf(-x));
    else if (op == 2) { const float s = b[r * ld_b + c]; y = x * s * (1.f - s); }
    else if (op == 3) { const float z = b[r * ld_b + c]; const float s = 1.f / (1.f + expf(-z)); y = x * (s * (1.f + z * (1.f - s))); }
    else y = x;
    if (of) of[r * ld_of + c] = y;
    if (ob) ob[r * ld_ob + c] = __float2bfloat16(y);
  }
}

// GEGLU backward on the tile-interleaved layout ([64 value | 64 gate] per 128 columns), fused with the column sums of
// d(vg) (= gradient of the FFN-in bias).  A thread owns one 8-column chunk of h (and the matching value / gate chunks)
// and walks `rpb` rows; its 16 column sums stay in registers and are flushed with one atomicAdd each per block.
// DROP: h was dropped in the forward (site FFN), so dh is first multiplied by the regenerated mask and 1 / (1 - p).
template <bool DROP>
__device__ __forceinline__ void geglu_bwd_body(const __nv_bfloat16* __restrict__ dh, const __nv_bfloat16* __restrict__ vg, __nv_bfloat16* __restrict__ dvg, long long M,
                                               int Ip, const int* __restrict__ col_map, float* __restrict__ dbias, float* __restrict__ partials, int rpb,
                                               const DropParams& drop) {
  const int cpr = Ip / 8;                 // 16-byte chunks per row of dh
  const int ch = threadIdx.x;
  if (ch >= cpr) return;
  const int c8 = ch * 8;
  const int tile = c8 >> 6, j = c8 & 63;
  const long long r0 = (long long)blockIdx.x * rpb, r1 = min(M, r0 + rpb);
  float sv[8], sg[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { sv[e] = 0.f; sg[e] = 0.f; }
#pragma unroll 2
  for (long long r = r0; r < r1; ++r) {
    const uint4 d4 = *reinterpret_cast<const uint4*>(dh + r * Ip + c8);
    const __nv_bfloat16* vrow = vg + r * 2 * Ip + tile * 128;
    const uint4 v4 = *reinterpret_cast<const uint4*>(vrow + j);
    const uint4 g4 = *reinterpret_cast<const uint4*>(vrow + 64 + j);
    const uint32_t dw[4] = {d4.x, d4.y, d4.z, d4.w}, vw[4] = {v4.x, v4.y, v4.z, v4.w}, gw[4] = {g4.x, g4.y, g4.z, g4.w};
    uint32_t ov[4], og[4];
    uint32_t keep = 0;
    if constexpr (DROP) keep = drop_keep8(drop, __ldg(drop.key), __ldg(drop.key + 1), DROP_SITE_FFN, 0, (uint32_t)r, (uint32_t)ch);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 d = unpack2_bf16(dw[k]);
      const float2 v = unpack2_bf16(vw[k]), g = unpack2_bf16(gw[k]);
      if constexpr (DROP) {
        d.x = (keep >> (2 * k)) & 1u ? d.x * drop.scale : 0.f;
        d.y = (keep >> (2 * k + 1)) & 1u ? d.y * drop.scale : 0.f;
      }
      float cdf0, pdf0, cdf1, pdf1;
      gelu_parts(g.x, cdf0, pdf0); gelu_parts(g.y, cdf1, pdf1);
      const float ov0 = d.x * g.x * cdf0, ov1 = d.y * g.y * cdf1;                       // d value = dh * gelu(g)
      const float og0 = d.x * v.x * fmaf(g.x, pdf0, cdf0), og1 = d.y * v.y * fmaf(g.y, pdf1, cdf1);   // d gate = dh * value * gelu'(g)
      sv[2 * k] += ov0; sv[2 * k + 1] += ov1; sg[2 * k] += og0; sg[2 * k + 1] += og1;
      ov[k] = pack2_bf16(ov0, ov1); og[k] = pack2_bf16(og0, og1);
    }
    __nv_bfloat16* orow = dvg + r * 2 * Ip + tile * 128;
    *reinterpret_cast<uint4*>(orow + j) = make_uint4(ov[0], ov[1], ov[2], ov[3]);
    *reinterpret_cast<uint4*>(orow + 64 + j) = make_uint4(og[0], og[1], og[2], og[3]);
  }
  if (partials) {
    // per-block partial column sums, reduced afterwards by tfx_colsum_f32 (same-address atomics from ~1000 blocks serialise in L2)
    float* prow = partials + (long long)blockIdx.x * 2 * Ip + tile * 128 + j;
    *reinterpret_cast<float4*>(prow) = make_float4(sv[0], sv[1], sv[2], sv[3]);
    *reinterpret_cast<float4*>(prow + 4) = make_float4(sv[4], sv[5], sv[6], sv[7]);
    *reinterpret_cast<float4*>(prow + 64) = make_float4(sg[0], sg[1], sg[2], sg[3]);
    *reinterpret_cast<float4*>(prow + 68) = make_float4(sg[4], sg[5], sg[6], sg[7]);
  } else if (dbias) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int cv = tile * 128 + j + e, cg = cv + 64;
      const int ov_ = col_map ? col_map[cv] : cv, og_ = col_map ? col_map[cg] : cg;
      if (ov_ >= 0) atomicAdd(dbias + ov_, sv[e]);
      if (og_ >= 0) atomicAdd(dbias + og_, sg[e]);
    }
  }
}

__global__ void geglu_bwd_k(const __nv_bfloat16* __restrict__ dh, const __nv_bfloat16* __restrict__ vg, __nv_bfloat16* __restrict__ dvg, long long M, int Ip,
                            const int* __restrict__ col_map, float* __restrict__ dbias, float* __restrict__ partials, int rpb) {
  geglu_bwd_body<false>(dh, vg, dvg, M, Ip, col_map, dbias, partials, rpb, DropParams{});
}
__global__ void geglu_bwd_drop_k(const __nv_bfloat16* __restrict__ dh, const __nv_bfloat16* __restrict__ vg, __nv_bfloat16* __restrict__ dvg, long long M, int Ip,
                                 const int* __restrict__ col_map, float* __restrict__ dbias, float* __restrict__ partials, int rpb, const DropParams drop) {
  geglu_bwd_body<true>(dh, vg, dvg, M, Ip, col_map, dbias, partials, rpb, drop);
}

// text cross-entropy, forward + backward in one pass (one warp per token)
// loss_sum += lse - logit[label] for label != ignore ; dlogits = (softmax - onehot) * gscale (bf16), 0 for ignored rows.
__global__ void __launch_bounds__(ROW_THREADS) ce_fwd_bwd_k(const float* __restrict__ logits, long long ld_l, const int* __restrict__ labels, int V, int vlimit,
                                                           float gscale, __nv_bfloat16* __restrict__ dlogits, long long ld_d, double* __restrict__ loss_sum,
                                                           int* __restrict__ n_valid, int M) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const int Vuse = vlimit > 0 ? min(vlimit, V) : V;
  double local = 0.0; int cnt = 0;
  for (int row = warp0; row < M; row += nwarps) {
    const int lab = labels[row];
    const float* lr = logits + (long long)row * ld_l;
    __nv_bfloat16* dr = dlogits ? dlogits + (long long)row * ld_d : nullptr;
    if (lab < 0) {
      if (dr) for (int c = lane; c < ld_d; c += 32) dr[c] = __float2bfloat16(0.f);
      continue;
    }
    float mx = -INFINITY;
    for (int c = lane; c < Vuse; c += 32) mx = fmaxf(mx, lr[c]);
    mx = warp_max(mx);
    float se = 0.f;
    for (int c = lane; c < Vuse; c += 32) se += __expf(lr[c] - mx);
    se = warp_sum(se);
    const float lse = mx + logf(se);
    // a label outside the un-masked vocabulary (text-only path, T.py:2653: logits >= num_text_tokens are filled with -finfo.max BEFORE the
    // cross entropy) sees the masked logit, exactly like the reference: loss = lse + FLT_MAX, gradient -1 on that column
    const float lab_logit = lab < Vuse ? lr[lab] : -3.402823466e+38f;
    if (lane == 0) { local += (double)lse - (double)lab_logit; ++cnt; }
    if (dr) {
      const float inv = 1.f / se;
      for (int c = lane; c < ld_d; c += 32) {
        float gq = 0.f;
        if (c < Vuse) gq = __expf(lr[c] - mx) * inv;
        if (c == lab) gq -= 1.f;
        dr[c] = __float2bfloat16(gq * gscale);
      }
    }
  }
  if (lane == 0 && cnt) { atomicAdd(loss_sum, local); atomicAdd(n_valid, cnt); }
}

// flow MSE, forward + backward:  sumsq += (pred - flow)^2 ; dpred = (pred - flow) * gscale (bf16)
__global__ void mse_fwd_bwd_k(const float* __restrict__ pred, long long ld_p, const float* __restrict__ flow, __nv_bfloat16* __restrict__ dpred, long long ld_d,
                              float gscale, double* __restrict__ sumsq, long long S, int dl) {
  const long long n = S * dl;
  float local = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / dl; const int c = (int)(i - r * dl);
    const float d = pred[r * ld_p + c] - flow[i];
    local += d * d;
    if (dpred) dpred[r * ld_d + c] = __float2bfloat16(d * gscale);
  }
  local = warp_sum(local);
  __shared__ float red[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[w] = local;
  __syncthreads();
  if (w == 0) {
    float v = lane < (blockDim.x >> 5) ? red[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0) atomicAdd(sumsq, (double)v);
  }
}

// flow MSE with the per-instance reconstruction loss (MP.py:177-194, T.py:3299-3308, 3420-3431; forward_modality T.py:2836-2856), forward +
// backward in one pass over a modality type's compact rows, one warp per row:
//   d = p - target                      (target: the flow, or the velocity blend)
//   r = a p - b g,  a = 1 - t,  b = t (interleaved: g = flow, since noised - noise = t flow) or 1 (forward_modality: g = orig - noise)
//   dpred = gscale d + rscale w_i a r   (bf16, written once) ;  sumsq += d^2 ;  inst_sumsq[i] += r^2 ;  type_sum += w_i r^2
// with i = row_inst[row] and w_i = inst_w[i] = 1 / (instances of the type x rows of instance i): type_sum / dl is the type's mean of the
// per-instance MSEs.  Instance index and weight are device data, so a captured graph replays batches with another instance split.
// A warp walks a contiguous run of rows and flushes its partial of the current instance with one atomic whenever the instance changes.
// SAME_G: g is the target (interleaved path without velocity): read once.
template <bool SAME_G>
__global__ void __launch_bounds__(256) mse_recon_fwd_bwd_k(const float* __restrict__ pred, long long ld_p, const float* __restrict__ target, const float* __restrict__ g,
                                                          const float* __restrict__ t_row, int b_is_t, const int* __restrict__ row_inst, const float* __restrict__ inst_w,
                                                          __nv_bfloat16* __restrict__ dpred, long long ld_d, float gscale, float rscale, double* __restrict__ sumsq,
                                                          double* __restrict__ inst_sumsq, double* __restrict__ type_sum, long long S, int dl, long long rows_per_warp) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long r0 = warp * rows_per_warp, r1 = min(S, r0 + rows_per_warp);
  float fl = 0.f, seg = 0.f, tsum = 0.f;           // flow sum of squares, recon sum of the current segment (lane partials); sum of w_i x segment (lane 0)
  int cur = -1;
  float cur_w = 0.f;
  for (long long r = r0; r < r1; ++r) {
    const int i = row_inst[r];
    if (i != cur) {
      if (cur >= 0) {
        const float s = warp_sum(seg);
        if (lane == 0) { atomicAdd(inst_sumsq + cur, (double)s); tsum += cur_w * s; }
        seg = 0.f;
      }
      cur = i; cur_w = inst_w[i];
    }
    const float t = t_row[r], a = 1.f - t, b = b_is_t ? t : 1.f;
    const float c = rscale * cur_w * a;
    const float* pr = pred + r * ld_p;
    const float* tr = target + r * dl;
    const float* gr = g + r * dl;
    __nv_bfloat16* dr = dpred + r * ld_d;
    for (int col = lane; col < dl; col += 32) {
      const float p = pr[col], f = tr[col];
      const float gv = SAME_G ? f : gr[col];
      const float d = p - f, rr = a * p - b * gv;
      fl += d * d; seg += rr * rr;
      float v = d * gscale;
      if (c != 0.f) v = fmaf(c, rr, v);              // c = 0 (w_r = 0): exactly the dpred of mse_fwd_bwd
      dr[col] = __float2bfloat16(v);
    }
  }
  if (cur >= 0) {
    const float s = warp_sum(seg);
    if (lane == 0) { atomicAdd(inst_sumsq + cur, (double)s); tsum += cur_w * s; }
  }
  fl = warp_sum(fl);
  __shared__ float red[2][8];
  if (lane == 0) { red[0][w] = fl; red[1][w] = tsum; }
  __syncthreads();
  if (w == 0) {
    float a = lane < (blockDim.x >> 5) ? red[0][lane] : 0.f, b = lane < (blockDim.x >> 5) ? red[1][lane] : 0.f;
    a = warp_sum(a); b = warp_sum(b);
    if (lane == 0) { atomicAdd(sumsq, (double)a); atomicAdd(type_sum, (double)b); }
  }
}

// out[col_map ? col_map[c] : c] += sum_r in[r][c]    (bias gradients)
__global__ void colsum_bf16_k(const __nv_bfloat16* __restrict__ in, long long ld, long long M, int N, const int* __restrict__ col_map, float* __restrict__ out, int rows_per_block) {
  const int cp = threadIdx.x & 31, rl = threadIdx.x >> 5;           // 32 column pairs x 8 row lanes
  const int c = blockIdx.x * 64 + cp * 2;
  const long long r0 = (long long)blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
  float a0 = 0.f, a1 = 0.f;
  if (c < N) {
    for (long long r = r0 + rl; r < r1; r += 8) {
      if (c + 1 < N) { const float2 v = unpack2_bf16(*reinterpret_cast<const uint32_t*>(in + r * ld + c)); a0 += v.x; a1 += v.y; }
      else a0 += __bfloat162float(in[r * ld + c]);
    }
  }
  __shared__ float s0[8][33], s1[8][33];
  s0[rl][cp] = a0; s1[rl][cp] = a1;
  __syncthreads();
  if (rl == 0 && c < N) {
#pragma unroll
    for (int k = 1; k < 8; ++k) { a0 += s0[k][cp]; a1 += s1[k][cp]; }
    const int o0 = col_map ? col_map[c] : c;
    if (o0 >= 0) atomicAdd(out + o0, a0);
    if (c + 1 < N) { const int o1 = col_map ? col_map[c + 1] : c + 1; if (o1 >= 0) atomicAdd(out + o1, a1); }
  }
}
__global__ void colsum_f32_k(const float* __restrict__ in, long long ld, long long M, int N, const int* __restrict__ col_map, float* __restrict__ out, int rows_per_block) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  const long long r0 = (long long)blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
  float a = 0.f;
  for (long long r = r0; r < r1; ++r) a += in[r * ld + c];
  const int o = col_map ? col_map[c] : c;
  if (o >= 0) atomicAdd(out + o, a);
}

// All per-step weight repacks in ONE launch: job j copies/casts a [R_dst x C_dst] destination from an fp32 source with an
// optional row gather; `blk_job[b]` maps a block to its job and `blk_first[j]` is the first block of job j.
__global__ void cast_pack_multi_k(const TfxPackJob* __restrict__ jobs, const int* __restrict__ blk_job, const int* __restrict__ blk_first) {
  const int j = blk_job[blockIdx.x];
  const TfxPackJob jb = jobs[j];
  const long long local = (long long)(blockIdx.x - blk_first[j]) * 2048;
  const long long n = jb.R_dst * (long long)jb.C_dst;
  const bool vec = (jb.C_dst & 7) == 0 && (jb.C_src & 3) == 0 && (jb.ld_src & 3) == 0 && !jb.dst_f32 &&
                   ((reinterpret_cast<uintptr_t>(jb.src) & 15) == 0) && ((reinterpret_cast<uintptr_t>(jb.dst) & 15) == 0);
  if (vec) {
    const long long i = local + (long long)threadIdx.x * 8;
    if (i >= n) return;
    const long long r = i / jb.C_dst; const int c = (int)(i - r * jb.C_dst);
    const long long sr = jb.row_src ? jb.row_src[r] : r;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
    if (sr >= 0) {
      const float* sp = jb.src + sr * jb.ld_src + c;
      if (c + 8 <= jb.C_src) {
        const float4 a = *reinterpret_cast<const float4*>(sp), b = *reinterpret_cast<const float4*>(sp + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) if (c + e < jb.C_src) v[e] = sp[e];
      }
    }
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(jb.dst) + i) = make_uint4(pack2_bf16(v[0], v[1]), pack2_bf16(v[2], v[3]), pack2_bf16(v[4], v[5]), pack2_bf16(v[6], v[7]));
  } else {
#pragma unroll 1
    for (int e = 0; e < 8; ++e) {
      const long long i = local + e * 256 + threadIdx.x;
      if (i >= n) break;
      const long long r = i / jb.C_dst; const int c = (int)(i - r * jb.C_dst);
      const long long sr = jb.row_src ? jb.row_src[r] : r;
      float v = 0.f;
      if (sr >= 0 && c < jb.C_src) v = jb.src[sr * jb.ld_src + c];
      if (jb.dst_f32) reinterpret_cast<float*>(jb.dst)[i] = v; else reinterpret_cast<__nv_bfloat16*>(jb.dst)[i] = __float2bfloat16(v);
    }
  }
}

__global__ void cast_f32_bf16_k(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = __float2bfloat16(src[i]);
}

__global__ void scale_bf16_k(__nv_bfloat16* __restrict__ p, const float* __restrict__ scale_ptr, long long n) {
  const float s = *scale_ptr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = __float2bfloat16(__bfloat162float(p[i]) * s);
}

__global__ void axpy_f32_k(float* __restrict__ y, const float* __restrict__ x, float a, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 yv = reinterpret_cast<float4*>(y)[i];
    const float4 xv = reinterpret_cast<const float4*>(x)[i];
    yv.x += a * xv.x; yv.y += a * xv.y; yv.z += a * xv.z; yv.w += a * xv.w;
    reinterpret_cast<float4*>(y)[i] = yv;
  }
}

// cos/sin table for RoPE: cs[p][i] = (cos(p*f_i), sin(p*f_i))   (rotary_embedding_torch; T.py:3223)
// cs_t (optional) is the same table stored [i][p]: consecutive tokens (consecutive positions) then read consecutive addresses, which is
// what the thread-per-row QKVG epilogue needs (with [p][i] every lane of a warp load hits a different 256-byte row).
__global__ void rope_table_k(const float* __restrict__ freqs, float2* __restrict__ cs, float2* __restrict__ cs_t, int max_pos, int nf) {
  const int n = max_pos * nf;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int p = i / nf, f = i - p * nf;
    const float a = (float)p * freqs[f];
    const float2 v = make_float2(cosf(a), sinf(a));
    cs[i] = v;
    if (cs_t) cs_t[(long long)f * max_pos + p] = v;
  }
}

// fused Adam(W): torch.optim.Adam semantics (L2 weight decay folded into the gradient unless decoupled).
// step_dev (optional): device-resident step counter - the bias corrections are then computed on the device (CUDA-graph replays cannot
// carry host-computed scalars); it is incremented by adam_step_inc_k right before this kernel.
__global__ void adam_step_inc_k(int* step_dev) { *step_dev += 1; }
__global__ void adam_k(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n, float lr, float b1, float b2,
                       float eps, float wd, int decoupled, float bc1, float bc2_sqrt, float gscale, int zero_grads, const int* __restrict__ step_dev) {
  if (step_dev) {
    const float st = (float)*step_dev;
    bc1 = 1.f - powf(b1, st);
    bc2_sqrt = sqrtf(1.f - powf(b2, st));
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float gi = g[i] * gscale, pi = p[i];
    if (wd != 0.f) { if (decoupled) pi *= (1.f - lr * wd); else gi += wd * pi; }
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi; v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] = pi - (lr / bc1) * (mi / denom);
    if (zero_grads) g[i] = 0.f;
  }
}

// ---- the rest of the train step the reference's examples run next to Adam (train_latent_with_text.py:142-153, train_image_only.py:90-110):
// global-norm gradient clipping (torch.nn.utils.clip_grad_norm_ semantics) and the EMA copy of the parameters (ema_pytorch lerp)
__global__ void grad_sumsq_k(const float* __restrict__ g, long long n, double* __restrict__ out) {
  double local = 0.0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) { const float v = g[i]; local += (double)v * v; }
  float lo = (float)local;                       // per-thread partial fits fp32 comfortably; the cross-block sum is in double
  lo = warp_sum(lo);
  __shared__ float red[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[w] = lo;
  __syncthreads();
  if (w == 0) {
    float v = lane < (blockDim.x >> 5) ? red[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0) atomicAdd(out, (double)v);
  }
}
// g *= min(1, max_norm / (pre_scale * sqrt(sumsq) + 1e-6))     (pre_scale = 1 / world_size when g holds the all-reduced SUM)
__global__ void clip_by_norm_k(float* __restrict__ g, long long n, const double* __restrict__ sumsq, float max_norm, float pre_scale) {
  const float total = pre_scale * (float)sqrt(*sumsq);
  const float coef = max_norm / (total + 1e-6f);
  if (coef >= 1.f) return;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) g[i] *= coef;
}
// ema = decay * ema + (1 - decay) * p
__global__ void ema_update_k(float* __restrict__ ema, const float* __restrict__ p, long long n, float decay) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) ema[i] = fmaf(decay, ema[i] - p[i], p[i]);
}

}  // namespace tfx

using namespace tfx;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int tfx_flow_noise(const float* x, const float* eps, const float* t_row, void* noised_bf16, long long ld_noised, float* noised_f32, float* flow, long long S, int dl, void* stream) {
  if (S <= 0) return 0;
  flow_noise_k<<<ew_grid(S * dl, 256), 256, 0, ST(stream)>>>(x, eps, t_row, (__nv_bfloat16*)noised_bf16, ld_noised, noised_f32, flow, S, dl);
  return check_launch("flow_noise");
}

int tfx_time_features(const float* times, const float* fourier_w, void* feats_bf16, int n, int half_dim, int ld, void* stream) {
  if (n <= 0) return 0;
  TFX_REQUIRE(ld >= 2 * half_dim + 1, "time_features: ld %d < %d", ld, 2 * half_dim + 1);
  time_features_k<<<ew_grid((long long)n * ld, 256), 256, 0, ST(stream)>>>(times, fourier_w, (__nv_bfloat16*)feats_bf16, n, half_dim, ld);
  return check_launch("time_features");
}

int tfx_table_op(const float* a, long long ld_a, const float* b, long long ld_b, float* out_f32, long long ld_of, void* out_bf16, long long ld_ob, long long rows, int cols,
                 int op, void* stream) {
  if (rows <= 0 || cols <= 0) return 0;
  table_op_k<<<ew_grid(rows * cols, 256), 256, 0, ST(stream)>>>(a, b, out_f32, (__nv_bfloat16*)out_bf16, rows, cols, ld_a, ld_b, ld_of, ld_ob, op);
  return check_launch("table_op");
}

int tfx_geglu_bwd_rows_per_block(void) { return 32; }

int tfx_geglu_bwd(const void* dh_bf16, const void* vg_bf16, void* dvg_bf16, long long M, int inner_pad, const int* col_map, float* dbias, float* partials, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(inner_pad % 64 == 0 && inner_pad <= 8192, "geglu_bwd: inner_pad %d must be a multiple of 64 and <= 8192", inner_pad);
  const int threads = ((inner_pad / 8) + 31) / 32 * 32;
  const int rpb = tfx_geglu_bwd_rows_per_block();
  geglu_bwd_k<<<(unsigned)((M + rpb - 1) / rpb), threads, 0, ST(stream)>>>((const __nv_bfloat16*)dh_bf16, (const __nv_bfloat16*)vg_bf16, (__nv_bfloat16*)dvg_bf16, M, inner_pad,
                                                                         col_map, dbias, partials, rpb);
  return check_launch("geglu_bwd");
}

int tfx_geglu_bwd_drop(const void* dh_bf16, const void* vg_bf16, void* dvg_bf16, long long M, int inner_pad, const int* col_map, float* dbias, float* partials,
                       const void* drop_key, float p_drop, int layer, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(inner_pad % 64 == 0 && inner_pad <= 8192, "geglu_bwd_drop: inner_pad %d must be a multiple of 64 and <= 8192", inner_pad);
  TFX_REQUIRE(drop_key && p_drop >= 0.f && p_drop <= 1.f && layer >= 0, "geglu_bwd_drop: needs a device key, p in [0, 1] (got %g) and layer >= 0 (got %d)", (double)p_drop, layer);
  const int threads = ((inner_pad / 8) + 31) / 32 * 32;
  const int rpb = tfx_geglu_bwd_rows_per_block();
  geglu_bwd_drop_k<<<(unsigned)((M + rpb - 1) / rpb), threads, 0, ST(stream)>>>((const __nv_bfloat16*)dh_bf16, (const __nv_bfloat16*)vg_bf16, (__nv_bfloat16*)dvg_bf16, M,
                                                                              inner_pad, col_map, dbias, partials, rpb, make_drop_params(drop_key, p_drop, layer));
  return check_launch("geglu_bwd_drop");
}

int tfx_ce_fwd_bwd(const float* logits, long long ld_logits, const int* labels, int V, int vlimit, float gscale, void* dlogits_bf16, long long ld_dlogits,
                   double* loss_sum, int* n_valid, int M, void* stream) {
  if (M <= 0) return 0;
  long long blocks = ((long long)M + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
  long long cap = (long long)num_sms() * 8;
  ce_fwd_bwd_k<<<(int)(blocks < cap ? blocks : cap), ROW_THREADS, 0, ST(stream)>>>(logits, ld_logits, labels, V, vlimit, gscale, (__nv_bfloat16*)dlogits_bf16, ld_dlogits, loss_sum,
                                                                               n_valid, M);
  return check_launch("ce_fwd_bwd");
}

int tfx_mse_fwd_bwd(const float* pred, long long ld_pred, const float* flow, void* dpred_bf16, long long ld_dpred, float gscale, double* sumsq, long long S, int dl, void* stream) {
  if (S <= 0) return 0;
  mse_fwd_bwd_k<<<ew_grid(S * dl, 256), 256, 0, ST(stream)>>>(pred, ld_pred, flow, (__nv_bfloat16*)dpred_bf16, ld_dpred, gscale, sumsq, S, dl);
  return check_launch("mse_fwd_bwd");
}

int tfx_mse_recon_fwd_bwd(const float* pred, long long ld_pred, const float* target, const float* g, const float* t_row, int b_is_t, const int* row_inst,
                          const float* inst_w, void* dpred_bf16, long long ld_dpred, float gscale, float rscale, double* sumsq, double* inst_sumsq, double* type_sum,
                          long long S, int dl, void* stream) {
  if (S <= 0) return 0;
  TFX_REQUIRE(pred && target && g && t_row && row_inst && inst_w && dpred_bf16 && sumsq && inst_sumsq && type_sum && dl > 0,
              "mse_recon_fwd_bwd: every pointer is required and dl (%d) must be > 0", dl);
  const int threads = 256, wpb = threads / 32;
  long long blocks = (S + wpb - 1) / wpb;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  const long long warps = blocks * wpb, rpw = (S + warps - 1) / warps;
  if (g == target)
    mse_recon_fwd_bwd_k<true><<<(unsigned)blocks, threads, 0, ST(stream)>>>(pred, ld_pred, target, g, t_row, b_is_t, row_inst, inst_w, (__nv_bfloat16*)dpred_bf16, ld_dpred,
                                                                          gscale, rscale, sumsq, inst_sumsq, type_sum, S, dl, rpw);
  else
    mse_recon_fwd_bwd_k<false><<<(unsigned)blocks, threads, 0, ST(stream)>>>(pred, ld_pred, target, g, t_row, b_is_t, row_inst, inst_w, (__nv_bfloat16*)dpred_bf16, ld_dpred,
                                                                           gscale, rscale, sumsq, inst_sumsq, type_sum, S, dl, rpw);
  return check_launch("mse_recon_fwd_bwd");
}

int tfx_colsum_bf16(const void* in_bf16, long long ld, long long M, int N, const int* col_map, float* out, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  const int rpb = 256;
  colsum_bf16_k<<<dim3((N + 63) / 64, (unsigned)((M + rpb - 1) / rpb)), 256, 0, ST(stream)>>>((const __nv_bfloat16*)in_bf16, ld, M, N, col_map, out, rpb);
  return check_launch("colsum_bf16");
}

int tfx_colsum_f32(const float* in, long long ld, long long M, int N, const int* col_map, float* out, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  const int rpb = 64;
  colsum_f32_k<<<dim3((N + 127) / 128, (unsigned)((M + rpb - 1) / rpb)), 128, 0, ST(stream)>>>(in, ld, M, N, col_map, out, rpb);
  return check_launch("colsum_f32");
}

int tfx_cast_pack_multi(const TfxPackJob* jobs_dev, const int* blk_job_dev, const int* blk_first_dev, int n_blocks, void* stream) {
  if (n_blocks <= 0) return 0;
  cast_pack_multi_k<<<n_blocks, 256, 0, ST(stream)>>>(jobs_dev, blk_job_dev, blk_first_dev);
  return check_launch("cast_pack_multi");
}

int tfx_cast_bf16(const float* src, void* dst_bf16, long long n, void* stream) {
  if (n <= 0) return 0;
  cast_f32_bf16_k<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(src, (__nv_bfloat16*)dst_bf16, n);
  return check_launch("cast_bf16");
}

int tfx_scale_bf16(void* p_bf16, const float* scale_ptr, long long n, void* stream) {
  if (n <= 0) return 0;
  scale_bf16_k<<<ew_grid(n, 256), 256, 0, ST(stream)>>>((__nv_bfloat16*)p_bf16, scale_ptr, n);
  return check_launch("scale_bf16");
}

int tfx_axpy_f32(float* y, const float* x, float a, long long n, void* stream) {
  if (n <= 0) return 0;
  TFX_REQUIRE(n % 4 == 0, "axpy_f32: n (%lld) must be a multiple of 4", n);
  axpy_f32_k<<<ew_grid(n / 4, 256), 256, 0, ST(stream)>>>(y, x, a, n / 4);
  return check_launch("axpy_f32");
}

int tfx_rope_table(const float* freqs, float* cos_sin, float* cos_sin_t, int max_pos, int n_freqs, void* stream) {
  if (max_pos <= 0) return 0;
  rope_table_k<<<ew_grid((long long)max_pos * n_freqs, 256), 256, 0, ST(stream)>>>(freqs, (float2*)cos_sin, (float2*)cos_sin_t, max_pos, n_freqs);
  return check_launch("rope_table");
}

int tfx_adam_step(float* params, float* grads, float* exp_avg, float* exp_avg_sq, long long n, float lr, float beta1, float beta2, float eps, float weight_decay,
                  int decoupled_wd, int step, float grad_scale, int zero_grads, int* step_dev, void* stream) {
  if (n <= 0) return 0;
  TFX_REQUIRE(step >= 1 || step_dev, "adam_step: step must be >= 1");
  float bc1 = 1.f, bc2s = 1.f;
  if (step_dev) adam_step_inc_k<<<1, 1, 0, ST(stream)>>>(step_dev);
  else { bc1 = 1.f - powf(beta1, (float)step); bc2s = sqrtf(1.f - powf(beta2, (float)step)); }
  adam_k<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, decoupled_wd, bc1, bc2s, grad_scale, zero_grads, step_dev);
  return check_launch("adam_step");
}

int tfx_grad_sumsq(const float* grads, long long n, double* sumsq_accum, void* stream) {
  if (n <= 0) return 0;
  grad_sumsq_k<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(grads, n, sumsq_accum);
  return check_launch("grad_sumsq");
}

int tfx_clip_by_norm(float* grads, long long n, const double* sumsq, float max_norm, float pre_scale, void* stream) {
  if (n <= 0) return 0;
  TFX_REQUIRE(max_norm > 0.f, "clip_by_norm: max_norm must be > 0");
  clip_by_norm_k<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(grads, n, sumsq, max_norm, pre_scale);
  return check_launch("clip_by_norm");
}

int tfx_ema_update(float* ema, const float* params, long long n, float decay, void* stream) {
  if (n <= 0) return 0;
  ema_update_k<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(ema, params, n, decay);
  return check_launch("ema_update");
}

}  // extern "C"
