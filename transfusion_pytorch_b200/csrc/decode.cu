// Device side of the kv-cache sampler (reference: transfusion.py:2079-2583 `sample_many`, 2669-2707 `generate_text_only`).
//
// The reference keeps one padded kv tensor per sample, re-pads and concatenates them on every step (T.py:2257-2277, 2323-2327,
// 2531-2533), builds a Bool[g, Lq, L+Lq] mask per step (T.py:2300-2304, 2415-2431) and reads every sampled token back to the host
// (`.item()`, T.py:2337).  Here the cache is a set of fixed slabs (sample s owns rows [s*cap, (s+1)*cap) of every layer's K / V matrix),
// the QKVG GEMM epilogue appends in place (tfx_gemm_qkvg kv_rows), "what may be attended" is two ints per sample (slab start, filled
// length), and the whole text loop - descriptor build, forward, token sampling, state update - runs from device-resident state so that a
// captured CUDA graph can be replayed step after step with no host round trip.
//
//   tfx_decode_prep      sampler state -> per-token metadata of the next text step (ids, RoPE position, cache row, tile = 1 query row)
//   tfx_attn_decode      one query row per (sample, head) against its slab: split-KV over the warps of a CTA, online softmax
//   tfx_sample_tokens    greedy / min-p + Gumbel-max sampling (T.py:580-591, 2692-2698) and the state machine update (T.py:2330-2349)
//   tfx_ode_pre/post     fixed-grid midpoint solver (torchdiffeq `midpoint`, T.py:1314-1318, 2523-2525) + classifier-free guidance
//                        combine (T.py:2521) on device-resident state: one captured graph per ODE evaluation, replayed 2 (steps-1) times
#include "common.cuh"
#include "../../include/tfx_b200.h"
#include <math.h>

namespace tfx {

int num_sms();

enum : int { ST_LEN = 0, ST_SEEN = 1, ST_LAST = 2, ST_PHASE = 3, ST_NTOK = 4, ST_HIST = 5 };

__global__ void decode_prep_k(const int* __restrict__ st, int S, int cap, int slab0, int* __restrict__ text_id, int* __restrict__ rope_pos, int* __restrict__ kv_row,
                              int* __restrict__ kv_limit, int* __restrict__ tq0, int* __restrict__ tqend, int* __restrict__ tkv0, int* __restrict__ tkvend,
                              int* __restrict__ counters) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s == 0 && counters) { counters[0] = 0; counters[1] += 1; }      // [0] samples still in the text phase after this step, [1] step number (RNG stream)
  if (s >= S) return;
  int len = st[ST_LEN * S + s];
  if (len > cap - 1) len = cap - 1;           // a finished sample that filled its slab: keep addresses inside the slab (its output is ignored)
  const int base = (slab0 + s) * cap;
  text_id[s] = st[ST_LAST * S + s];
  rope_pos[s] = st[ST_SEEN * S + s];
  kv_row[s] = base + len;
  kv_limit[s] = base + len;
  tq0[s] = s; tqend[s] = s + 1; tkv0[s] = base; tkvend[s] = base + len + 1;
}

// one CTA = one (single-query-row tile, head); 4 warps split the keys of the slab; lane <-> key for the scores, lane <-> 2 output dims for P V
__global__ void __launch_bounds__(128) attn_decode_k(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v,
                                                    long long ld_q, long long ld_k, long long ld_v, const float* __restrict__ gates, int H, const int* __restrict__ kv_limit,
                                                    const int* __restrict__ tile_q0, const int* __restrict__ tile_kv0, const int* __restrict__ tile_kvend,
                                                    __nv_bfloat16* __restrict__ o, long long ld_o, float scale, float cap) {
  __shared__ float sq[64];
  __shared__ float s_m[4], s_l[4];
  __shared__ float s_o[4][64];
  const int tile = blockIdx.x, head = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row = tile_q0[tile];
  const int kv0 = tile_kv0[tile];
  const int kv_end = min(tile_kvend[tile], kv_limit[row] + 1);
  if (tid < 64) sq[tid] = __bfloat162float(q[(long long)row * ld_q + head * 64 + tid]) * scale;
  __syncthreads();
  const float inv_cap = 1.f / cap;
  float m = -INFINITY, l = 0.f, a0 = 0.f, a1 = 0.f;
  for (int base = kv0 + warp * 32; base < kv_end; base += 128) {
    const int key = base + lane;
    const bool ok = key < kv_end;
    float s = -INFINITY;
    if (ok) {
      const uint4* kp = reinterpret_cast<const uint4*>(k + (long long)key * ld_k + head * 64);
      float d = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 t = kp[c];
        const float2 x0 = unpack2_bf16(t.x), x1 = unpack2_bf16(t.y), x2 = unpack2_bf16(t.z), x3 = unpack2_bf16(t.w);
        d += x0.x * sq[c * 8] + x0.y * sq[c * 8 + 1] + x1.x * sq[c * 8 + 2] + x1.y * sq[c * 8 + 3] + x2.x * sq[c * 8 + 4] + x2.y * sq[c * 8 + 5] +
             x3.x * sq[c * 8 + 6] + x3.y * sq[c * 8 + 7];
      }
      s = cap * tanh_acc(d * inv_cap);
    }
    const float mn = fmaxf(m, warp_max(s));            // finite: lane 0 of this chunk is a valid key
    const float p = ok ? __expf(s - mn) : 0.f;
    const float corr = __expf(m - mn);
    l = l * corr + warp_sum(p);
    a0 *= corr; a1 *= corr; m = mn;
    const int nk = min(32, kv_end - base);
#pragma unroll 4
    for (int j = 0; j < nk; ++j) {
      const float pj = __shfl_sync(0xffffffffu, p, j);
      const float2 vv = unpack2_bf16(*reinterpret_cast<const uint32_t*>(v + (long long)(base + j) * ld_v + head * 64 + 2 * lane));
      a0 = fmaf(pj, vv.x, a0); a1 = fmaf(pj, vv.y, a1);
    }
  }
  if (lane == 0) { s_m[warp] = m; s_l[warp] = l; }
  s_o[warp][2 * lane] = a0; s_o[warp][2 * lane + 1] = a1;
  __syncthreads();
  if (warp == 0) {
    float M4 = fmaxf(fmaxf(s_m[0], s_m[1]), fmaxf(s_m[2], s_m[3]));
    float L = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float c = s_m[w] == -INFINITY ? 0.f : __expf(s_m[w] - M4);
      L += s_l[w] * c; o0 += s_o[w][2 * lane] * c; o1 += s_o[w][2 * lane + 1] * c;
    }
    float g = L > 0.f ? 1.f / L : 0.f;
    if (gates) g *= 1.f / (1.f + __expf(-gates[(long long)row * H + head]));
    *reinterpret_cast<uint32_t*>(o + (long long)row * ld_o + head * 64 + 2 * lane) = pack2_bf16(o0 * g, o1 * g);
  }
}

// head dim 128: lane <-> DH / 32 output dims for P V.  Instantiated at 128 only: the 64-wide kernel above keeps its own code, because this
// template at DH = 64 (a uint32_t pair per lane) schedules differently and measured 0.2 % slower (129.6 vs 129.4 us per call, H100 80GB HBM3, 700 W).
template <int DH>
__global__ void __launch_bounds__(128) attn_decode_dh_k(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v,
                                                       long long ld_q, long long ld_k, long long ld_v, const float* __restrict__ gates, int H, const int* __restrict__ kv_limit,
                                                       const int* __restrict__ tile_q0, const int* __restrict__ tile_kv0, const int* __restrict__ tile_kvend,
                                                       __nv_bfloat16* __restrict__ o, long long ld_o, float scale, float cap) {
  constexpr int NV = DH / 32;
  static_assert(NV == 4, "the P V loop and the output store move 4 dims per lane");
  __shared__ float sq[DH];
  __shared__ float s_m[4], s_l[4];
  __shared__ float s_o[4][DH];
  const int tile = blockIdx.x, head = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row = tile_q0[tile];
  const int kv0 = tile_kv0[tile];
  const int kv_end = min(tile_kvend[tile], kv_limit[row] + 1);
  if (tid < DH) sq[tid] = __bfloat162float(q[(long long)row * ld_q + head * DH + tid]) * scale;
  __syncthreads();
  const float inv_cap = 1.f / cap;
  float m = -INFINITY, l = 0.f, a[NV];
#pragma unroll
  for (int e = 0; e < NV; ++e) a[e] = 0.f;
  for (int base = kv0 + warp * 32; base < kv_end; base += 128) {
    const int key = base + lane;
    const bool ok = key < kv_end;
    float s = -INFINITY;
    if (ok) {
      const uint4* kp = reinterpret_cast<const uint4*>(k + (long long)key * ld_k + head * DH);
      float d = 0.f;
#pragma unroll
      for (int c = 0; c < DH / 8; ++c) {
        const uint4 t = kp[c];
        const float2 x0 = unpack2_bf16(t.x), x1 = unpack2_bf16(t.y), x2 = unpack2_bf16(t.z), x3 = unpack2_bf16(t.w);
        d += x0.x * sq[c * 8] + x0.y * sq[c * 8 + 1] + x1.x * sq[c * 8 + 2] + x1.y * sq[c * 8 + 3] + x2.x * sq[c * 8 + 4] + x2.y * sq[c * 8 + 5] +
             x3.x * sq[c * 8 + 6] + x3.y * sq[c * 8 + 7];
      }
      s = cap * tanh_acc(d * inv_cap);
    }
    const float mn = fmaxf(m, warp_max(s));            // finite: lane 0 of this chunk is a valid key
    const float p = ok ? __expf(s - mn) : 0.f;
    const float corr = __expf(m - mn);
    l = l * corr + warp_sum(p);
#pragma unroll
    for (int e = 0; e < NV; ++e) a[e] *= corr;
    m = mn;
    const int nk = min(32, kv_end - base);
#pragma unroll 4
    for (int j = 0; j < nk; ++j) {
      const float pj = __shfl_sync(0xffffffffu, p, j);
      const uint2 w = *reinterpret_cast<const uint2*>(v + (long long)(base + j) * ld_v + head * DH + NV * lane);
      const float2 v0 = unpack2_bf16(w.x), v1 = unpack2_bf16(w.y);
      a[0] = fmaf(pj, v0.x, a[0]); a[1] = fmaf(pj, v0.y, a[1]); a[2] = fmaf(pj, v1.x, a[2]); a[3] = fmaf(pj, v1.y, a[3]);
    }
  }
  if (lane == 0) { s_m[warp] = m; s_l[warp] = l; }
#pragma unroll
  for (int e = 0; e < NV; ++e) s_o[warp][NV * lane + e] = a[e];
  __syncthreads();
  if (warp == 0) {
    float M4 = fmaxf(fmaxf(s_m[0], s_m[1]), fmaxf(s_m[2], s_m[3]));
    float L = 0.f, out[NV];
#pragma unroll
    for (int e = 0; e < NV; ++e) out[e] = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float c = s_m[w] == -INFINITY ? 0.f : __expf(s_m[w] - M4);
      L += s_l[w] * c;
#pragma unroll
      for (int e = 0; e < NV; ++e) out[e] += s_o[w][NV * lane + e] * c;
    }
    float g = L > 0.f ? 1.f / L : 0.f;
    if (gates) g *= 1.f / (1.f + __expf(-gates[(long long)row * H + head]));
    *reinterpret_cast<uint2*>(o + (long long)row * ld_o + head * DH + NV * lane) = make_uint2(pack2_bf16(out[0] * g, out[1] * g), pack2_bf16(out[2] * g, out[3] * g));
  }
}

__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// one warp per sample.  Samples that are not in the text phase are left untouched.
//   temperature == 0: argmax over the V logits, lowest index on ties (T.py:583-584, 2692-2693)
//   otherwise: logits / temperature -> min-p filter (T.py:574-578) -> [restrict to ids < vlimit, T.py:2697] -> Gumbel-max draw
// then the reference's per-sample bookkeeping (T.py:2330-2349): the fed token's key/value row is committed (len += 1), the position advances,
// [eos] / length limit end the sample, a [som] id parks it for the modality phase.
__global__ void __launch_bounds__(ROW_THREADS) sample_tokens_k(const float* __restrict__ logits, long long ld, const int* __restrict__ rows, int V, int vlimit,
                                                              int* __restrict__ st, int S, int* __restrict__ hist, int hist_cap, int eos_id, const int* __restrict__ som_ids,
                                                              int n_som, int max_length, float temperature, float min_p, unsigned long long seed, int* __restrict__ counters,
                                                              int advance) {
  const int lane = threadIdx.x & 31;
  const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (s >= S) return;
  if (st[ST_PHASE * S + s] != 0) return;
  const float* lr = logits + (long long)(rows ? rows[s] : s) * ld;
  float best = -INFINITY; int bi = 0x7fffffff;
  if (temperature == 0.f) {
    for (int c = lane; c < V; c += 32) { const float x = lr[c]; if (x > best) { best = x; bi = c; } }
  } else {
    const float it = 1.f / temperature;
    float mx = -INFINITY;
    for (int c = lane; c < V; c += 32) mx = fmaxf(mx, lr[c] * it);
    mx = warp_max(mx);
    // min-p: keep p_c >= min_p * p_max  <=>  x_c - mx >= log(min_p)
    const float thr = min_p > 0.f ? logf(min_p) : -INFINITY;
    const unsigned long long step = counters ? (unsigned long long)(unsigned)counters[1] : 0ull;
    const int Vs = vlimit > 0 ? min(vlimit, V) : V;
    for (int c = lane; c < Vs; c += 32) {
      const float x = lr[c] * it;
      if (x - mx < thr) continue;
      const unsigned long long h = mix64(seed ^ mix64((step << 40) ^ ((unsigned long long)s << 20) ^ (unsigned long long)c));
      // 23 bits: (k + 1/2) 2^-23 is exact in fp32 and lies in [2^-24, 1 - 2^-24].  (24 bits + 0.5 rounds 2^24 - 1/2 up to u = 1, a +inf Gumbel.)
      const float u = ((float)(h >> 41) + 0.5f) * (1.f / 8388608.f);
      const float gmb = -logf(-logf(u));                   // __logf's absolute error near u = 1 is as large as -log u itself
      const float y = x + gmb;
      if (y > best) { best = y; bi = c; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (lane == 0) {
    const int tok = bi == 0x7fffffff ? 0 : bi;
    int hl = st[ST_HIST * S + s];
    if (hl < hist_cap) hist[(long long)s * hist_cap + hl] = tok;
    st[ST_HIST * S + s] = hl + 1;
    st[ST_LAST * S + s] = tok;
    if (advance) { st[ST_LEN * S + s] += 1; st[ST_SEEN * S + s] += 1; }
    const int nt = st[ST_NTOK * S + s] + 1;
    st[ST_NTOK * S + s] = nt;
    int phase = 0;
    if (tok == eos_id) phase = 2;
    else if (nt > max_length) phase = 2;
    else { for (int i = 0; i < n_som; ++i) if (tok == som_ids[i]) phase = 1; }
    st[ST_PHASE * S + s] = phase;
    if (phase == 0 && counters) atomicAdd(&counters[0], 1);
  }
}
__global__ void counter_inc_k(int* c) { *c += 1; }

// ---------------------------------------------------------------- fixed-grid midpoint ODE on device-resident state
// tab[e] = (t_e, c_e, h_e, mode_e): evaluation e runs the model at  y + c_e * f_prev  and time t_e;
// mode 0 (first half step):  f_prev = f ;  mode 1 (second half step):  y += h_e * f.      f = u + cfg (c - u)   (T.py:2521)
__global__ void ode_pre_k(const float* __restrict__ y, const float* __restrict__ fprev, float* __restrict__ x_eval, long long n, int dup, const float4* __restrict__ tab,
                          const int* __restrict__ idx, float* __restrict__ cond_times, int n_cond) {
  const float4 e = tab[*idx];
  const long long gid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (gid < n_cond && cond_times) cond_times[gid] = e.x;
  for (long long i = gid; i < n; i += (long long)gridDim.x * blockDim.x) {
    float xv = y[i];
    if (e.y != 0.f) xv = fmaf(e.y, fprev[i], xv);
    for (int d = 0; d < dup; ++d) x_eval[d * n + i] = xv;
  }
}
__global__ void ode_post_k(float* __restrict__ y, float* __restrict__ fprev, const float* __restrict__ pc, const float* __restrict__ pu, float cfg, long long n,
                           const float4* __restrict__ tab, const int* __restrict__ idx) {
  const float4 e = tab[*idx];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float f = pc[i];
    if (pu) { const float u = pu[i]; f = u + cfg * (f - u); }
    if (e.w == 0.f) fprev[i] = f; else y[i] = fmaf(e.z, f, y[i]);
  }
}

static inline int ew_grid_d(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  long long cap = (long long)num_sms() * 8;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

}  // namespace tfx

using namespace tfx;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int tfx_decode_prep(const int* state, int S, int cap, int slab0, int* text_id, int* rope_pos, int* kv_row, int* kv_limit, int* tile_q0, int* tile_qend, int* tile_kv0,
                    int* tile_kvend, int* counters, void* stream) {
  if (S <= 0) return 0;
  TFX_REQUIRE(cap > 0, "decode_prep: slab capacity must be > 0");
  decode_prep_k<<<(S + 127) / 128, 128, 0, ST(stream)>>>(state, S, cap, slab0, text_id, rope_pos, kv_row, kv_limit, tile_q0, tile_qend, tile_kv0, tile_kvend, counters);
  return check_launch("decode_prep");
}

int tfx_attn_decode(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H, const int* kv_limit,
                    const int* tile_q0, const int* tile_kv0, const int* tile_kvend, int n_tiles, void* o, long long ld_o, float scale, float softcap, void* stream) {
  if (n_tiles <= 0) return 0;
  TFX_REQUIRE(softcap > 0.f, "attn_decode: softcap must be > 0 (got %f)", softcap);
  TFX_REQUIRE(ld_k % 8 == 0 && ld_v % 2 == 0 && ld_o % 2 == 0, "attn_decode: row pitches must keep 16-byte key rows and 4-byte value / output pairs aligned");
  attn_decode_k<<<dim3(n_tiles, H), 128, 0, ST(stream)>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, ld_q, ld_k, ld_v, gates, H, kv_limit, tile_q0,
                                                         tile_kv0, tile_kvend, (__nv_bfloat16*)o, ld_o, scale, softcap);
  return check_launch("attn_decode");
}

int tfx_attn_decode_d128(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H, const int* kv_limit,
                         const int* tile_q0, const int* tile_kv0, const int* tile_kvend, int n_tiles, void* o, long long ld_o, float scale, float softcap, void* stream) {
  if (n_tiles <= 0) return 0;
  TFX_REQUIRE(softcap > 0.f, "attn_decode_d128: softcap must be > 0 (got %f)", softcap);
  TFX_REQUIRE(ld_k % 8 == 0 && ld_v % 4 == 0 && ld_o % 4 == 0, "attn_decode_d128: row pitches must keep 16-byte key rows and 8-byte value / output quads aligned");
  attn_decode_dh_k<128><<<dim3(n_tiles, H), 128, 0, ST(stream)>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, ld_q, ld_k, ld_v, gates, H, kv_limit,
                                                                 tile_q0, tile_kv0, tile_kvend, (__nv_bfloat16*)o, ld_o, scale, softcap);
  return check_launch("attn_decode_d128");
}

int tfx_sample_tokens(const float* logits, long long ld_logits, const int* rows, int V, int vlimit, int* state, int S, int* hist, int hist_cap, int eos_id, const int* som_ids,
                      int n_som, int max_length, float temperature, float min_p, unsigned long long seed, int* counters, int advance, void* stream) {
  if (S <= 0) return 0;
  TFX_REQUIRE(V > 0 && temperature >= 0.f, "sample_tokens: bad arguments");
  sample_tokens_k<<<(S + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, ROW_THREADS, 0, ST(stream)>>>(logits, ld_logits, rows, V, vlimit, state, S, hist, hist_cap, eos_id, som_ids, n_som,
                                                                                            max_length, temperature, min_p, seed, counters, advance);
  return check_launch("sample_tokens");
}

int tfx_ode_pre(const float* y, const float* f_prev, float* x_eval, long long n, int dup, const float* tab, const int* idx, float* cond_times, int n_cond, void* stream) {
  if (n <= 0) return 0;
  TFX_REQUIRE(dup >= 1 && (((uintptr_t)tab) & 15) == 0, "ode_pre: dup must be >= 1 and tab 16-byte aligned");
  ode_pre_k<<<ew_grid_d(n > n_cond ? n : n_cond, 256), 256, 0, ST(stream)>>>(y, f_prev, x_eval, n, dup, (const float4*)tab, idx, cond_times, n_cond);
  return check_launch("ode_pre");
}

int tfx_ode_post(float* y, float* f_prev, const float* pred_cond, const float* pred_uncond, float cfg_scale, long long n, const float* tab, const int* idx, void* stream) {
  if (n <= 0) return 0;
  ode_post_k<<<ew_grid_d(n, 256), 256, 0, ST(stream)>>>(y, f_prev, pred_cond, pred_uncond, cfg_scale, n, (const float4*)tab, idx);
  return check_launch("ode_post");
}

int tfx_counter_inc(int* counter, void* stream) {
  counter_inc_k<<<1, 1, 0, ST(stream)>>>(counter);
  return check_launch("counter_inc");
}

}  // extern "C"
