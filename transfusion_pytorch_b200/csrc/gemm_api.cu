// C-ABI entry points of the wgmma GEMM family (see gemm_sm90.cuh).  Each replaces an ATen matmul call
// site of the reference (cited per function in include/tfx_b200.h).
#include "gemm_sm90.cuh"
#include "common.cuh"
#include "../../include/tfx_b200.h"
#include <string.h>

namespace tfx { int num_sms(); }
using namespace tfx;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

static int finish(int rc, const char* what) {
  if (rc == 0) return 0;
  if (rc <= -1000) set_error("%s: cuTensorMapEncodeTiled failed (CUresult %d) - check 16-byte alignment of pointers and row pitches", what, -(rc + 1000));
  else if (rc == -1) set_error("%s: cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)", what);
  else if (rc == -2) set_error("%s: cudaFuncSetAttribute(max dynamic smem) failed: %s", what, cudaGetErrorString(cudaGetLastError()));
  else set_error("%s: kernel launch failed: %s", what, cudaGetErrorString(cudaGetLastError()));
  return rc;
}

static int dispatch_major(const GemmOperand& A, const GemmOperand& B, const GemmParams& p, cudaStream_t st) {
  const int sms = num_sms();
  if (gemm_store_wide(p.K, p.k_splits)) {
    if (!A.mn_major && !B.mn_major) return launch_gemm_wide_t<false, false>(A, B, p, sms, st);
    if (!A.mn_major && B.mn_major) return launch_gemm_wide_t<false, true>(A, B, p, sms, st);
    if (A.mn_major && B.mn_major) return launch_gemm_wide_t<true, true>(A, B, p, sms, st);
    return launch_gemm_wide_t<true, false>(A, B, p, sms, st);
  }
  if (!A.mn_major && !B.mn_major) return launch_gemm_t<false, false, EPI_STORE>(A, B, p, sms, st);
  if (!A.mn_major && B.mn_major) return launch_gemm_t<false, true, EPI_STORE>(A, B, p, sms, st);
  if (A.mn_major && B.mn_major) return launch_gemm_t<true, true, EPI_STORE>(A, B, p, sms, st);
  return launch_gemm_t<true, false, EPI_STORE>(A, B, p, sms, st);
}

// the four tfx_gemm_qkvg* entry points; `name` is the entry point's name for error messages.  W is [to_qk | to_v | gate tile] with
// N = 3 H DH + 128, the 128-row gate tile holding to_gates (rows [0, H)) and the value-residual mix (rows [round_even(H), + H)); with
// neither gates nor mix_pre there is no gate tile and N = 3 H DH.  At DH = 64 a 128-column tile holds two heads, so H is even; at 128 it
// holds one, so any H in [1, 16].
template <int EPI>
static int gemm_qkvg(const char* name, const void* u, long long ldu, const void* W, long long ldw, int M, int H, int D, void* q, void* k, void* v,
                     float* gates, float* qk_inv, const float* q_gamma, const float* k_gamma, const int* rope_pos, const float* rope_cs_t, int rope_len,
                     const int* kv_rows, float* mix_pre, void* stream) {
  constexpr int DH = qkvg_dh(EPI);
  if (M <= 0) return 0;
  if constexpr (DH == 64) {
    TFX_REQUIRE(H >= 2 && H % 2 == 0 && H <= 32, "%s: heads must be even and in [2, 32] (got %d)", name, H);
  } else {
    TFX_REQUIRE(H >= 1 && H <= 16, "%s: heads must be in [1, 16] (got %d)", name, H);
  }
  TFX_REQUIRE(ldu % 8 == 0 && ldw % 8 == 0, "%s: row pitches must be multiples of 8", name);
  GemmParams p; memset(&p, 0, sizeof(p));
  p.M = M; p.N = 3 * H * DH + (gates || mix_pre ? 128 : 0); p.K = D; p.k_splits = 1; p.H = H;
  p.q = (__nv_bfloat16*)q; p.k = (__nv_bfloat16*)k; p.v = (__nv_bfloat16*)v; p.gates = gates; p.qk_inv = qk_inv;
  p.q_gamma = q_gamma; p.k_gamma = k_gamma; p.rope_pos = rope_pos; p.rope_cs = (const float2*)rope_cs_t; p.rope_len = rope_len; p.kv_rows = kv_rows; p.mix_pre = mix_pre;
  GemmOperand a{u, ldu, false}, b{W, ldw, false};
  return finish(launch_gemm_t<false, false, EPI>(a, b, p, num_sms(), ST(stream)), name);
}

extern "C" {

int tfx_gemm_set_cluster_mode(int mode) {
  TFX_REQUIRE(mode >= 1 && mode <= 3, "gemm_set_cluster_mode: mode %d not in {1 (never pair, default), 2 (always pair), 3 (pair long-K launches)}", mode);
  gemm_cluster_mode_ref() = mode;
  return 0;
}

int tfx_gemm_set_wide_mode(int mode) {
  TFX_REQUIRE(mode >= 1 && mode <= 3, "gemm_set_wide_mode: mode %d not in {1 (long work items, default), 2 (always), 3 (never)}", mode);
  gemm_wide_mode_ref() = mode;
  return 0;
}

int tfx_gemm_store_items(int M, int N, int K, int a_mn_major, int b_mn_major, int k_splits, int* geometry) {
  TFX_REQUIRE(M > 0 && N > 0 && K > 0 && geometry, "gemm_store_items: needs M, N, K > 0 (got %d, %d, %d) and an output array", M, N, K);
  (void)a_mn_major; (void)b_mn_major;      // the tile does not depend on the operand layouts today
  const int tile_m = gemm_store_wide(K, k_splits) ? GemmWideCfg::BM : GEMM_BM;
  const int s = gemm_effective_splits(K, k_splits);
  geometry[0] = ((M + tile_m - 1) / tile_m) * ((N + GEMM_BN - 1) / GEMM_BN) * s;
  geometry[1] = gemm_kb_per_item(K, s);
  geometry[2] = tile_m;
  geometry[3] = s;
  return 0;
}

int tfx_gemm_store(const void* A, long long lda, int a_mn_major, const void* B, long long ldb, int b_mn_major, int M, int N, int K,
                   float* out_f32, long long ld_f32, void* out_bf16, long long ld_bf16, const float* bias, const long long* row_off,
                   float alpha, int accumulate, int k_splits, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  TFX_REQUIRE(K > 0, "gemm_store: K must be > 0");
  TFX_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "gemm_store: operand row pitches (%lld, %lld) must be multiples of 8 bf16", lda, ldb);
  TFX_REQUIRE(!(k_splits > 1) || (accumulate && out_f32 && !out_bf16 && !bias), "gemm_store: split-K requires fp32 accumulate output only");
  GemmParams p; memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K; p.k_splits = k_splits < 1 ? 1 : k_splits;
  p.out_f32 = out_f32; p.ld_f32 = ld_f32; p.out_bf16 = (__nv_bfloat16*)out_bf16; p.ld_bf16 = ld_bf16; p.bias = bias; p.row_off = row_off;
  p.alpha = alpha; p.accumulate_f32 = accumulate;
  GemmOperand a{A, lda, a_mn_major != 0}, b{B, ldb, b_mn_major != 0};
  const int rc = dispatch_major(a, b, p, ST(stream));
  return finish(rc, "gemm_store");
}

int tfx_gemm_qkvg(const void* u, long long ldu, const void* W, long long ldw, int M, int H, int D, void* q, void* k, void* v, float* gates, float* qk_inv,
                  const float* q_gamma, const float* k_gamma, const int* rope_pos, const float* rope_cs_t, int rope_len, const int* kv_rows, float* mix_pre, void* stream) {
  return gemm_qkvg<EPI_QKVG>("gemm_qkvg", u, ldu, W, ldw, M, H, D, q, k, v, gates, qk_inv, q_gamma, k_gamma, rope_pos, rope_cs_t, rope_len, kv_rows, mix_pre, stream);
}

int tfx_gemm_qkvg_rope(const void* u, long long ldu, const void* W, long long ldw, int M, int H, int D, void* q, void* k, void* v, float* gates,
                       const int* rope_pos, const float* rope_cs_t, int rope_len, const int* kv_rows, float* mix_pre, void* stream) {
  return gemm_qkvg<EPI_QKVG_ROPE>("gemm_qkvg_rope", u, ldu, W, ldw, M, H, D, q, k, v, gates, nullptr, nullptr, nullptr, rope_pos, rope_cs_t, rope_len, kv_rows,
                                  mix_pre, stream);
}

int tfx_gemm_qkvg_d128(const void* u, long long ldu, const void* W, long long ldw, int M, int H, int D, void* q, void* k, void* v, float* gates, float* qk_inv,
                       const float* q_gamma, const float* k_gamma, const int* rope_pos, const float* rope_cs_t, int rope_len, const int* kv_rows, float* mix_pre, void* stream) {
  return gemm_qkvg<EPI_QKVG_D128>("gemm_qkvg_d128", u, ldu, W, ldw, M, H, D, q, k, v, gates, qk_inv, q_gamma, k_gamma, rope_pos, rope_cs_t, rope_len, kv_rows,
                                  mix_pre, stream);
}

int tfx_gemm_qkvg_rope_d128(const void* u, long long ldu, const void* W, long long ldw, int M, int H, int D, void* q, void* k, void* v, float* gates,
                            const int* rope_pos, const float* rope_cs_t, int rope_len, const int* kv_rows, float* mix_pre, void* stream) {
  return gemm_qkvg<EPI_QKVG_ROPE_D128>("gemm_qkvg_rope_d128", u, ldu, W, ldw, M, H, D, q, k, v, gates, nullptr, nullptr, nullptr, rope_pos, rope_cs_t, rope_len,
                                       kv_rows, mix_pre, stream);
}

int tfx_gemm_resid(const void* A, long long lda, const void* A2, long long lda2, int K1, const void* W, long long ldw, int M, int N, int K, const float* bias,
                   const float* x_res, float* x_out, void* x_out_bf16, void* y_bf16, const int* cond_row, const float* zgate, long long zgate_ld,
                   const float* layerscale, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(N % 32 == 0, "gemm_resid: N (%d) must be a multiple of 32", N);
  TFX_REQUIRE(!A2 || K1 % 64 == 0, "gemm_resid: K1 (%d) must be a multiple of 64", K1);
  TFX_REQUIRE(x_out || x_out_bf16, "gemm_resid: at least one of x_out (fp32) / x_out_bf16 is required");
  GemmParams p; memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K; p.k_splits = 1; p.K1 = A2 ? K1 : K; p.bias = bias;
  p.x_res = x_res; p.x_out = x_out; p.x_out_bf16 = (__nv_bfloat16*)x_out_bf16; p.y_bf16 = (__nv_bfloat16*)y_bf16;
  p.cond_row = cond_row; p.zgate = zgate; p.zgate_ld = zgate_ld; p.ls = layerscale;
  GemmOperand a{A, lda, false, A2, lda2}, b{W, ldw, false};
  return finish(launch_gemm_t<false, false, EPI_RESID>(a, b, p, num_sms(), ST(stream)), "gemm_resid");
}

int tfx_gemm_geglu(const void* u, long long ldu, const void* W1p, long long ldw, const float* b1p, int M, int Np, int K, void* vg, void* h, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(Np % 128 == 0, "gemm_geglu: packed N (%d) must be a multiple of 128", Np);
  GemmParams p; memset(&p, 0, sizeof(p));
  p.M = M; p.N = Np; p.K = K; p.k_splits = 1; p.bias = b1p; p.vg = (__nv_bfloat16*)vg; p.h = (__nv_bfloat16*)h;
  GemmOperand a{u, ldu, false}, b{W1p, ldw, false};
  return finish(launch_gemm_t<false, false, EPI_GEGLU>(a, b, p, num_sms(), ST(stream)), "gemm_geglu");
}

int tfx_gemm_geglu_drop(const void* u, long long ldu, const void* W1p, long long ldw, const float* b1p, int M, int Np, int K, void* vg, void* h,
                        const void* drop_key, float p_drop, int layer, void* stream) {
  if (M <= 0) return 0;
  TFX_REQUIRE(Np % 128 == 0, "gemm_geglu_drop: packed N (%d) must be a multiple of 128", Np);
  TFX_REQUIRE(drop_key && p_drop >= 0.f && p_drop <= 1.f && layer >= 0, "gemm_geglu_drop: needs a device key, p in [0, 1] (got %g) and layer >= 0 (got %d)", (double)p_drop, layer);
  GemmParams p; memset(&p, 0, sizeof(p));
  p.M = M; p.N = Np; p.K = K; p.k_splits = 1; p.bias = b1p; p.vg = (__nv_bfloat16*)vg; p.h = (__nv_bfloat16*)h;
  p.drop = make_drop_params(drop_key, p_drop, layer);
  GemmOperand a{u, ldu, false}, b{W1p, ldw, false};
  return finish(launch_gemm_t<false, false, EPI_GEGLU_DROP>(a, b, p, num_sms(), ST(stream)), "gemm_geglu_drop");
}

}  // extern "C"
