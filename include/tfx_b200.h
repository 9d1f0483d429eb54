/* tfx_b200.h - C ABI of the CUDA-native Transfusion hot path (libtfx_b200.so, sm_90a / H100 only).
 *
 * The reference (lucidrains/transfusion-pytorch) has no FFI: its hot path is ATen calls inside
 * transfusion_pytorch/transfusion.py ("T.py") and modality_processing.py ("MP.py").  Each entry
 * point below replaces the ATen call sites cited beside it; the Python host in
 * transfusion_pytorch_b200/ binds them with ctypes (see INTEGRATION.md for the stub a maintainer of
 * the reference would add).
 *
 * Conventions: plain device pointers (no torch types), explicit sizes and row pitches in ELEMENTS,
 * `stream` is a cudaStream_t passed as void*, every call is asynchronous on that stream, allocates
 * nothing, and returns 0 or a negative code with the message in tfx_last_error() (thread-local).
 * bf16 buffers are passed as void*.  "M" is the number of packed tokens of the ragged batch.
 */
#ifndef TFX_B200_H
#define TFX_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define TFX_B200_VERSION 200

/* Deepest model the AttentionResidual kernels take: hidden-state lists hold x0 plus TFX_MAX_DEPTH layer outputs.  Transformer(...) rejects deeper
 * models with the same number (transfusion.py MAX_DEPTH). */
#define TFX_MAX_DEPTH 64

const char* tfx_last_error(void);
int tfx_version(void);
int tfx_init(int device);                       /* checks the device is sm_90 */

/* ---------------------------------------------------------------- wgmma GEMM family
 * D[m][n] = sum_k A(m,k) B(n,k); operands bf16, fp32 accumulation.
 * x_mn_major = 0: operand stored [MN][K] (row pitch ld); 1: stored [K][MN].                      */

/* CTA pairing of the GEMM family (clusters of 2 CTAs computing vertically adjacent tiles; each loads half of the shared B tile and multicasts it
 * to both): 1 = never (default), 2 = every launch, 3 = launches with K >= 1024 per work item and at least two tiles per SM.  Also read once from
 * the environment (TFX_GEMM_CLUSTER).  No reference counterpart: a tuning knob of this library.   */
int tfx_gemm_set_cluster_mode(int mode);

/* Tile of tfx_gemm_store: 1 = 256 x 128 cooperative tile for launches with at least 16 k-blocks (K / 64 / splits) per work item and CTA pairing
 * off, else 128 x 128 ping-pong (default); 2 = always the 256 x 128 tile; 3 = never.  Both compute bit-identical outputs; this is for tests and
 * benchmarks that compare them.  No reference counterpart. */
int tfx_gemm_set_wide_mode(int mode);

/* Launch geometry tfx_gemm_store would use for these arguments under the current modes: geometry[0] work items (tiles x splits),
 * [1] k-blocks (64 deep) per item, [2] tile rows (128 or 256), [3] split-K factor after clamping.  Launches nothing.  No reference counterpart. */
int tfx_gemm_store_items(int M, int N, int K, int a_mn_major, int b_mn_major, int k_splits, int* geometry);

/* generic: out = alpha*acc + bias[n]  -> fp32 (store / atomic accumulate, optional per-row offsets) and/or bf16.
 * Replaces nn.Linear call sites with no fused tail: to_time_cond Linear (T.py:1070,1132), to_film /
 * to_ada_ln_zero evaluated per distinct time (T.py:700,712,749,767), to_text_logits (T.py:3280,2640),
 * model_to_latent (T.py:3302), latent_to_model (MP.py:667), and every dgrad / wgrad product of autograd. */
int tfx_gemm_store(const void* A, long long lda, int a_mn_major, const void* B, long long ldb, int b_mn_major, int M, int N, int K,
                   float* out_f32, long long ld_f32, void* out_bf16, long long ld_bf16, const float* bias, const long long* row_off,
                   float alpha, int accumulate, int k_splits, void* stream);

/* to_qk | to_v | to_gates in one GEMM (W packed [3*H*64 + 128][D]: q rows, k rows, v rows, gate rows, zero pad) with the
 * per-head qk-RMSNorm and interleaved-pair RoPE applied in the epilogue.  T.py:946 (to_qk, to_v), 950-952
 * (q_norm, k_norm), 964-965 (apply_rotary_emb), 1027 (to_gates).  Outputs q,k (post-RoPE), v: bf16 [M][H*64];
 * gates fp32 [M][H] (logits); qk_inv fp32 [M][2H] (saved 1/|x| for backward).
 * kv_rows (optional, [M]): in-place kv-cache append - token m's post-RoPE key and its value are written to ROW kv_rows[m] of k / v, which
 * then point at one layer of the slab cache (replaces the cat / pad / stack of T.py:969-977, 2257-2277); q stays dense.
 * mix_pre (optional, fp32 [M][H], any accepted H): rows [3*H*64 + H, 3*H*64 + 2H) of W hold `to_learned_value_residual` (T.py:894-898); their
 * products are written here (pre-bias, pre-sigmoid).
 * gates may be null (`Attention(gate_values = False)`, T.py:901-904, 1026-1027): no gate logits are written.  The 128 rows behind to_v (the gate
 * tile: gate rows, mix rows, zero pad) exist iff gates or mix_pre is given: then W is [3*H*64 + 128][D] as above, otherwise [3*H*64][D] and the
 * GEMM computes no gate tile. */
int tfx_gemm_qkvg(const void* u, long long ldu, const void* W, long long ldw, int M, int H, int D, void* q, void* k, void* v, float* gates, float* qk_inv,
                  const float* q_gamma, const float* k_gamma, const int* rope_pos, const float* rope_cs_t /* [32][rope_len][2], see tfx_rope_table */, int rope_len,
                  const int* kv_rows, float* mix_pre, void* stream);

/* the same GEMM for `qk_rmsnorm = False` (T.py:949-951 skipped): q, k = RoPE(u W^T) with no norm, so no qk_inv and no gammas; v, gates,
 * mix_pre and the kv_rows append are those of tfx_gemm_qkvg (same accumulators, bit for bit). */
int tfx_gemm_qkvg_rope(const void* u, long long ldu, const void* W, long long ldw, int M, int H, int D, void* q, void* k, void* v, float* gates,
                       const int* rope_pos, const float* rope_cs_t, int rope_len, const int* kv_rows, float* mix_pre, void* stream);
/* dim_head = 128 forms of the two: W = [to_qk | to_v | gate tile], N = 3*H*128 + 128 (3*H*128 without gates and mix_pre, as above), one head per
 * 128-column tile, so 1 <= H <= 16 (odd H too).
 * The qk-RMSNorm spans the head's 128 columns (scale sqrt(128)); RoPE takes 64 frequency pairs: rope_cs_t is [64][rope_len][2] (tfx_rope_table, n_freqs 64);
 * qk_inv is [M][2H] as above; q, k, v are [M][H*128]; gates are rows [3*H*128, +H) of W as in the 64-wide forms, the mix_pre rows start at the next
 * even row, 3*H*128 + H rounded up to even (so that an odd H keeps the bf16 pairs of their gradient 4-byte aligned). */
int tfx_gemm_qkvg_d128(const void* u, long long ldu, const void* W, long long ldw, int M, int H, int D, void* q, void* k, void* v, float* gates, float* qk_inv,
                       const float* q_gamma, const float* k_gamma, const int* rope_pos, const float* rope_cs_t, int rope_len, const int* kv_rows, float* mix_pre, void* stream);
int tfx_gemm_qkvg_rope_d128(const void* u, long long ldu, const void* W, long long ldw, int M, int H, int D, void* q, void* k, void* v, float* gates,
                            const int* rope_pos, const float* rope_cs_t, int rope_len, const int* kv_rows, float* mix_pre, void* stream);

/* branch output projection + AdaptiveWrapper output gate + residual:
 *   y = [A | A2] W^T + bias ;  x_out = x_res + y * (cond_row[m] >= 0 ? zgate[cond_row[m]] : layerscale + 1)
 * to_out (T.py:1031) / FeedForward net.3 (T.py:849) with T.py:765-769 and the residual adds T.py:1238,1242;
 * with A2 != NULL and no gate it is skip_proj on cat(x, skip) (T.py:1217-1219) without materialising the concat. */
int tfx_gemm_resid(const void* A, long long lda, const void* A2, long long lda2, int K1, const void* W, long long ldw, int M, int N, int K, const float* bias,
                   const float* x_res, float* x_out, void* x_out_bf16, void* y_bf16, const int* cond_row, const float* zgate, long long zgate_ld,
                   const float* layerscale, void* stream);

/* FeedForward net.0 + GEGLU (T.py:833-834, 846-847): W1 packed so every 128-column tile is [64 value | 64 gate];
 * writes the pre-activations vg [M][Np] (saved for backward) and h = gelu_erf(gate)*value [M][Np/2].           */
int tfx_gemm_geglu(const void* u, long long ldu, const void* W1p, long long ldw, const float* b1p, int M, int Np, int K, void* vg, void* h, void* stream);
/* the same with FeedForward dropout (T.py:845-850, nn.Dropout after GEGLU): h = gelu_erf(gate)*value * keep / (1 - p), vg undropped.
 * keep is the counter-based mask of csrc/dropout.cuh (site 1: row = packed token, column = inner column, head 0), drawn from the
 * device key drop_key (2 x u32, read at run time: a captured graph sees the key of each replay); p = 1 drops everything. */
int tfx_gemm_geglu_drop(const void* u, long long ldu, const void* W1p, long long ldw, const float* b1p, int M, int Np, int K, void* vg, void* h,
                        const void* drop_key /* device, 2 x u32 */, float p, int layer, void* stream);

/* ---------------------------------------------------------------- attention (T.py:998-1027, mask T.py:452-470)
 * Flash-style, span mask from kv_limit[m] (last visible key of query m), tanh soft-cap, value gates in the epilogue.
 * Tile tables (host-built, 64-row tiles that never straddle a sequence): forward per query tile, backward per key tile. */
int tfx_attn_fwd(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H,
                 const int* kv_limit, const int* tile_q0, const int* tile_qend, const int* tile_kv0, const int* tile_kvend, int n_tiles,
                 void* o, long long ld_o, float* lse, int M, float scale, float softcap, const float* skip_if_fast /* optional, see below */, void* stream);
/* Bounded-logit fast path on wgmma / TMA (128-row tiles).  q, k are RMS-normalised (T.py:950-952), so the soft-cap argument is
 * bounded by the two gamma vectors; tfx_attn_fast_params writes params[0] = 1 when |s/cap| <= 0.75 is guaranteed (polynomial tanh on the
 * FMA pipe, fixed softmax maximum params[1], output accumulator never rescaled).  Host code enqueues BOTH tfx_attn_fwd_tc(params) and
 * tfx_attn_fwd(skip_if_fast = params); the kernel whose precondition fails returns at once - no host synchronisation. */
int tfx_attn_fast_params(const float* q_gamma, const float* k_gamma, int dim_head, float scale, float softcap, float* params /* [>=2] device */, void* stream);
int tfx_attn_fwd_tc(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H,
                    const int* kv_limit, const int* tile_q0, const int* tile_qend, const int* tile_kv0, const int* tile_kvend, int n_tiles,
                    void* o, long long ld_o, float* lse, int M, int M_kv /* rows of k / v when they are a kv cache (T.py:969-972); 0 = M */, float scale, float softcap,
                    const float* fast_params, void* stream);
/* dq_zero (optional): fp32 [M][H*64] accumulator of tfx_attn_bwd, cleared here in the same pass */
int tfx_attn_bwd_prep(const void* do_gated, const void* o_gated, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero, int M, int H, void* stream);
int tfx_attn_bwd(const void* q, const void* k, const void* v, const void* do_pre, long long ld_q, long long ld_k, long long ld_v, long long ld_do,
                 const float* lse, const float* dsum_hm, const int* kv_limit, const int* kt_kv0, const int* kt_kvend, const int* kt_q0, const int* kt_qend,
                 int n_kv_tiles, float* dq, float* dk, void* dv, long long ld_dv, int M, int H, float scale, float softcap, const float* skip_if_fast /* optional */,
                 void* stream);
/* bounded-logit backward on wgmma: 128-key tiles (k2_* tables), transposed scores, dV / dK accumulated in registers, dQ added with fp32 reductions.
 * Same dual-launch protocol as the forward (fast_params from tfx_attn_fast_params; dq must be zero on entry, see tfx_attn_bwd_prep). */
int tfx_attn_bwd_tc(const void* q, const void* k, const void* v, const void* do_pre, long long ld_q, long long ld_k, long long ld_v, long long ld_do,
                    const float* lse, const float* dsum_hm, const int* kv_limit, const int* kt_kv0, const int* kt_kvend, const int* kt_q0, const int* kt_qend,
                    const int* kt_order /* optional: key-tile indices, most query tiles first (load balance of the persistent grid) */,
                    int n_kv_tiles, float* dq, float* dk, void* dv, long long ld_dv, int M, int H, float scale, float softcap, const float* fast_params, void* stream);
/* dim_head = 128 forms of tfx_attn_fwd / tfx_attn_bwd_prep / tfx_attn_bwd: the same tile tables, span mask, soft-cap, gates and buffer layouts with
 * 128-wide heads ([M][H*128]); no bounded-logit variant exists at this head dim, so there is no skip flag.  dq must be zero on entry of the backward. */
int tfx_attn_fwd_d128(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H,
                      const int* kv_limit, const int* tile_q0, const int* tile_qend, const int* tile_kv0, const int* tile_kvend, int n_tiles,
                      void* o, long long ld_o, float* lse, int M, float scale, float softcap, void* stream);
int tfx_attn_bwd_prep_d128(const void* do_gated, const void* o_gated, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero, int M, int H, void* stream);
int tfx_attn_bwd_d128(const void* q, const void* k, const void* v, const void* do_pre, long long ld_q, long long ld_k, long long ld_v, long long ld_do,
                      const float* lse, const float* dsum_hm, const int* kv_limit, const int* kt_kv0, const int* kt_kvend, const int* kt_q0, const int* kt_qend,
                      int n_kv_tiles, float* dq, float* dk, void* dv, long long ld_dv, int M, int H, float scale, float softcap, void* stream);
/* backward of the qk-RMSNorm + RoPE epilogue; packs d[q | k | (v written by attn_bwd) | gates] bf16 [M][out_ld].  gates null (ungated model):
 * no gate-gradient column is written and dsum_mh is not read (may be null).  The same holds for the three packs below. */
int tfx_qk_bwd_pack(const float* dq, const float* dk, const void* q_bf16, const void* k_bf16, const float* qk_inv, const float* q_gamma, const float* k_gamma,
                    const int* rope_pos, const float* rope_cs, const float* gates, const float* dsum_mh, void* dqkvg_bf16, long long out_ld,
                    float* dq_gamma, float* dk_gamma, int M, int H, void* stream);

/* backward of the RoPE-only epilogue (tfx_gemm_qkvg_rope): d q_pre = R(pos)^T dq, d k_pre = R(pos)^T dk and the gate-logit column of
 * tfx_qk_bwd_pack, packed into the same d[q | k | . | gates] layout */
int tfx_qk_bwd_pack_rope(const float* dq, const float* dk, const int* rope_pos, const float* rope_cs, const float* gates, const float* dsum_mh, void* dqkvg_bf16,
                         long long out_ld, int M, int H, void* stream);
/* dim_head = 128 forms of the two packs (1 <= H <= 16): rope_cs is [rope_len][64][2], the gammas are [128], the norm scale is sqrt(128) */
int tfx_qk_bwd_pack_d128(const float* dq, const float* dk, const void* q_bf16, const void* k_bf16, const float* qk_inv, const float* q_gamma, const float* k_gamma,
                         const int* rope_pos, const float* rope_cs, const float* gates, const float* dsum_mh, void* dqkvg_bf16, long long out_ld,
                         float* dq_gamma, float* dk_gamma, int M, int H, void* stream);
int tfx_qk_bwd_pack_rope_d128(const float* dq, const float* dk, const int* rope_pos, const float* rope_cs, const float* gates, const float* dsum_mh, void* dqkvg_bf16,
                              long long out_ld, int M, int H, void* stream);

/* AttentionResidual backward with DEFERRED assembly (exact; rowops.cu): instead of read-modify-writing the gradient of every earlier hidden at every layer, layer i
 * stores three scalars per (token, hidden) and the complete gradient of ONE hidden is assembled when the backward pass needs it:
 *   G_k = sum_{i' >= k-1} [a_{i',k} dx_{i'} + c1_{i',k} w_{i'}] - (sum c2_{i',k}) h_k,
 * with c2 = 0 on a row shorter than the 1e-12 norm clamp (the clamped norm is a constant for the gradient, as in F.normalize).
 * own = 1: layer with hiddens h_0..h_{n-1}; writes the scalars of h_0..h_{n-2} to scalars_out[token][k][3] (row stride scalar_stride floats), the parameter gradients,
 * and grad_hidden = G_{n-1} from its own term plus the n_later later layers (dx_later[j], scalars_later[j] -> element [token 0][k = n-1][0], gammas / pseudo_queries[1 + j]).
 * own = 0: assembly only (gammas[0] / pseudo_queries[0] unused): the gradient of h_0 after the first layer.
 * 1 <= n_hiddens <= TFX_MAX_DEPTH + 1, 0 <= n_later <= TFX_MAX_DEPTH.  Up to 10 later layers take one launch (plus the parameter-gradient fold when own = 1);
 * more are assembled in chunks of 10: each further launch adds its chunk's sum_j [a_j dx_j + c1_j w_j] - (sum_j c2_j) h into grad_hidden. */
int tfx_attn_residual_bwd2(const void* const* hiddens_bf16, int n_hiddens, int own, const float* const* gammas, const float* const* pseudo_queries,
                           const float* const* dx_later, const float* const* scalars_later, int n_later, const float* dx_out, const float* x_out, const float* lse,
                           float* grad_hidden, float* scalars_out, int scalar_stride, float* dgamma, float* dpseudo_query, float* workspace, int M, int D, void* stream);

/* ---------------------------------------------------------------- optional attention variants (attn_variants.cu), HBM-bound row kernels
 * LASER (T.py:981-983, 1021-1022): v' = exp(c tanh(v / c)) before the attention, att = log(o') * sigmoid(gate) after it; `rows` (optional) maps token m to its
 * kv-cache row (raw values stay in the cache, T.py:976-977; the transformed copy is a second slab).  Backward: tfx_laser_bwd_prep replaces tfx_attn_bwd_prep
 * (dO' = dAtt sg / o', D = sum_d dAtt sg, gate sums = sum_d dAtt att), tfx_laser_v_bwd turns dv' into dv in place. */
int tfx_laser_v_fwd(const void* v, long long ld_v, const int* rows, void* v_laser, long long ld_vl, int M, int H, float clamp, void* stream);
int tfx_laser_out_fwd(const void* o_laser, const float* gates, void* att, int M, int H, void* stream);
int tfx_laser_bwd_prep(const void* d_att, const void* o_laser, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero, int M, int H, void* stream);
int tfx_laser_v_bwd(void* dv_inout, long long ld_dv, const void* v, long long ld_v, int M, int H, float clamp, void* stream);
/* learned value residual (T.py:956-960, 1234): v = v mix + v_first (1 - mix), mix = sigmoid(mix_pre + bias) per token and head, in place (also on cache rows).
 * Backward (dv_inout: d v_mixed -> d v_raw): dv_first_acc (fp32 [M][H*64]) += d v_mixed (1 - mix); d mix_pre -> bf16 column block of the packed dqkvg matrix. */
int tfx_vmix_fwd(void* v_inout, long long ld_v, const int* rows, const void* v_first, long long ld_v0, const float* mix_pre, const float* mix_bias, int M, int H, void* stream);
int tfx_vmix_bwd(void* dv_inout, long long ld_dv, const void* v_mixed, long long ld_v, const void* v_first, long long ld_v0, const float* mix_pre, const float* mix_bias,
                 float* dv_first_acc, void* dmix_bf16, long long ld_dmix, int M, int H, void* stream);
int tfx_add_f32_into_bf16(void* dst_bf16, long long ld_dst, const float* src, long long ld_src, int M, int N, void* stream);
/* dim_head = 128 forms of the per-head row kernels (heads of 128 columns).  tfx_laser_v_fwd / tfx_laser_v_bwd are elementwise: at dim_head = 128 they
 * are called with 2H 64-wide heads. */
int tfx_laser_out_fwd_d128(const void* o_laser, const float* gates, void* att, int M, int H, void* stream);
int tfx_laser_bwd_prep_d128(const void* d_att, const void* o_laser, const float* gates, void* do_pre, float* dsum_hm, float* dsum_mh, float* dq_zero, int M, int H, void* stream);
int tfx_vmix_fwd_d128(void* v_inout, long long ld_v, const int* rows, const void* v_first, long long ld_v0, const float* mix_pre, const float* mix_bias, int M, int H, void* stream);
int tfx_vmix_bwd_d128(void* dv_inout, long long ld_dv, const void* v_mixed, long long ld_v, const void* v_first, long long ld_v0, const float* mix_pre, const float* mix_bias,
                      float* dv_first_acc, void* dmix_bf16, long long ld_dmix, int M, int H, void* stream);

/* ---------------------------------------------------------------- warp-per-token kernels (D = model dim: 128, 256, 384, 512, 768 or 1024)
 * AdaptiveWrapper input side (T.py:747-755, text-only 677-679): u = isM ? LN(x)(gamma_c+1)+beta_c : LN(x)(g+1).
 * film points at [n_cond][film_ld] with gamma at +0 and beta at +D; cond_row NULL = all text.      */
int tfx_adaln_fwd(const float* x, const int* cond_row, const float* film, long long film_ld, const float* ln_gamma,
                  void* u_bf16, float* stats, int M, int D, void* stream);
int tfx_adaln_bwd(const float* du, const float* x, const float* stats, const int* cond_row, const float* film, long long film_ld,
                  const float* ln_gamma, float* dx_accum, float* dfilm, long long dfilm_ld, float* dln_gamma, int M, int D, void* stream);
/* backward of the output gate of tfx_gemm_resid: dy = dx*scale (bf16), d zgate / d layerscale accumulated;
 * dbias (optional, [D]) += column sums of dy (gradient of the bias of the producing Linear, T.py:849) */
int tfx_resid_bwd(const float* dx, const void* y_bf16, const int* cond_row, const float* zgate, long long zgate_ld, const float* layerscale,
                  void* dy_bf16, float* dzgate, long long dzgate_ld, float* dlayerscale, float* dbias, int M, int D, void* stream);
/* AttentionResidual forward (T.py:803-829): softmax mix over all hiddens so far, single pass.  The hiddens are bf16 (the layer outputs are kept
 * in bf16 only: reading them is the largest HBM term of the step); x_out fp32, x_out_bf16 (optional) its bf16 copy.  lse_out [M] (optional) =
 * log-sum-exp of the depth softmax, consumed by the backward (tfx_attn_residual_bwd2) together with x_out so that every hidden is read once per layer.
 * 1 <= n_hiddens <= TFX_MAX_DEPTH + 1. */
int tfx_attn_residual_fwd_h16(const void* const* hiddens_bf16, int n_hiddens, const float* gamma, const float* pseudo_query,
                              float* x_out, void* x_out_bf16, float* lse_out, int M, int D, void* stream);
long long tfx_attn_residual_bwd_workspace_floats(int M, int D);   /* fp32 scratch of tfx_attn_residual_bwd2 for the per-block parameter-gradient partial sums */
/* final RMSNorm (T.py:1250, 785-786) (+ compaction of modality rows for the flow head) */
int tfx_rmsnorm_fwd(const float* x, const float* gamma, float* out_f32, void* out_bf16, const int* slot, void* out_mod_bf16, int M, int D, void* stream);
int tfx_rmsnorm_bwd(const float* dout, const float* x, const float* gamma, float* dx, float* dgamma, int M, int D, void* stream);
/* Self-Flow representation loss (T.py:3458-3460): loss = 1 - mean over the M rows of cosine_similarity(a_r, b_r), norms clamped to 1e-8 each
 * (torch.nn.functional.cosine_similarity), written to `loss` (float, device); in the same pass da = d(g * loss)/da in bf16, g a device scalar,
 * the mean taken over n_mean rows.  a fp32 [M][D]; b [M][D], bf16 if b_bf16 else fp32.  partials: tfx_rep_cos_blocks(M) doubles; ticket: one
 * zero-initialised u32 the kernel leaves at zero.  The sum is deterministic for a given M and GPU. */
int tfx_rep_cos_blocks(int M);
int tfx_rep_cos_fwd_bwd(const float* a, const void* b, int b_bf16, const float* g, int n_mean, void* da_bf16, double* partials, unsigned int* ticket, float* loss,
                        int M, int D, void* stream);
/* token assemble: where(is_modality, modality_token, text_embed[id]) (T.py:3173-3184) and its backward */
int tfx_embed_assemble(const int* text_id, const float* emb, const float* modtok, const int* slot, float* x0, void* x0_bf16, int M, int D, void* stream);
int tfx_embed_bwd(const float* dx0, const int* text_id, const int* slot, float* demb, void* dmodtok_bf16, int M, int D, void* stream);
/* model_output_clean (MP.py:100-126, 790-793; T.py:2454-2455): omod[s] = (out[row_token[s]] - modtok[s]) / max(1 - t, eps), t = cond_times[cond_row[token]];
 * backward: dmod *= 1 / max(1 - t, eps) in place (then scattered into d out), dmodtok_neg = -dmod (added to the modality-token gradient) */
int tfx_clean_flow_fwd(const float* out, const int* row_token, const float* modtok, const float* cond_times, const int* cond_row, float eps, void* omod_bf16, int S, int D, void* stream);
int tfx_clean_flow_bwd(float* dmod_inout, float* dmodtok_neg, const int* row_token, const float* cond_times, const int* cond_row, float eps, int S, int D, void* stream);
int tfx_scatter_add_rows(float* dst, const float* src, const int* row_map, int S, int D, void* stream);

/* ---------------------------------------------------------------- elementwise / reductions
 * flow-match noise inject (MP.py:645-656): noised = x t + eps (1-t) ; flow = x - eps.  eps NULL = plain cast. */
int tfx_flow_noise(const float* x, const float* eps, const float* t_row, void* noised_bf16, long long ld_noised, float* noised_f32, float* flow, long long S, int dl, void* stream);
/* RandomFourierEmbed (T.py:625-635): [t, sin(2 pi t w), cos(2 pi t w)] zero padded to ld */
int tfx_time_features(const float* times, const float* fourier_w, void* feats_bf16, int n, int half_dim, int ld, void* stream);
/* small table ops of the conditioning path: op 0 sigmoid(a), 1 silu(a), 2 a*b*(1-b), 3 a*silu'(b), 4 copy */
int tfx_table_op(const float* a, long long ld_a, const float* b, long long ld_b, float* out_f32, long long ld_of, void* out_bf16, long long ld_ob, long long rows, int cols,
                 int op, void* stream);
/* GEGLU backward on the tile-interleaved layout.  Bias gradient (column sums of dvg, T.py:845): either `partials`
 * [ceil(M / tfx_geglu_bwd_rows_per_block())][2*inner_pad] fp32 receives per-block partial sums (reduce with tfx_colsum_f32 + col_map -
 * preferred: ~1000 blocks adding to the same addresses serialise in the L2 atomic units), or, if partials is NULL, dbias[col_map[c]] is
 * updated with atomics directly. */
int tfx_geglu_bwd_rows_per_block(void);
int tfx_geglu_bwd(const void* dh_bf16, const void* vg_bf16, void* dvg_bf16, long long M, int inner_pad, const int* col_map, float* dbias, float* partials, void* stream);
/* the same after tfx_gemm_geglu_drop: dh is multiplied by the regenerated mask and 1 / (1 - p) first */
int tfx_geglu_bwd_drop(const void* dh_bf16, const void* vg_bf16, void* dvg_bf16, long long M, int inner_pad, const int* col_map, float* dbias, float* partials,
                       const void* drop_key /* device, 2 x u32 */, float p, int layer, void* stream);
/* text cross-entropy fwd+bwd (T.py:3320-3331; text-only 2653-2659 with vlimit = num_text_tokens) */
int tfx_ce_fwd_bwd(const float* logits, long long ld_logits, const int* labels, int V, int vlimit, float gscale, void* dlogits_bf16, long long ld_dlogits,
                   double* loss_sum, int* n_valid, int M, void* stream);
/* flow MSE fwd+bwd (T.py:3354-3362) */
int tfx_mse_fwd_bwd(const float* pred, long long ld_pred, const float* flow, void* dpred_bf16, long long ld_dpred, float gscale, double* sumsq, long long S, int dl, void* stream);
/* the same with the per-instance reconstruction loss folded into dpred (replaces the recon closures of MP.py:177-194 evaluated per instance at
   T.py:3299-3308 and averaged per type at T.py:3420-3431; forward_modality: T.py:2836-2856).  Per row: d = pred - target, r = a pred - b g with
   a = 1 - t_row, b = t_row (b_is_t) or 1; dpred = gscale d + rscale inst_w[i] a r (bf16), sumsq += d^2, inst_sumsq[i] += r^2,
   type_sum += inst_w[i] r^2, i = row_inst[row].  All per-instance data is on the device (CUDA-graph replay across instance splits).
   rscale = 0 writes exactly the dpred of tfx_mse_fwd_bwd. */
int tfx_mse_recon_fwd_bwd(const float* pred, long long ld_pred, const float* target, const float* g, const float* t_row, int b_is_t, const int* row_inst,
                          const float* inst_w, void* dpred_bf16, long long ld_dpred, float gscale, float rscale, double* sumsq, double* inst_sumsq, double* type_sum,
                          long long S, int dl, void* stream);
int tfx_colsum_bf16(const void* in_bf16, long long ld, long long M, int N, const int* col_map, float* out, void* stream);
int tfx_colsum_f32(const float* in, long long ld, long long M, int N, const int* col_map /* optional */, float* out, void* stream);
/* all per-optimizer-step weight repacks in one launch; jobs / block tables live in device memory (built once by the host) */
typedef struct TfxPackJob {
  const float* src; long long ld_src; const int* row_src /* optional row gather, -1 = zero row */; void* dst /* bf16, or fp32 if dst_f32 */;
  long long R_dst; int C_src; int C_dst; int dst_f32; int pad_;
} TfxPackJob;
int tfx_cast_pack_multi(const TfxPackJob* jobs_dev, const int* blk_job_dev, const int* blk_first_dev, int n_blocks, void* stream);
int tfx_cast_bf16(const float* src, void* dst_bf16, long long n, void* stream);
int tfx_scale_bf16(void* p_bf16, const float* scale_ptr, long long n, void* stream);          /* p *= *scale_ptr (device scalar) */
int tfx_axpy_f32(float* y, const float* x, float a, long long n, void* stream);   /* y += a*x */
/* cos_sin [max_pos][n_freqs][2]; cos_sin_t (optional) the same table stored [n_freqs][max_pos][2] (coalesced reads for thread-per-row epilogues) */
int tfx_rope_table(const float* freqs, float* cos_sin, float* cos_sin_t, int max_pos, int n_freqs, void* stream);
/* fused Adam / AdamW over the flat parameter buffer (the optimizer the reference's examples use, train_latent_with_text.py:142-153) */
int tfx_adam_step(float* params, float* grads, float* exp_avg, float* exp_avg_sq, long long n, float lr, float beta1, float beta2, float eps, float weight_decay,
                  int decoupled_wd, int step, float grad_scale, int zero_grads /* 1: clear grads in the same pass */,
                  int* step_dev /* optional device-resident step counter (incremented here; bias corrections computed on the device - CUDA-graph safe) */,
                  void* stream);

/* global-norm gradient clipping with torch.nn.utils.clip_grad_norm_ semantics (train_latent_with_text.py:142-153): accumulate the squared
 * norm of the flat gradient buffer into *sumsq_accum (caller zeroes it), then scale by min(1, max_norm / (pre_scale*sqrt(sumsq) + 1e-6));
 * pre_scale = 1 / world_size when the buffer holds the all-reduced SUM.  No host synchronisation. */
int tfx_grad_sumsq(const float* grads, long long n, double* sumsq_accum, void* stream);
int tfx_clip_by_norm(float* grads, long long n, const double* sumsq, float max_norm, float pre_scale, void* stream);
/* EMA copy of the flat parameter buffer (ema_pytorch update, T.py:1687-1697): ema = decay*ema + (1-decay)*params */
int tfx_ema_update(float* ema, const float* params, long long n, float decay, void* stream);

/* ---------------------------------------------------------------- kv-cache sampler (sample_many T.py:2079-2583, generate_text_only T.py:2669-2707)
 * Cache layout: per layer one K and one V matrix bf16 [n_slabs * cap][H*64]; sample s owns rows [(slab0+s)*cap, (slab0+s+1)*cap).  Appends are
 * in place (tfx_gemm_qkvg kv_rows) - this replaces the per-step pad / cat of T.py:2257-2277, 2323-2327, 2531-2533 - and visibility is
 * (slab start, filled length) per sample instead of the Bool[g, Lq, L+Lq] masks of T.py:2300-2304, 2415-2431.
 * Sampler state: int32 [6][S] = len (committed cache rows), tokens_seen (next RoPE position, T.py:2332), last_token, phase (0 text, 1 waiting for
 * the modality phase, 2 done), num_tokens, hist_len;  hist int32 [S][hist_cap] = every sampled token;  counters int32 [2] = {samples still in the
 * text phase after the last step, step number}. */

/* per-token metadata of the next text step from the sampler state: token s = (last_token[s], RoPE position tokens_seen[s]) is appended at row
 * len[s] of its slab and attends rows [0, len[s]] (step_text, T.py:2279-2310).  One single-row attention tile per sample. */
int tfx_decode_prep(const int* state, int S, int cap, int slab0, int* text_id, int* rope_pos, int* kv_row, int* kv_limit, int* tile_q0, int* tile_qend, int* tile_kv0,
                    int* tile_kvend, int* counters, void* stream);
/* decode attention: every tile holds ONE query row (T.py:998-1027 with the cache concat of T.py:969-972): keys / values are rows
 * [tile_kv0, min(tile_kvend, kv_limit[row]+1)) of the cache; soft-cap, softmax, value gate as tfx_attn_fwd. */
int tfx_attn_decode(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H, const int* kv_limit,
                    const int* tile_q0, const int* tile_kv0, const int* tile_kvend, int n_tiles, void* o, long long ld_o, float scale, float softcap, void* stream);
/* the same at dim_head = 128 (q, k, v, o rows of H*128) */
int tfx_attn_decode_d128(const void* q, const void* k, const void* v, long long ld_q, long long ld_k, long long ld_v, const float* gates, int H, const int* kv_limit,
                         const int* tile_q0, const int* tile_kv0, const int* tile_kvend, int n_tiles, void* o, long long ld_o, float scale, float softcap, void* stream);
/* token sampling + state update for every sample in the text phase (sample_text_token T.py:580-591; greedy / gumbel of generate_text_only
 * T.py:2692-2698 with vlimit = num_text_tokens; bookkeeping T.py:2330-2349).  rows (optional): logits row of sample s (first token after the
 * prefill, taken at the last prompt position, T.py:2225-2250: advance = 0 - that token only gets its cache row on the next step).
 * Tempered draw of sample s: argmax over the kept ids c of logit / T - log(-log u), u = ((h >> 41) + 1/2) 2^-23 with
 * h = mix64(seed ^ mix64((counters[1] << 40) ^ (s << 20) ^ c)) (splitmix64 finaliser; counters NULL: step 0). */
int tfx_sample_tokens(const float* logits, long long ld_logits, const int* rows, int V, int vlimit, int* state, int S, int* hist, int hist_cap, int eos_id, const int* som_ids,
                      int n_som, int max_length, float temperature, float min_p, unsigned long long seed, int* counters, int advance, void* stream);
/* fixed-grid explicit midpoint (torchdiffeq method='midpoint', T.py:1314-1318, 2523-2525) on device state; tab [n_evals][4] = (t, c, h, mode), *idx = the
 * current evaluation.  pre: x_eval (dup copies back to back) = y + c f_prev, cond_times[0..n_cond) = t.  post: f = u + cfg (c - u) (T.py:2521; pred_uncond
 * NULL = no guidance); mode 0: f_prev = f, mode 1: y += h f. */
int tfx_ode_pre(const float* y, const float* f_prev, float* x_eval, long long n, int dup, const float* tab, const int* idx, float* cond_times, int n_cond, void* stream);
int tfx_ode_post(float* y, float* f_prev, const float* pred_cond, const float* pred_uncond, float cfg_scale, long long n, const float* tab, const int* idx, void* stream);
int tfx_counter_inc(int* counter, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFX_B200_H */
