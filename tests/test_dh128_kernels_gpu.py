"""GPU: every `dim_head = 128` kernel against float64, through the per-kernel tests of the 64-wide heads (their helpers and bodies take the head
width; same layouts, invariants, sentinels and bound definitions):

- attention.cu's general forward / backward prep / backward at 128 (attn_fwd_k<128>, attn_bwd_prep_k<128> and the split-role attn_bwd_dh_k):
  every ragged layout of tests/test_attention_layer_gpu.py at H = 1, 3, 16 and both long ring sequences at H = 3, 8, with logits
  inside the qk-RMSNorm range (|s / cap| ~ 0.7 from planted q = +-k rows), at gamma = 0, and unnormalised (|s / cap| > 3, the soft cap
  saturated); per-(token, head) row errors against the magnitudes of the summed terms; dv into the packed dqkvg matrix between sentinels,
  dq / dk pre-filled.  Keys and queries that cannot see each other change nothing, bit for bit (64-key backward tiles); cached prefill from
  a slab cache; the LASER / value-residual chain in engine order, and its row kernels one by one (laser_out_fwd_k<128>,
  laser_bwd_prep_k<128>, vmix_fwd_k<128>, vmix_bwd_k<128>).
- decode.cu's attn_decode_dh_k<128>: every fill length, out-of-order slabs, NaN past the visible keys, padded pitches, saturated and LASER.
- the QKVG d128 epilogues (qk-RMSNorm and RoPE-only) in both GEMM cluster modes, with and without the mix rows, the kv-cache append of prefill
  and of a decode step, guard rows; qk_bwd_pack_d128 / _rope_d128 (qk_bwd_pack_k<128, true> / <128, false>).

Bounds: the attention bounds are TOL_D128 in tests/test_attention_layer_gpu.py (about 3x the worst error measured over this file, measured
value beside each); the decode and GEMM-epilogue bounds are the first-principles bounds of their 64-wide tests with the head width put in.
Run with -s to print the worst error (attention) and worst err / bound (the others) of every check."""
import pytest
import torch

import test_attention_layer_gpu as att
import test_block_epilogues_gpu as epi
import test_decode_kernels_gpu as dec
import test_noqknorm_gpu as nqk
from helpers import cluster_mode, gen  # noqa: F401  (cluster_mode: a fixture)
from test_ops_gpu import make_rb
from transfusion_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DH = 128
CAP = att.CAP
# gamma0: |s / cap| <= 0.23; inside: 0.70 (the planted q = +-k rows), as a qk-RMSNorm model with gamma = 0.76 gives; unnormed: q, k = 4 x,
# |s / cap| up to ~3.6 (qk_rmsnorm = False)
GAMMAS = {'gamma0': 0.0, 'inside': att.INSIDE[DH], 'unnormed': None}
# (model dim, heads, learned value residual) of the QKVG tests: odd H, H = 16, D = 2048, HI both above and below D
QKVG = [(128, 1, False), (256, 2, True), (512, 3, True), (384, 5, False), (768, 8, True), (1024, 11, False), (1536, 15, True), (2048, 16, True)]
QKVG_IDS = [f'd{d}h{h}' + ('mix' if m else '') for d, h, m in QKVG]


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


@pytest.fixture(scope = 'module', autouse = True)
def _report():
    yield
    for (dh, name), e in sorted(att.WORST.items()):
        if dh == DH:
            print(f'worst over the file: attention {name:20s} {e:.3g} (bound {att.TOL_D128[name]:.2g})')
    for shown in (dec.SHOWN, epi.SHOWN, nqk.SHOWN):
        for name, r in sorted(shown.items()):
            print(f'worst over the file: {name:40s} err / bound {r:.3g}')


# ================================================================================================ attention vs float64
def general_vs_fp64(ops, lens, spans, H, gamma, seed):
    """the general kernels at 128 (the only attention a 128-wide model runs) against float64 autograd"""
    rb = make_rb(lens, spans)
    M, T = rb.M, att.tables(rb)
    g = gen(seed)
    q, k = att.qk_inputs(rb.cu, H, gamma, g, DH)
    y = (q.double() * k.double()).reshape(M, H, DH).sum(-1) * DH ** -0.5 / CAP
    if gamma is None:
        assert y.max().item() > 3 and y.min().item() < -3
    elif gamma > 0:
        assert 0.69 < y.max().item() < 0.72 and -0.72 < y.min().item() < -0.69
    v = (torch.randn(M, H * DH, device = 'cuda', generator = g) * 2).to(BF16)
    gates = torch.randn(M, H, device = 'cuda', generator = g) if H > 1 else None
    dog = torch.randn(M, H * DH, device = 'cuda', generator = g).to(BF16)
    out = att.attention_pass(ops, T, q, k, v, gates, dog, H, None, dh = DH)
    ref = att.reference(q, k, v, gates, dog, T['kv_limit'], att.seqs_of(rb), H, DH)
    mag = ref['mag']
    att.check('o', att.row_err(out['o'], ref['o'], H, DH, mag = mag['o']), DH)
    att.check('lse', att.lse_err(out['lse'], ref['lse']), DH)
    for name in ('dq', 'dk', 'dv'):
        att.check(name, att.row_err(out[name], ref[name], H, DH, mag = mag[name]), DH)
    if gates is not None:
        att.check('dgate', att.row_err((1 - torch.sigmoid(gates)) * out['dsum_mh'], ref['dgate'], H, 1, mag = mag['dgate']), DH)


@pytest.mark.parametrize('gamma', list(GAMMAS), ids = list(GAMMAS))
@pytest.mark.parametrize('H', [1, 3, 16])
@pytest.mark.parametrize('layout', list(att.LAYOUTS))
def test_attention_vs_fp64(ops, layout, H, gamma):
    general_vs_fp64(ops, *att.LAYOUTS[layout], H, GAMMAS[gamma], seed = 20 + H)


@pytest.mark.parametrize('gamma', list(GAMMAS), ids = list(GAMMAS))
@pytest.mark.parametrize('H', [3, 8])
@pytest.mark.parametrize('layout', list(att.RINGS))
def test_attention_vs_fp64_long_sequences(ops, layout, H, gamma):
    """up to 64 query steps of the backward's double-buffered Q / dO loop per key tile"""
    general_vs_fp64(ops, *att.RINGS[layout], H, GAMMAS[gamma], seed = 30 + H)


@pytest.mark.parametrize('H', [3, 16])
def test_invisible_keys_do_not_matter(ops, H):
    att.test_invisible_keys_do_not_matter(ops, H, dh = DH)


@pytest.mark.parametrize('H', [3, 16])
def test_invisible_queries_do_not_matter(ops, H):
    att.test_invisible_queries_do_not_matter(ops, H, dh = DH)


@pytest.mark.parametrize('H', [3, 16])
def test_cached_prefill_vs_fp64(ops, H):
    att.test_cached_prefill_vs_fp64(ops, H, dh = DH)


@pytest.mark.parametrize('laser', [True, False], ids = ['laser', 'plain'])
@pytest.mark.parametrize('H', [3, 16])
def test_layer_chain_vs_fp64(ops, H, laser):
    att.test_layer_chain_vs_fp64(ops, H, laser, dh = DH)


# ================================================================================================ LASER / value-residual row kernels
@pytest.mark.parametrize('clamp', [15., 5.])
@pytest.mark.parametrize('H', [1, 3, 16])
def test_laser_v_fwd_vs_fp64(ops, H, clamp):
    att.test_laser_v_fwd_vs_fp64(ops, H, clamp, dh = DH)


@pytest.mark.parametrize('gated', [True, False])
@pytest.mark.parametrize('H', [1, 3, 16])
def test_laser_out_fwd_vs_fp64(ops, H, gated):
    att.test_laser_out_fwd_vs_fp64(ops, H, gated, dh = DH)


@pytest.mark.parametrize('H', [1, 3, 16])
def test_laser_bwd_prep_vs_fp64(ops, H):
    att.test_laser_bwd_prep_vs_fp64(ops, H, dh = DH)


@pytest.mark.parametrize('H', [1, 3, 16])
def test_laser_v_bwd_vs_fp64(ops, H):
    att.test_laser_v_bwd_vs_fp64(ops, H, dh = DH)


@pytest.mark.parametrize('H', [1, 3, 16])
def test_vmix_fwd_vs_fp64(ops, H):
    att.test_vmix_fwd_vs_fp64(ops, H, dh = DH)


@pytest.mark.parametrize('H', [1, 3, 16])
def test_vmix_bwd_vs_fp64(ops, H):
    att.test_vmix_bwd_vs_fp64(ops, H, dh = DH)


# ================================================================================================ decode attention
@pytest.mark.parametrize('case', ['gated', 'laser', 'saturated'])
@pytest.mark.parametrize('H', [1, 3, 8, 16])
def test_attn_decode_vs_fp64(ops, H, case):
    dec.test_attn_decode_vs_fp64(ops, H, case, dh = DH)


# ================================================================================================ QKVG epilogues and their backward
@pytest.mark.parametrize('D,H,mix', QKVG, ids = QKVG_IDS)
def test_gemm_qkvg_vs_float64(ops, cluster_mode, D, H, mix):
    epi.test_gemm_qkvg_vs_float64(ops, cluster_mode, D, H, mix, dh = DH)


@pytest.mark.parametrize('D,H,mix', QKVG, ids = QKVG_IDS)
def test_qk_bwd_pack_vs_float64(ops, D, H, mix):
    epi.test_qk_bwd_pack_vs_float64(ops, D, H, mix, dh = DH)


@pytest.mark.xfail(strict = True, reason = 'as at dim_head 64 (tests/test_block_epilogues_gpu.py): where gamma_j = -1 the forward wrote y_j = 0, so '
                                          'qk_bwd_pack_d128 cannot rebuild xhat_j and returns dx_j = 0 and dgamma_j = 0')
def test_qk_bwd_pack_at_gamma_minus_one(ops):
    epi.test_qk_bwd_pack_at_gamma_minus_one(ops, dh = DH)


@pytest.mark.parametrize('H', [1, 3, 8, 16])
def test_gemm_qkvg_rope_vs_float64(ops, cluster_mode, H):
    nqk.test_gemm_qkvg_rope_vs_float64(ops, H, dh = DH)


@pytest.mark.parametrize('H', [1, 3, 8, 16])
def test_qk_bwd_pack_rope_vs_float64(ops, H):
    nqk.test_qk_bwd_pack_rope_vs_float64(ops, H, dh = DH)
