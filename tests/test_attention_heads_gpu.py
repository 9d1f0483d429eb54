"""GPU: the 64-wide attention kernels against float64 at 6 to 32 heads, gated and ungated, through the bodies and helpers of
tests/test_attention_layer_gpu.py (same layouts, launch pattern, sentinels, bounds).  A model takes 64-wide heads at every even count from 2 to
32; that file runs the attention kernels at H = 2 and 8 and the row kernels at 2, 6 and 8.  The counts here are chosen by code path:

- 6 and 30: H % 4 == 2, so the row kernels (4 heads per warp pass) end on a partial pass, after 1 and 7 full ones;
- 16: the last count of the old value-residual limit; 18: the first above it;
- 24: the 1536-wide model;
- 32: the largest count: inner width 2048, the widest dQ tensor map, and [H, M] lse / dsum maps of 32 M rows.

What runs at those counts:
- the bounded-logit fast path (attention_sm90.cu) and the general kernels (attention.cu) with their backward pre-pass, as the engine launches
  them: gated with the gate / mix tile (dqkvg pitch 3 HI + 128), ungated without it (pitch 3 HI), and ungated at 3 HI + 128 as a model with
  the value residual has it; unnormed logits (|s / cap| > 3) on the general kernels alone; the long ring sequences at H = 32;
- the pre-pass of an ungated model (gates = None, no gate-sum buffer) writes what it writes when given one;
- exact head isolation: new q, k, v, dO and gate in one head leave every other head's o, lse, dk, dv and gate sums bit for bit unchanged
  (dq: reduction-order noise only), on both paths; and the invisible-key / invisible-query invariants and cached prefill at H = 30, 32;
- the LASER / value-residual row kernels (attn_variants.cu) at 18, 24, 30 and 32 heads, and the layer chain in engine order at 24 and 32.

Bounds: TOL of tests/test_attention_layer_gpu.py (errors are per (token, head) row and heads are independent, so a larger H moves no
bound).  The worst errors at H = 24 to 32 are those of H = 8 (e.g. o 7.3e-3, dq 1.5e-3, dv 1.0e-2).  The one check that grew with H was the
chain's d mix_pre: its magnitude took |d v_mixed| where the error follows the terms d v_mixed sums, so the worst row grew with the number of
rows (0.078 at H = 8, 0.46 at H = 32).  With that magnitude fixed it is 1.2e-2 at H = 8 and 2.2e-2 at H = 32.  The float64 reference
evaluates at most 8 heads at once (att.HEAD_GROUP).  Run with -s to print the worst error of each check per head count.

Measured on an H100 80GB HBM3 (700 W power limit): peak device memory (torch.cuda.max_memory_allocated) 7.3 GiB; runtime 24 s for the 158
tests, against 21 s for tests/test_attention_layer_gpu.py on the same card."""
import pytest
import torch

import test_attention_layer_gpu as att
from helpers import gen, guarded, same_bits, untouched
from transfusion_pytorch_b200 import _lib
from transfusion_pytorch_b200.transfusion import MAX_HEADS

pytestmark = pytest.mark.gpu
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
INSIDE, OUTSIDE = att.GAMMAS['inside'], att.GAMMAS['outside']
HEADS = (6, 16, 24, 30, 32)
ROW_HEADS = (18, 24, 30, 32)
SHORT = ('mixed4', 'tiles128', 'nine', 'seven', 'random0', 'random1', 'random2', 'random3')

# (H, gamma, gated, dqkvg pad) x layouts of the float64 comparison
CASES = ([(32, 'inside', True, 128, l) for l in att.LAYOUTS] + [(32, 'outside', True, 128, l) for l in att.LAYOUTS]
         + [(32, 'inside', False, 0, l) for l in att.LAYOUTS]
         + [(30, 'inside', True, 128, l) for l in att.LAYOUTS] + [(24, 'inside', False, 0, l) for l in att.LAYOUTS]
         + [(16, 'inside', True, 128, l) for l in SHORT] + [(6, 'inside', False, 128, l) for l in SHORT])
CASE_IDS = [f'h{h}-{gm}-{"gated" if gt else "ungated"}-nq{p}-{l}' for h, gm, gt, p, l in CASES]

WORST = {}                                    # (H, check) -> worst error over the file


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


@pytest.fixture(scope = 'module', autouse = True)
def _report():
    torch.cuda.reset_peak_memory_stats()
    yield
    for (H, name), e in sorted(WORST.items()):
        print(f'worst over the file: H = {H:2d} {name:12s} {e:.3g} (bound {att.TOL[name]:.2g})')
    print(f'peak device memory over the file: {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB')


@pytest.fixture(autouse = True)
def _worst_by_heads(request):
    """att.check keeps the worst error per check name; keep it per head count as well"""
    saved = dict(att.WORST)
    att.WORST.clear()
    yield
    H = request.node.callspec.params.get('H') if hasattr(request.node, 'callspec') else None
    if H is None and hasattr(request.node, 'callspec') and 'case' in request.node.callspec.params:
        H = request.node.callspec.params['case'][0]
    for (dh, name), e in att.WORST.items():
        if dh == 64 and H is not None:
            WORST[H, name] = max(WORST.get((H, name), 0.), e)
    for key, e in saved.items():
        att.WORST[key] = max(att.WORST.get(key, 0.), e)


def test_heads_cover_the_accepted_range():
    assert MAX_HEADS in HEADS and MAX_HEADS in ROW_HEADS
    assert any(h > 16 and h % 4 == 2 for h in HEADS) and any(h > 16 and h % 4 == 2 for h in ROW_HEADS)
    assert all(h % 2 == 0 for h in HEADS + ROW_HEADS)


# ================================================================================================ fast path and general kernels vs float64
@pytest.mark.parametrize('case', CASES, ids = CASE_IDS)
def test_attention_vs_fp64(ops, case):
    H, gamma, gated, pad, layout = case
    att.fast_vs_fp64(ops, *att.LAYOUTS[layout], H, att.GAMMAS[gamma], seed = 20 + H, gated = gated, pad = pad)


@pytest.mark.parametrize('layout', ['two1024', 'seven', 'random1'])
@pytest.mark.parametrize('H', [32])
def test_attention_unnormed_vs_fp64(ops, H, layout):
    """q, k = 4 x without the RMSNorm (qk_rmsnorm = False): |s / cap| > 3, the general kernels alone with no fast-path parameters"""
    att.fast_vs_fp64(ops, *att.LAYOUTS[layout], H, None, seed = 20 + H, gated = True)


@pytest.mark.parametrize('gamma', ['inside', 'outside'])
@pytest.mark.parametrize('layout', list(att.RINGS))
@pytest.mark.parametrize('H', [32])
def test_attention_vs_fp64_long_sequences(ops, H, layout, gamma):
    att.fast_vs_fp64(ops, *att.RINGS[layout], H, att.GAMMAS[gamma], seed = 30 + H, gated = True)


@pytest.mark.parametrize('H', HEADS)
def test_attn_bwd_prep_without_gate_sums(ops, H):
    """the pre-pass of an ungated model (gates = None, dsum_mh = None) writes dop, dsum and the cleared dq bit for bit as the same call given a
    gate-sum buffer, and touches no row past its outputs.  Without gates dop = dO exactly, dsum = sum dO o, and the gate sums equal dsum"""
    M, HI = att.VAR_M, H * 64
    g = gen(140 + H)
    dog, o = att._rand(g, M, HI).to(BF16), att._rand(g, M, HI, scale = 2.).to(BF16)
    runs = []
    for with_buffer in (True, False):
        (dop_b, dop), (dsum_b, dsum), (dq_b, dq) = guarded(M, HI, BF16), guarded(H, M, F32), guarded(M, HI, F32)
        mh_b, mh = guarded(M, H, F32) if with_buffer else (None, None)
        ops.attn_bwd_prep(dog, o, None, dop, dsum, mh, dq, M, H)
        torch.cuda.synchronize()
        for buf, rows in ((dop_b, M), (dsum_b, H), (dq_b, M)) + (((mh_b, M),) if with_buffer else ()):
            assert untouched(buf[rows:]), 'the pre-pass wrote past the last row of an output'
        runs.append(dict(dop = dop, dsum = dsum, dq = dq, mh = mh))
    a, b = runs
    for name in ('dop', 'dsum', 'dq'):
        assert same_bits(a[name], b[name]), name
    assert torch.equal(a['dop'], dog) and (a['dq'] == 0).all()
    assert same_bits(a['mh'], a['dsum'].t())
    terms = (dog.double() * o.double()).reshape(M, H, 64)
    att.check('var_sum', att.row_err(a['dsum'].t(), terms.sum(-1), H, 1, mag = terms.abs().sum(-1)))


# ================================================================================================ exact invariants across heads
ISOLATION_HEADS = (32, 30)


@pytest.mark.parametrize('path', ['fast', 'general'])
@pytest.mark.parametrize('H', ISOLATION_HEADS)
def test_heads_are_isolated(ops, H, path):
    """new data in every row of one head j (q and k new unit rows inside the norm bound, v = +-1e3, new dO and gate): in every other head o,
    lse, dk, dv and the gate sums stay bit-identical, and dq moves by reduction-order noise only.  A CTA that reads or writes a neighbouring
    head's columns, or a wrong head stride into lse / dsum, fails this whatever the tolerance.  Head j itself must change."""
    rb, T, g, fp, q, k, v, gates, dog = att._inv_setup(ops, H)
    M = rb.M
    general_only = path == 'general'
    base = att.attention_pass(ops, T, q, k, v, gates, dog, H, fp, general_only)
    for j in (0, 17, H - 1):
        c = slice(64 * j, 64 * (j + 1))
        q2, k2, v2, dog2, gates2 = (t.clone() for t in (q, k, v, dog, gates))
        q2[:, c] = att.unit_rows(torch.randn(M, 1, 64, device = 'cuda', generator = g, dtype = F64), INSIDE)
        k2[:, c] = att.unit_rows(torch.randn(M, 1, 64, device = 'cuda', generator = g, dtype = F64), INSIDE)
        v2[:, c] = (torch.randint(0, 2, (M, 64), device = 'cuda', generator = g) * 2000. - 1000.).to(BF16)
        dog2[:, c] = torch.randn(M, 64, device = 'cuda', generator = g).to(BF16)
        gates2[:, j] = torch.randn(M, device = 'cuda', generator = g)
        new = att.attention_pass(ops, T, q2, k2, v2, gates2, dog2, H, fp, general_only)
        keep = torch.ones(H, dtype = torch.bool, device = 'cuda'); keep[j] = False
        cols = keep.repeat_interleave(64)
        for name in ('o', 'dk', 'dv'):
            assert torch.equal(new[name][:, cols], base[name][:, cols]), f'{name} of another head moved when head {j} changed'
            assert not torch.equal(new[name][:, c], base[name][:, c]), f'{name} of head {j} did not change with its inputs'
        assert torch.equal(new['lse'][keep], base['lse'][keep]) and not torch.equal(new['lse'][j], base['lse'][j])
        assert torch.equal(new['dsum_mh'][:, keep], base['dsum_mh'][:, keep])
        d = (new['dq'] - base['dq']).abs().reshape(M, H, 64)[:, keep].amax(-1)
        assert (d <= 1e-5 * base['dq'].abs().reshape(M, H, 64)[:, keep].amax(-1)).all(), f'dq of another head moved when head {j} changed'
        assert not torch.equal(new['dq'][:, c], base['dq'][:, c])


@pytest.mark.parametrize('H', ISOLATION_HEADS)
def test_invisible_keys_do_not_matter(ops, H):
    att.test_invisible_keys_do_not_matter(ops, H)


@pytest.mark.parametrize('H', ISOLATION_HEADS)
def test_invisible_queries_do_not_matter(ops, H):
    att.test_invisible_queries_do_not_matter(ops, H)


@pytest.mark.parametrize('H', ISOLATION_HEADS)
def test_cached_prefill_vs_fp64(ops, H):
    att.test_cached_prefill_vs_fp64(ops, H)


# ================================================================================================ LASER / value-residual row kernels
@pytest.mark.parametrize('clamp', [15., 5.])
@pytest.mark.parametrize('H', ROW_HEADS)
def test_laser_v_fwd_vs_fp64(ops, H, clamp):
    att.test_laser_v_fwd_vs_fp64(ops, H, clamp)


@pytest.mark.parametrize('H', ROW_HEADS)
def test_laser_v_bwd_vs_fp64(ops, H):
    att.test_laser_v_bwd_vs_fp64(ops, H)


@pytest.mark.parametrize('gated', [True, False])
@pytest.mark.parametrize('H', ROW_HEADS)
def test_laser_out_fwd_vs_fp64(ops, H, gated):
    att.test_laser_out_fwd_vs_fp64(ops, H, gated)


@pytest.mark.parametrize('gates', ['gated', 'ungated', 'ungated-no-sums'])
@pytest.mark.parametrize('H', ROW_HEADS)
def test_laser_bwd_prep_vs_fp64(ops, H, gates):
    att.test_laser_bwd_prep_vs_fp64(ops, H, gated = gates == 'gated', dsum_mh_none = gates == 'ungated-no-sums')


@pytest.mark.parametrize('H', ROW_HEADS)
def test_vmix_fwd_vs_fp64(ops, H):
    att.test_vmix_fwd_vs_fp64(ops, H)


@pytest.mark.parametrize('H', ROW_HEADS)
def test_vmix_bwd_vs_fp64(ops, H):
    """d mix_pre into its dqkvg columns from MIX = 3 HI + H rounded up to even: up to 3 HI + 64 at H = 32"""
    att.test_vmix_bwd_vs_fp64(ops, H)


@pytest.mark.parametrize('H', [32])
def test_add_f32_into_bf16_vs_fp64(ops, H):
    """HI = 2048"""
    att.test_add_f32_into_bf16_vs_fp64(ops, H)


# ================================================================================================ the layer chain in engine order
@pytest.mark.parametrize('gated', [True, False], ids = ['gated', 'ungated'])
@pytest.mark.parametrize('laser', [True, False], ids = ['laser', 'plain'])
@pytest.mark.parametrize('H', [24, 32])
def test_layer_chain_vs_fp64(ops, H, laser, gated):
    att.test_layer_chain_vs_fp64(ops, H, laser, gated = gated)

