"""GPU: the per-layer normalisation row kernels against float64, at every dispatched model width.

    adaln_fwd    u = LN(x) (gamma_c + 1) + beta_c on modality rows (FiLM row c of the strided table), LN(x) (g + 1) on text rows;
                 stats = (mean, rstd) per row
    adaln_bwd    dx += LN'(du scale); d gamma_c, d beta_c into the strided gradient table; d g (text rows) accumulated
    rmsnorm_fwd  out = x / max(|x|, 1e-12) sqrt(D) (gamma + 1): fp32, bf16 and the modality rows compacted through `slot`
    rmsnorm_bwd  dx overwritten, d gamma accumulated
    embed_bwd    text rows add into the embedding gradient (id -1 lands on row 0), modality rows go to the bf16 compact matrix through `slot`

Each kernel is called through the C ABI with the argument patterns of engine.forward / engine.backward and the Self-Flow head.

Reference and bounds (|got - ref| <= bound element-wise; the worst err / bound of each check is printed, run with -s):
  - references are float64 from the same fp32 inputs.  A row reduction of the kernels sums NCH * 4 terms per lane, then 5 butterfly
    levels: its fp32 error is at most NSUM = NCH * 4 + 5 roundings (2^-24 relative each) of the sum of |terms|.
  - adaln_fwd: mean and rstd to those roundings (rstd also to rsqrtf's 2 ulp); u (bf16) to 2^-8 |ref| plus the fp32 error of mean and
    rstd carried through (x - mean) rstd scale + shift.
  - adaln_bwd reads the stats the forward kernel wrote.  Its reference is float64 autograd of LN(x) scale + shift; the bound adds the
    exact float64 effect of the kernel's fp32 stats (the LN backward evaluated with them minus with the exact stats) to the roundings.
  - sums (dfilm, dln_gamma, dgamma, demb) are held to REL_SUM times the sum of |terms| plus |initial value|: one warp's rows lost is
    hundreds of times that.  Every sum output starts from a non-zero value.
  - bf16 copies of fp32 values (dmodtok) are compared bit for bit with torch's round-to-nearest cast.
  - bytes a kernel must not write (a guard row past M or past the table in every output, the zero-gate columns and the other
    wrappers' columns of the FiLM gradient table, compact rows no slot maps to) hold a sentinel and are compared bit for bit.
M = 20011 rows: prime, so no rows-per-warp of the chunked kernels divides it and the last warp's chunk is partial; and more than twice
the warps any of these grids can have resident, so every warp of the persistent grids walks at least two rows (the adaln_fwd cp.async
ring wraps, the condition-row prefetch is used).  Each input has an all-zero row and a constant row (LayerNorm variance 0: rstd =
1 / sqrt(1e-5)), as a text row and as a modality row; the RMSNorm input also has rows shorter than the 1e-12 clamp."""
import math

import numpy as np
import pytest
import torch

from helpers import SENT, Checks as _Checks, gen, guarded, same_bits, untouched
from transfusion_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
BF16, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
U8, U24 = 2.0 ** -8, 2.0 ** -24
DISPATCH_D = (128, 256, 384, 512, 768, 1024)
M_ROWS = 20011
NC = 37                                # condition rows (modality instances)
WRAPPERS, W = 6, 4                     # AdaptiveWrappers of the table (depth 3) and the one under test
LN_EPS, RMS_EPS = 1e-5, 1e-12
REL_SUM = 1e-6                         # sums / atomics, relative to sum |terms| + |initial| (the value test_block_epilogues_gpu.py uses)
# Measured worst err / bound on an H100 80GB HBM3 (700 W power limit), with the constants above: u and out_bf16 0.996 (the bf16 cast's
# rounding, which the bound states exactly); adaln_fwd mean 0.11, rstd 0.21; adaln_bwd dx 0.37, dfilm 0.18, dln_gamma 0.044;
# rmsnorm_fwd out_f32 0.44; rmsnorm_bwd dx 0.21, dgamma 0.044; embed_bwd demb 0.26.

SHOWN = {}


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


@pytest.fixture(scope = 'module', autouse = True)
def _report():
    yield
    for name, r in sorted(SHOWN.items()):
        print(f'worst over the file: {name:32s} {r:.3g}')


def Checks(what):
    return _Checks(what, SHOWN)


def nsum(D):
    return D // 128 * 4 + 5


def test_rows_cover_every_warp_twice():
    """M is prime and above twice the warps of every grid here: adaln_fwd's persistent grid holds at most the warps the thread limit lets
    reside on an SM (its ring's shared memory can only lower that), the row_grid kernels launch at most 8 blocks of 8 warps per SM"""
    assert all(M_ROWS % p for p in range(2, math.isqrt(M_ROWS) + 1)) and M_ROWS % 32
    p = torch.cuda.get_device_properties(0)
    warps = p.multi_processor_count * max(p.max_threads_per_multi_processor // 32, 8 * 8)
    assert M_ROWS > 2 * warps, warps


# ------------------------------------------------------------------------------------------------ inputs
def cond_layout(M, nc, seed):
    """condition row per token as the engine lays it out: runs of one modality instance (0 .. nc-1) and text runs (-1) in shuffled order,
    runs of one to 400 rows (crossing warp chunks and blocks), the same instance in several runs, instance nc - 1 and 0 present"""
    rng = np.random.default_rng(seed)
    out = [-1] * 7 + [nc - 1] * 90 + [0] * 3
    while len(out) < M:
        out += [int(rng.integers(-1, nc))] * int(rng.integers(1, 401))
    return torch.tensor(out[:M], dtype = I32, device = 'cuda')


def special_rows(cond):
    """(zero text row, zero modality row, constant text row, constant modality row)"""
    t = (cond < 0).nonzero().squeeze(1).tolist()
    m = (cond >= 0).nonzero().squeeze(1).tolist()
    return t[len(t) // 3], m[len(m) // 3], t[2 * len(t) // 3], m[2 * len(m) // 3]


def ln_inputs(D, seed, with_cond = True):
    g = gen(seed)
    M = M_ROWS
    x = torch.randn(M, D, device = 'cuda', generator = g) * 2 + 0.5
    cond = cond_layout(M, NC, seed) if with_cond else torch.full((M,), -1, dtype = I32, device = 'cuda')
    zt, zm, ct, cm = special_rows(cond) if with_cond else (11, 12, 13, 14)
    x[zt] = 0; x[zm] = 0; x[ct] = 1.5; x[cm] = 1.5          # 1.5 sums exactly: mean 1.5, variance 0
    tab = torch.randn(NC, WRAPPERS * 3 * D, device = 'cuda', generator = g) * 0.3
    lg = torch.randn(D, device = 'cuda', generator = g) * 0.3
    return x, cond, tab, lg


def film_cols(D):
    return slice(W * 3 * D, W * 3 * D + 2 * D)


def scale_shift(cond, tab, lg, D):
    """per-row float64 scale and shift: FiLM row of the wrapper for modality rows, (g + 1, 0) for text rows"""
    isM = (cond >= 0)[:, None]
    cr = cond.long().clamp(min = 0)
    f = tab[:, W * 3 * D:].double()
    sc = torch.where(isM, f[cr, :D] + 1., lg.double() + 1.)
    sh = torch.where(isM, f[cr, D:2 * D], torch.zeros((), dtype = F64, device = 'cuda'))
    return sc, sh


def ln_exact(x):
    x64 = x.double()
    mean = x64.mean(1, keepdim = True)
    var = ((x64 - mean) ** 2).mean(1, keepdim = True)
    return mean, var, 1. / (var + LN_EPS).sqrt()


def run_adaln_fwd(ops, x, cond, tab, lg, D, with_cond):
    M = M_ROWS
    ub, u = guarded(M, D, BF16)
    sb, st = guarded(M, 2, F32)
    ops.adaln_fwd(x, cond if with_cond else None, tab[:, W * 3 * D:] if with_cond else None, WRAPPERS * 3 * D, lg, u, st, M, D)
    return ub, u, sb, st


# ================================================================================================ adaln_fwd
@pytest.mark.parametrize('D', DISPATCH_D)
def test_adaln_fwd_vs_float64(ops, D):
    ck = Checks(f'adaln_fwd D={D}')
    n = nsum(D)
    for with_cond in (True, False):
        tag = 'adaln_fwd' + ('' if with_cond else ' text-only')
        x, cond, tab, lg = ln_inputs(D, 10 + D, with_cond)
        tab0 = tab.clone()
        ub, u, sb, st = run_adaln_fwd(ops, x, cond, tab, lg, D, with_cond)
        mean, var, rstd = ln_exact(x)
        sc, sh = scale_shift(cond, tab, lg, D)
        E_mean = (n + 2) * U24 * x.double().abs().mean(1, keepdim = True)
        E_var = (n + 6) * U24 * (var + E_mean ** 2) + E_mean ** 2 + 2 * U24 * LN_EPS
        rel_rstd = 0.5 * E_var / (var + LN_EPS) + 5 * U24                                  # + rsqrtf (2 ulp) and one rounding
        ck(f'{tag} mean', st[:, :1], mean, E_mean)
        ck(f'{tag} rstd', st[:, 1:], rstd, rel_rstd * rstd)
        xm = x.double() - mean
        ref = xm * rstd * sc + sh
        E32 = sc.abs() * rstd * (E_mean * (1 + U24) + xm.abs() * (rel_rstd + 4 * U24)) + 2 * U24 * (xm * rstd * sc).abs() + U24 * ref.abs()
        ck(f'{tag} u', u, ref, U8 * ref.abs() + (1 + U8) * E32)
        zt, zm, ct, cm = special_rows(cond) if with_cond else (11, 12, 13, 14)
        inv = 1. / torch.tensor(LN_EPS, dtype = F32, device = 'cuda').sqrt()
        for r, what in ((zt, 'zero row'), (zm, 'zero row'), (ct, 'constant row'), (cm, 'constant row')):
            ck.true(f'{tag} {what} {r}: mean exact, rstd = 1 / sqrt(1e-5)',
                    st[r, 0].item() == float(x[r, 0]) and abs(st[r, 1].item() / inv.item() - 1) < 8 * U24)
            ck.true(f'{tag} {what} {r}: u = bf16(shift)', bool((u[r].float() == sh[r].float().to(BF16).float()).all()))
        ck.true(f'{tag}: guard rows untouched', untouched(ub[M_ROWS]) and untouched(sb[M_ROWS]))
        ck.true(f'{tag}: FiLM table not written', same_bits(tab, tab0))
    ck.done()


# ================================================================================================ adaln_bwd
def ln_backward64(du, x, mean, rstd, sc):
    """dx of u = (x - mean) rstd sc + shift with mean / rstd the row statistics (their dependence on x included), and xhat"""
    xh = (x.double() - mean) * rstd
    d = du.double() * sc
    m1, m2 = d.mean(1, keepdim = True), (d * xh).mean(1, keepdim = True)
    return rstd * (d - m1 - xh * m2), xh


@pytest.mark.parametrize('D', DISPATCH_D)
def test_adaln_bwd_vs_float64(ops, D):
    ck = Checks(f'adaln_bwd D={D}')
    n, M = nsum(D), M_ROWS
    for with_cond in (True, False):
        tag = 'adaln_bwd' + ('' if with_cond else ' text-only')
        x, cond, tab, lg = ln_inputs(D, 20 + D, with_cond)
        _, _, _, st = run_adaln_fwd(ops, x, cond, tab, lg, D, with_cond)
        g = gen(30 + D)
        du = torch.randn(M, D, device = 'cuda', generator = g)
        dxb = torch.randn(M + 1, D, device = 'cuda', generator = g)          # accumulated into; the last row is a guard
        dtab = torch.randn(NC + 1, WRAPPERS * 3 * D, device = 'cuda', generator = g)   # the last row is a guard
        dgb = torch.randn(D + 1, device = 'cuda', generator = g)
        dxb0, dtab0, dgb0 = dxb.clone(), dtab.clone(), dgb.clone()
        ops.adaln_bwd(du, x, st, cond if with_cond else None, tab[:, W * 3 * D:] if with_cond else None, WRAPPERS * 3 * D, lg, dxb[:M],
                      dtab[:, W * 3 * D:] if with_cond else None, WRAPPERS * 3 * D, dgb[:D], M, D)
        sc, sh = scale_shift(cond, tab, lg, D)
        # float64 autograd of the forward function with exact statistics
        xa = x.double().requires_grad_(True)
        fa = tab[:, W * 3 * D:W * 3 * D + 2 * D].double().requires_grad_(True)
        ga = lg.double().requires_grad_(True)
        isM = (cond >= 0)[:, None]
        cr = cond.long().clamp(min = 0)
        xn = torch.nn.functional.layer_norm(xa, (D,), eps = LN_EPS)
        uu = torch.where(isM, xn * (fa[cr, :D] + 1) + fa[cr, D:], xn * (ga + 1))
        uu.backward(du.double())
        mean, _, rstd = ln_exact(x)
        dx_exact, xh_exact = ln_backward64(du, x, mean, rstd, sc)
        scale = xa.grad.abs().amax().item()
        ck.true(f'{tag}: float64 LN backward formula = autograd', (dx_exact - xa.grad).abs().amax().item() <= 1e-9 * scale)
        # the same formula with the fp32 statistics the forward kernel wrote: their effect on dx is part of the bound
        mk, rk = st[:, :1].double(), st[:, 1:].double()
        dx_k, xh_k = ln_backward64(du, x, mk, rk, sc)
        dd = du.double() * sc
        T = dd.abs() + dd.abs().mean(1, keepdim = True) + xh_k.abs() * (dd * xh_k).abs().mean(1, keepdim = True)
        ref = dxb0[:M].double() + xa.grad
        bound = (dx_k - dx_exact).abs() + rk * (n + 8) * U24 * T + U24 * ref.abs()
        ck(f'{tag} dx', dxb[:M], ref, bound)
        ck.true(f'{tag}: dx guard row untouched', same_bits(dxb[M], dxb0[M]))
        dxh = (xh_k - xh_exact).abs()
        du64 = du.double()
        text = ~isM[:, 0]
        want = dgb0[:D].double() + ga.grad
        terms = (du64 * xh_k)[text].abs().sum(0)
        ck(f'{tag} dln_gamma', dgb[:D], want, REL_SUM * (terms + dgb0[:D].double().abs()) + (du64.abs() * dxh)[text].sum(0))
        ck.true(f'{tag}: dln_gamma guard untouched', same_bits(dgb[D:], dgb0[D:]))
        ck.true(f'{tag}: gradient table guard row untouched', same_bits(dtab[NC], dtab0[NC]))
        if with_cond:
            rows = isM[:, 0].nonzero().squeeze(1)
            idx = cr[rows]
            T_g = torch.zeros(NC, D, dtype = F64, device = 'cuda').index_add_(0, idx, (du64 * xh_k)[rows].abs())
            P_g = torch.zeros(NC, D, dtype = F64, device = 'cuda').index_add_(0, idx, (du64.abs() * dxh)[rows])
            T_b = torch.zeros(NC, D, dtype = F64, device = 'cuda').index_add_(0, idx, du64[rows].abs())
            fc = film_cols(D)
            d0 = dtab0[:NC, fc].double()
            ck(f'{tag} dfilm gamma', dtab[:NC, fc][:, :D], d0[:, :D] + fa.grad[:, :D], REL_SUM * (T_g + d0[:, :D].abs()) + P_g)
            ck(f'{tag} dfilm beta', dtab[:NC, fc][:, D:], d0[:, D:] + fa.grad[:, D:], REL_SUM * (T_b + d0[:, D:].abs()))
            other = torch.ones(WRAPPERS * 3 * D, dtype = torch.bool, device = 'cuda'); other[fc] = False
            ck.true(f'{tag}: zero-gate and other wrappers\' columns of the gradient table untouched', same_bits(dtab[:NC, other], dtab0[:NC, other]))
    ck.done()


# ================================================================================================ rmsnorm_fwd / rmsnorm_bwd
def rms_inputs(D, seed, tiny):
    g = gen(seed)
    M = M_ROWS
    x = torch.randn(M, D, device = 'cuda', generator = g) * 1.5
    x[101] = 0
    x[M - 1] = 0.75                                                       # the last row: a constant row in the last, partial chunk
    if tiny:
        x[202] *= 1e-14; x[303] *= 1e-14                                  # |x| < 1e-12: the norm is clamped
    gamma = torch.randn(D, device = 'cuda', generator = g) * 0.3
    return x, gamma


def slot_map(M, seed):
    """slot per row: a third of the rows map to a permutation of compact rows (slot 0 included); S_CAP - S compact rows stay unmapped"""
    g = gen(seed)
    S = M // 3
    rows = torch.randperm(M, device = 'cuda', generator = g)[:S]
    perm = torch.randperm(S + 50, device = 'cuda', generator = g)[:S]
    perm[(perm == 0).nonzero().squeeze(1)] = perm[0].clone()
    perm[0] = 0
    slot = torch.full((M,), -1, dtype = I32, device = 'cuda')
    slot[rows] = perm.to(I32)
    return slot, S + 50


def rms_exact(x, gamma):
    x64 = x.double()
    nrm = x64.norm(dim = 1, keepdim = True)
    return x64 / nrm.clamp_min(RMS_EPS) * x.shape[1] ** 0.5 * (gamma.double() + 1.)


@pytest.mark.parametrize('D', DISPATCH_D)
def test_rmsnorm_fwd_vs_float64(ops, D):
    ck = Checks(f'rmsnorm_fwd D={D}')
    M, n = M_ROWS, nsum(D)
    x, gamma = rms_inputs(D, 40 + D, tiny = True)
    slot, cap = slot_map(M, 50 + D)
    ref = rms_exact(x, gamma)
    E32 = ((n + 1) / 2 + 6) * U24 * ref.abs()
    Eb = U8 * ref.abs() + (1 + U8) * E32
    # final norm: fp32 + bf16 rows and the compacted modality rows
    fb, f = guarded(M, D, F32); bb, b = guarded(M, D, BF16)
    mb, om = guarded(cap, D, BF16)
    ops.rmsnorm_fwd(x, gamma, f, b, slot, om, M, D)
    ck('rmsnorm_fwd out_f32', f, ref, E32)
    ck('rmsnorm_fwd out_bf16', b, ref, Eb)
    ck.true('zero row: out exactly 0', bool((f[101] == 0).all()))
    rows = (slot >= 0).nonzero().squeeze(1)
    ck.true('out_mod rows = bytes of the bf16 rows they compact', same_bits(om[slot[rows].long()], b[rows]))
    unmapped = torch.ones(cap, dtype = torch.bool, device = 'cuda'); unmapped[slot[rows].long()] = False
    ck.true('out_mod rows no slot maps to untouched', untouched(om[unmapped]) and int(unmapped.sum()) == cap - rows.numel())
    ck.true('guard rows untouched', untouched(fb[M]) and untouched(bb[M]) and untouched(mb[cap]))
    # Self-Flow head: bf16 only, no compaction
    bb2, b2 = guarded(M, D, BF16)
    ops.rmsnorm_fwd(x, gamma, None, b2, None, None, M, D)
    ck.true('bf16-only call = bytes of the full call', same_bits(b2, b) and untouched(bb2[M]))
    ck.done()


def check_rmsnorm_bwd(ops, ck, x, gamma, seed):
    """rmsnorm_bwd on rows x against float64 autograd of F.normalize(x, eps = 1e-12) sqrt(D) (gamma + 1): on a row shorter than the clamp
    the clamped norm is a constant, so dx = d xhat / 1e-12 there"""
    M, D = x.shape
    n = nsum(D)
    g = gen(seed)
    dout = torch.randn(M, D, device = 'cuda', generator = g)
    dxb, dx = guarded(M, D, F32)
    dx.normal_(generator = g)                                              # overwritten
    dgb = torch.randn(D + 1, device = 'cuda', generator = g)
    dgb0 = dgb.clone()
    ops.rmsnorm_bwd(dout, x, gamma, dx, dgb[:D], M, D)
    xa = x.double().requires_grad_(True)
    ga = gamma.double().requires_grad_(True)
    (torch.nn.functional.normalize(xa, dim = -1, eps = RMS_EPS) * D ** 0.5 * (ga + 1)).backward(dout.double())
    x64 = x.double()
    rn = 1. / x64.norm(dim = 1, keepdim = True).clamp_min(RMS_EPS)
    xh = x64 * rn
    dd = dout.double() * D ** 0.5 * (gamma.double() + 1.)
    Edx = rn * (n + 8) * U24 * (dd.abs() + xh.abs() * (dd * xh).abs().sum(1, keepdim = True)) + ((n + 1) / 2 + 3) * U24 * xa.grad.abs()
    ck('rmsnorm_bwd dx', dx, xa.grad, Edx)
    terms = (dout.double() * xh).abs().sum(0) * D ** 0.5
    ck('rmsnorm_bwd dgamma', dgb[:D], dgb0[:D].double() + ga.grad, REL_SUM * (terms + dgb0[:D].double().abs()))
    ck.true('guard row / element untouched', untouched(dxb[M]) and same_bits(dgb[D:], dgb0[D:]))


@pytest.mark.parametrize('D', DISPATCH_D)
def test_rmsnorm_bwd_vs_float64(ops, D):
    ck = Checks(f'rmsnorm_bwd D={D}')
    x, gamma = rms_inputs(D, 60 + D, tiny = True)
    check_rmsnorm_bwd(ops, ck, x, gamma, 70 + D)
    ck.done()


def test_rmsnorm_bwd_below_the_norm_clamp(ops):
    """every row shorter than the 1e-12 clamp: the projection term -xhat (xhat . dxhat) of the unclamped backward must be absent"""
    D, M = 256, 333
    ck = Checks('rmsnorm_bwd below the clamp')
    g = gen(80)
    x = torch.randn(M, D, device = 'cuda', generator = g) * 3e-14
    gamma = torch.randn(D, device = 'cuda', generator = g) * 0.3
    check_rmsnorm_bwd(ops, ck, x, gamma, 81)
    ck.done()


# ================================================================================================ embed_bwd
@pytest.mark.parametrize('D', DISPATCH_D)
def test_embed_bwd_vs_float64(ops, D):
    ck = Checks(f'embed_bwd D={D}')
    M, V = M_ROWS, 70
    g = gen(90 + D)
    dx0 = torch.randn(M, D, device = 'cuda', generator = g)
    text_id = torch.randint(-1, V, (M,), device = 'cuda', generator = g, dtype = I32)      # every row a valid id, modality rows too
    slot, cap = slot_map(M, 95 + D)
    for with_slot in (True, False):
        tag = 'embed_bwd' + ('' if with_slot else ' text-only')
        demb = torch.randn(V + 1, D, device = 'cuda', generator = g)                          # accumulated into; the last row is a guard
        demb0 = demb.clone()
        mb, dmod = guarded(cap, D, BF16)
        ops.embed_bwd(dx0, text_id, slot if with_slot else None, demb[:V], dmod if with_slot else None, M, D)
        text = slot < 0 if with_slot else torch.ones(M, dtype = torch.bool, device = 'cuda')
        ids = text_id.long().clamp(min = 0)[text]
        want = torch.zeros(V, D, dtype = F64, device = 'cuda').index_add_(0, ids, dx0[text].double())
        terms = torch.zeros(V, D, dtype = F64, device = 'cuda').index_add_(0, ids, dx0[text].double().abs())
        ck(f'{tag} demb', demb[:V], demb0[:V].double() + want, REL_SUM * (terms + demb0[:V].double().abs()))
        ck.true(f'{tag}: demb guard row untouched', same_bits(demb[V], demb0[V]))
        if with_slot:
            rows = (~text).nonzero().squeeze(1)
            ck.true('dmodtok rows = bf16 of the rows they take', same_bits(dmod[slot[rows].long()], dx0[rows].to(BF16)))
            unmapped = torch.ones(cap, dtype = torch.bool, device = 'cuda'); unmapped[slot[rows].long()] = False
            ck.true('dmodtok rows no slot maps to untouched', untouched(dmod[unmapped]))
        ck.true(f'{tag}: dmodtok guard row untouched', untouched(mb[cap]) and (with_slot or untouched(mb)))
    ck.done()
