"""GPU: the fused GEMM epilogues of a transformer layer and the kernels that differentiate them, against float64, at every accepted
head-count class and every dispatched model width.

    gemm_qkvg          (qk-RMSNorm, (gamma + 1), interleaved RoPE, gates, value-residual mix, kv-cache row scatter)  <->  qk_bwd_pack
    gemm_resid         (bias, adaLN-zero gate or layerscale, residual, two-operand skip projection)                 <->  resid_bwd
    gemm_geglu[_drop]  (tile-interleaved value / gate, bias, erf-GELU, FFN dropout)                                 <->  geglu_bwd[_drop] + colsum_f32

Each kernel is called through the C ABI with the argument patterns of engine.forward / engine.backward.

Reference and bounds (every check is |got - ref| <= bound element-wise; the worst err / bound of each check is printed, run with -s):
  - GEMM part: y64 = u.double() @ W.double().T from the same bf16 operands, mag = |u| @ |W|^T in float64.  The fp32 tensor-core
    accumulation over kb = ceil(K / 64) k-blocks is bounded by c_acc(kb) * mag per element (helpers.py: 1.6e-6 up to 43 k-blocks, growing
    with sqrt(kb / 43) past that); C_ACC below stands for c_acc(kb) of the GEMM at hand.
  - epilogue outputs are computed in float64 from y64.  A bf16 output may differ by 2^-8 |ref| (the rounding of the cast) plus the
    accumulator bound carried through the epilogue; for q / k that is 8 |gamma + 1| inv times the rope pair's C_ACC * mag, plus the
    error of inv, plus a few fp32 roundings (2^-24 relative each).  fp32 outputs (gates, mix, qk_inv, x_out) get the accumulator term
    plus a few fp32 roundings.
  - RoPE uses the kernel's own cos / sin table (ops.rope_table) read back and promoted to float64, so these tests do not depend on the
    table, which test_aux_kernels_gpu.py checks.
  - backward kernels read bf16 values the forward saved: their references are float64 autograd (or the float64 formula) of the same
    function, with the bf16 input error propagated to first order.  qk_bwd_pack rebuilds xhat_j = (R^T q)_j / (8 (gamma_j + 1)):
    an error in the rope pair of q is amplified by 1 / |gamma_j + 1|.
  - sums (dgamma, dlayerscale, dzgate, dbias, the GEGLU partials reduced by colsum_f32) are held to REL_SUM times the sum of the
    magnitudes of their terms: one block's contribution lost is thousands of times that.
  - bytes a kernel must not write (a guard row past M in every output, kv-cache rows not in kv_rows, the dqkvg columns qk_bwd_pack
    leaves to the attention backward and the pad columns engine.backward clears once per step, output entries a column map skips)
    hold a sentinel and are compared bit for bit.
M = 9011 rows: not a multiple of 32 (the last warp slab of the last GEMM tile is partial), several work items per GEMM CTA, several
rows per warp in the row kernels, and a ragged last block of geglu_bwd.  The worst errors measured over the whole file on an H100 80GB
HBM3 (700 W power limit) are in the comments beside the constants; with -s the file prints them again at the end."""
import numpy as np
import pytest
import torch

from helpers import SENT, Checks as _Checks, c_acc, cluster_mode, gen, guarded, same_bits, show_c_acc, untouched  # noqa: F401  (cluster_mode: a fixture)
from transfusion_pytorch_b200 import _lib, engine as E
from oracle.dropout_mask import keep_mask, scale as drop_scale, SITE_FFN

pytestmark = pytest.mark.gpu
BF16, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
U8, U24 = 2.0 ** -8, 2.0 ** -24       # bf16 cast, one fp32 rounding (relative)
M_ROWS = 9011
N_POS = 16384                         # RoPE table length; positions run to its last entry
ZERO_ROW = 4321                       # an all-zero row of u in the QKVG test
# float64 values of [rows, 2 Ip] per row chunk of the GEGLU forward reference: one chunk up to D = 1024 (M_ROWS x 5504), two at 1536 and
# 2048, where the whole reference would peak past 10 GB of device memory (measured on the H100: 10.3 GiB at D = 2048 in one chunk, 5.8 GiB in
# two)
REF_VALUES = 50_000_000

# fp32 accumulation of the wgmma GEMMs: c_acc(kb) of helpers.py, relative to |u| @ |W|^T; measured 5.4e-7 (x_out, K <= 2752; QKVG gates 4.0e-7)
REL_SUM = 1e-6     # column sums / atomics, relative to the sum of |terms|; measured 1.2e-7 (resid_bwd dzgate)
PHI_ABS = 7.5e-8   # Abramowitz-Stegun 7.1.26 in gelu_parts: |erf error| <= 1.5e-7, so Phi is off by at most half of it (not a fit)
# Measured worst err / bound of the checks (same H100 run, with the constants above): every bf16 output 0.99 - 0.996 (the cast's rounding,
# which the bound states exactly); qkvg gates 0.25, mix 0.18, qk_inv 0.054; resid x_out 0.32 - 0.36; qk_bwd dgamma 0.003 (own terms),
# 0.020 (autograd, with the propagated xhat error); resid_bwd sums 0.025 - 0.12; geglu_bwd dbias 0.012 - 0.018.

# (model dim D, heads H, learned value residual): every dispatched width, H from 2 to 32 (H % 4 == 2 after full head groups at 6, 10,
# 30), HI = 64 H both larger and smaller than D, the mix columns filling the 32-column gate slab at H = 16
CONFIGS = [(128, 32, False), (256, 2, True), (384, 6, False), (512, 8, False), (768, 10, True), (1024, 16, True), (1024, 30, False)]
CFG_IDS = [f'd{d}h{h}' + ('mix' if m else '') for d, h, m in CONFIGS]
DISPATCH_D = (128, 256, 384, 512, 768, 1024)


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


SHOWN = {}


@pytest.fixture(scope = 'module', autouse = True)
def _report():
    yield
    for name, r in sorted(SHOWN.items()):
        print(f'worst over the file: {name:28s} {r:.3g}')


def Checks(what):
    return _Checks(what, SHOWN)


def gemm64(a, w):
    a64, w64 = a.double(), w.double()
    return a64 @ w64.t(), a64.abs() @ w64.abs().t()


def kblocks(a):
    """k-blocks of 64 of a GEMM over the columns of its operand a"""
    return (a.shape[1] + 63) // 64


def cond_runs(M, nc, seed):
    """condition row per token as a packed batch has them: runs of one modality instance (0 .. nc-1) and text runs (-1), shuffled"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < M:
        out += [int(rng.integers(-1, nc))] * int(rng.integers(1, 160))
    return torch.tensor(out[:M], dtype = I32, device = 'cuda')


def rope_tables(ops, dh = 64):
    freqs = 1. / (10000 ** (torch.arange(0, dh, 2, device = 'cuda').float() / dh))
    t = torch.empty(N_POS, dh // 2, 2, device = 'cuda'); tt = torch.empty(dh // 2, N_POS, 2, device = 'cuda')
    ops.rope_table(freqs, t, tt, N_POS, dh // 2)
    return t, tt


def rope64(y, c, s):
    """interleaved pairs (y0, y1) -> (y0 c - y1 s, y1 c + y0 s); c, s broadcast against y[..., 0::2]"""
    y0, y1 = y[..., 0::2], y[..., 1::2]
    return torch.stack((y0 * c - y1 * s, y1 * c + y0 * s), -1).flatten(-2)


def unrope64(q, c, s):
    q0, q1 = q[..., 0::2], q[..., 1::2]
    return torch.stack((q0 * c + q1 * s, q1 * c - q0 * s), -1).flatten(-2)


def pair_sum(x):
    """x_a + x_b over the rope pair of every element"""
    return (x[..., 0::2] + x[..., 1::2]).repeat_interleave(2, -1)


def gammas(seed, dh = 64):
    """gamma + 1 in [0.1, 2]: both signs of gamma, the ends included"""
    g = gen(seed)
    gm = torch.rand(dh, device = 'cuda', generator = g) * 1.9 - 0.9
    i = torch.randperm(dh, device = 'cuda', generator = g)[:2]
    gm[i[0]], gm[i[1]] = -0.9, 1.0
    return gm


def qkvg_inputs(D, H, mix, seed, dh = 64):
    g = gen(seed)
    HI, NQ = dh * H, 3 * dh * H + 128
    u = torch.randn(M_ROWS, D, device = 'cuda', generator = g).to(BF16)
    u[ZERO_ROW] = 0
    W = (torch.randn(NQ, D, device = 'cuda', generator = g) / D ** 0.5).to(BF16)       # pad rows too: the kernel must ignore them
    gq, gk = gammas(seed + 1, dh), gammas(seed + 2, dh)
    pos = torch.randint(0, N_POS, (M_ROWS,), device = 'cuda', generator = g, dtype = I32)
    pos[::97] = N_POS - 1
    return dict(D = D, H = H, dh = dh, HI = HI, NQ = NQ, mix = mix, u = u, W = W, gq = gq, gk = gk, pos = pos)


def run_qkvg(ops, x, tt, M = M_ROWS, rows = None, kv = None):
    """gemm_qkvg (gemm_qkvg_d128 for 128-wide heads) into fresh guarded outputs; with M: the first M rows of u, with kv: k / v scattered to
    kv = (k cache, v cache, kv_rows)"""
    H, HI, D = x['H'], x['HI'], x['D']
    out = {}
    for n, c, dt in (('q', HI, BF16), ('k', HI, BF16), ('v', HI, BF16), ('gates', H, F32), ('inv', 2 * H, F32), ('mix', H, F32)):
        out[n + '_buf'], out[n] = guarded(M, c, dt)
    k, v, kv_rows = (kv if kv is not None else (out['k'], out['v'], None))
    args = (x['u'], D, x['W'], D, M, H, D, out['q'], k, v, out['gates'], out['inv'], x['gq'], x['gk'], x['pos'], tt, N_POS, kv_rows,
            out['mix'] if x['mix'] else None)
    if x['dh'] == 128:
        ops.gemm_qkvg_d128(*args)
    else:
        ops.gemm_qkvg(*args)
    return out


def qk_forward_ref(x, mag, gamma, c, s, kb):
    """float64 q (or k) of one GEMM section x [M, H, dh] over kb k-blocks and its bound; also returns inv64 and the bound on inv's relative
    error"""
    ca = c_acc(kb)
    nrm = x.norm(dim = -1, keepdim = True)
    inv = 1. / nrm.clamp_min(1e-12)
    g1 = gamma.double() + 1.
    rt = x.shape[-1] ** 0.5                               # sqrt(dh): 8 at dh = 64
    y = x * inv * rt * g1
    ref = rope64(y, c, s)
    rel_inv = ca * (x.abs() * mag).sum(-1, keepdim = True) / (nrm * nrm).clamp_min(1e-300) + 40 * U24
    Ey = rt * g1.abs() * inv * (ca * mag + x.abs() * rel_inv) + 3 * U24 * y.abs()
    Ep = pair_sum(Ey + 3 * U24 * y.abs())
    return ref, U8 * ref.abs() + (1 + U8) * Ep, inv, rel_inv


# ================================================================================================ gemm_qkvg
@pytest.mark.parametrize('D,H,mix', CONFIGS, ids = CFG_IDS)
def test_gemm_qkvg_vs_float64(ops, cluster_mode, D, H, mix, dh = 64):
    x = qkvg_inputs(D, H, mix, seed = 100 + D + H, dh = dh)
    HI, NQ, M = x['HI'], x['NQ'], M_ROWS
    t, tt = rope_tables(ops, dh)
    o = run_qkvg(ops, x, tt)
    tag = '' if dh == 64 else f' dh={dh}'
    ck = Checks(f'qkvg{tag} D={D} H={H}')
    y, mag = gemm64(x['u'], x['W'])
    kb = kblocks(x['u'])
    ca = c_acc(kb)
    cs = t[x['pos'].long()].double()
    c, s = cs[:, None, :, 0], cs[:, None, :, 1]
    for which, gam in ((0, x['gq']), (1, x['gk'])):
        sec = slice(which * HI, (which + 1) * HI)
        ref, bound, inv, rel_inv = qk_forward_ref(y[:, sec].reshape(M, H, dh), mag[:, sec].reshape(M, H, dh), gam, c, s, kb)
        name = 'qk'[which]
        ck(f'qkvg{tag} {name}', o[name].reshape(M, H, dh), ref, bound)
        ck(f'qkvg{tag} inv_{name}', o['inv'][:, which * H:(which + 1) * H], inv[..., 0], inv[..., 0] * rel_inv[..., 0] * (1 + U8))
    ck(f'qkvg{tag} v', o['v'], y[:, 2 * HI:3 * HI], U8 * y[:, 2 * HI:3 * HI].abs() + (1 + U8) * ca * mag[:, 2 * HI:3 * HI])
    m0 = 3 * HI + (H + 1) // 2 * 2                       # the mix rows start at an even row (an odd H exists at dh = 128 only)
    gsl, msl = slice(3 * HI, 3 * HI + H), slice(m0, m0 + H)
    ck(f'qkvg{tag} gates', o['gates'], y[:, gsl], ca * mag[:, gsl])
    acc = ((o['gates'].double() - y[:, gsl]).abs() / mag[:, gsl].clamp_min(1e-300)).max().item()
    if mix:
        ck(f'qkvg{tag} mix', o['mix'], y[:, msl], ca * mag[:, msl])
        acc = max(acc, ((o['mix'].double() - y[:, msl]).abs() / mag[:, msl].clamp_min(1e-300)).max().item())
    else:
        ck.true('mix buffer untouched without mix_pre', untouched(o['mix_buf']))
    show_c_acc(SHOWN, kb, acc)
    print(f'qkvg D={D} H={H}: measured accumulator error {acc:.3g} of |u| |W|^T')
    # the all-zero row: q and k exactly 0, inv = 1 / 1e-12 (the clamp), nothing non-finite
    z = ZERO_ROW
    ck.true('zero row: q, k exactly 0', bool((o['q'][z] == 0).all() and (o['k'][z] == 0).all()))
    ck.true('zero row: qk_inv = 1 / 1e-12f', bool((o['inv'][z] == torch.tensor(1., device = 'cuda') / torch.tensor(1e-12, device = 'cuda')).all()))
    for n in ('q', 'k', 'v', 'gates', 'inv', 'mix'):
        ck.true(f'{n}: guard row untouched', untouched(o[n + '_buf'][M]))
    # kv-cache append (prefill): k / v rows land at kv_rows[m] of a larger matrix, everything else is the dense call's bytes
    R = 2 * M + 50
    rows = torch.randperm(R, device = 'cuda', generator = gen(7))[:M].to(I32)
    kc, vc = (torch.full((R, HI), SENT, device = 'cuda', dtype = BF16) for _ in range(2))
    o2 = run_qkvg(ops, x, tt, kv = (kc, vc, rows))
    for n in ('q', 'gates', 'inv') + (('mix',) if mix else ()):
        ck.true(f'kv_rows call: {n} = dense bytes', same_bits(o2[n], o[n]))
    ck.true('kv_rows call: k, v dense buffers untouched', untouched(o2['k_buf']) and untouched(o2['v_buf']))
    ck.true('kv_rows call: cache rows = dense k, v bytes', same_bits(kc[rows.long()], o['k']) and same_bits(vc[rows.long()], o['v']))
    other = torch.ones(R, dtype = torch.bool, device = 'cuda'); other[rows.long()] = False
    ck.true('kv_rows call: other cache rows untouched', untouched(kc[other]) and untouched(vc[other]))
    # decode step: a handful of rows appended at the end of their slabs
    S, cap = 7, 64
    rows_s = (torch.arange(S, device = 'cuda', dtype = I32) * cap + torch.tensor([0, 5, 63, 1, 17, 40, 2], device = 'cuda', dtype = I32))
    kc2, vc2 = (torch.full((S * cap, HI), SENT, device = 'cuda', dtype = BF16) for _ in range(2))
    o3 = run_qkvg(ops, x, tt, M = S, kv = (kc2, vc2, rows_s))
    ck.true('decode call: q = dense bytes', same_bits(o3['q'], o['q'][:S]) and same_bits(o3['gates'], o['gates'][:S]))
    ck.true('decode call: cache rows = dense k, v bytes', same_bits(kc2[rows_s.long()], o['k'][:S]) and same_bits(vc2[rows_s.long()], o['v'][:S]))
    if mix:
        ck.true('decode call: mix = dense bytes', same_bits(o3['mix'], o['mix'][:S]))
    other = torch.ones(S * cap, dtype = torch.bool, device = 'cuda'); other[rows_s.long()] = False
    ck.true('decode call: other cache rows untouched', untouched(kc2[other]) and untouched(vc2[other]))
    ck.done()


# ================================================================================================ qk_bwd_pack
def qk_backward(ops, x, o, t, seed):
    """qk_bwd_pack (qk_bwd_pack_d128 for 128-wide heads) on the forward's outputs o; returns (inputs, outputs, float64 autograd reference)"""
    H, HI, NQ, M, dh = x['H'], x['HI'], x['NQ'], M_ROWS, x['dh']
    g = gen(seed)
    dq = torch.randn(M, HI, device = 'cuda', generator = g); dk = torch.randn(M, HI, device = 'cuda', generator = g)
    dsum = torch.randn(M, H, device = 'cuda', generator = g)
    dgam = torch.randn(2, dh, device = 'cuda', generator = g) * 0.1          # accumulated into
    dgam0 = dgam.clone()
    out_buf, out = guarded(M, NQ, BF16)
    args = (dq, dk, o['q'], o['k'], o['inv'], x['gq'], x['gk'], x['pos'], t, o['gates'], dsum, out, NQ, dgam[0], dgam[1], M, H)
    if dh == 128:
        ops.qk_bwd_pack_d128(*args)
    else:
        ops.qk_bwd_pack(*args)
    # float64 autograd through normalize, (gamma + 1) and RoPE, from the exact GEMM output
    y, _ = gemm64(x['u'], x['W'][:2 * HI])
    cs = t[x['pos'].long()].double()
    c, s = cs[:, None, None, :, 0], cs[:, None, None, :, 1]
    xx = y.reshape(M, 2, H, dh).clone().requires_grad_(True)
    gam = torch.stack((x['gq'], x['gk'])).double().requires_grad_(True)
    qk = rope64(torch.nn.functional.normalize(xx, dim = -1, eps = 1e-12) * dh ** 0.5 * (gam[None, :, None, :] + 1.), c, s)
    d64 = torch.stack((dq, dk), 1).double().reshape(M, 2, H, dh)
    (qk * d64).sum().backward()
    return dict(dq = dq, dk = dk, dsum = dsum, dgam = dgam, dgam0 = dgam0, out = out, out_buf = out_buf, c = c, s = s, x = xx.detach(),
                qk_ref = qk.detach(), dx_ref = xx.grad, dgam_ref = gam.grad + dgam0.double(), d64 = d64)


@pytest.mark.parametrize('D,H,mix', CONFIGS, ids = CFG_IDS)
def test_qk_bwd_pack_vs_float64(ops, D, H, mix, dh = 64):
    x = qkvg_inputs(D, H, mix, seed = 200 + D + H, dh = dh)
    HI, NQ, M = x['HI'], x['NQ'], M_ROWS
    rt = dh ** 0.5                                                                           # sqrt(dh): 8 at dh = 64
    t, tt = rope_tables(ops, dh)
    o = run_qkvg(ops, x, tt)
    b = qk_backward(ops, x, o, t, seed = 300 + D + H)
    tag = '' if dh == 64 else f' dh={dh}'
    ck = Checks(f'qk_bwd_pack{tag} D={D} H={H}')
    c, s, xx, d64 = b['c'], b['s'], b['x'], b['d64']
    g1 = torch.stack((x['gq'], x['gk'])).double()[None, :, None, :] + 1.                    # [1, 2, 1, 64]
    qb = torch.stack((o['q'], o['k']), 1).double().reshape(M, 2, H, dh)
    # first-order error of the kernel's xhat: the bf16 q / k it reads differ from the float64 values by dq_err; un-rotating mixes the
    # two elements of a rope pair, dividing by sqrt(dh) (gamma_j + 1) amplifies the pair's error by 1 / |gamma_j + 1|
    q_err = (qb - b['qk_ref']).abs()
    Exh = pair_sum(q_err + 4 * U24 * qb.abs()) / (rt * g1.abs())
    nrm = xx.norm(dim = -1, keepdim = True)
    inv = 1. / nrm.clamp_min(1e-12)
    xh = xx * inv
    Dh = rt * g1 * unrope64(d64, c, s)                                                       # d xhat
    dot = (xh * Dh).sum(-1, keepdim = True)
    Edot = (Exh * Dh.abs()).sum(-1, keepdim = True) + 2 * dh * U24 * (xh * Dh).abs().sum(-1, keepdim = True)
    inv_k = o['inv'].double().reshape(M, 2, H, 1)
    rho = (inv_k - inv).abs() / inv + 2 * U24
    ref = b['dx_ref']
    bound = U8 * ref.abs() + (1 + U8) * (rho * ref.abs() + inv * (1 + rho) * (Exh * dot.abs() + (xh.abs() + Exh) * Edot
                                                                             + 4 * U24 * (Dh.abs() + xh.abs() * dot.abs())))
    got = b['out'][:, :2 * HI].reshape(M, 2, H, dh)
    ck(f'qk_bwd{tag} dx', got, ref, bound)
    # gate logits: (1 - sigmoid(g)) dsum; __expf carries |g| 2^-21 relative
    gl, ds = o['gates'].double(), b['dsum'].double()
    sg = torch.sigmoid(gl)
    gref = (1 - sg) * ds
    ck(f'qk_bwd{tag} gate column', b['out'][:, 3 * HI:3 * HI + H], gref, U8 * gref.abs() + (1 + U8) * ds.abs() * (3 * U24 + (1 - sg) * (gl.abs() * 2 ** -21 + 3 * U24)))
    # dgamma as a sum: (a) against the float64 sum of the kernel's own terms sqrt(dh) dy_j xhat'_j (xhat' rebuilt from the bf16 q / k it
    # read); (b) against float64 autograd, with the propagated xhat error added term by term
    dy = unrope64(d64, c, s)
    xh_k = unrope64(qb, c, s) / (rt * g1)
    own = b['dgam0'].double() + (rt * dy * xh_k).sum((0, 2))
    T = (pair_sum(d64.abs()) * pair_sum(qb.abs()) / g1.abs()).sum((0, 2)) + b['dgam0'].double().abs()
    ck(f'qk_bwd{tag} dgamma (own terms)', b['dgam'], own, REL_SUM * T)
    ck(f'qk_bwd{tag} dgamma (autograd)', b['dgam'], b['dgam_ref'], REL_SUM * T + (rt * dy.abs() * Exh).sum((0, 2)))
    # columns qk_bwd_pack must not write: dv (written by the attention backward) and the pad / mix columns
    ck.true('dv columns untouched', untouched(b['out'][:, 2 * HI:3 * HI]))
    ck.true('pad columns untouched', untouched(b['out'][:, 3 * HI + H:]))
    ck.true('guard row untouched', untouched(b['out_buf'][M]))
    ck.done()


@pytest.mark.xfail(strict = True, reason = 'qk_bwd_pack rebuilds xhat from the bf16 q / k; where gamma_j = -1 the forward wrote y_j = 0, so xhat_j is '
                                          'not recoverable from what the forward saves: the kernel returns dx_j = 0 and dgamma_j = 0 instead of '
                                          '-inv xhat_j (xhat . dxhat) and sum 8 dy_j xhat_j')
def test_qk_bwd_pack_at_gamma_minus_one(ops, dh = 64):
    D, H, M = 256, 4, M_ROWS
    x = qkvg_inputs(D, H, False, seed = 400, dh = dh)
    x['gq'][5] = -1.; x['gk'][41] = -1.
    t, tt = rope_tables(ops, dh)
    o = run_qkvg(ops, x, tt)
    b = qk_backward(ops, x, o, t, seed = 401)
    got = b['out'][:, :2 * H * dh].double().reshape(M, 2, H, dh)
    ref = b['dx_ref']
    for which, j in ((0, 5), (1, 41)):
        r = ref[:, which, :, j]
        assert (got[:, which, :, j] - r).abs().max().item() <= 1e-2 * r.abs().max().item(), ('dx', which, j)
        assert abs(b['dgam'][which, j].item() - b['dgam_ref'][which, j].item()) <= 1e-2 * abs(b['dgam_ref'][which, j].item()), ('dgamma', which, j)


# ================================================================================================ gemm_resid
def resid_bounds(y, mag, kb, x_res, sc):
    """y64 (+ bias) over kb k-blocks, the bound of bf16(y), x_out = x_res + y sc and its fp32 bound (sc None: plain residual add)"""
    Ey = c_acc(kb) * mag + U24 * y.abs()
    ys = y if sc is None else y * sc
    xo = x_res + ys
    Exo = (1. if sc is None else sc.abs()) * Ey + 3 * U24 * (x_res.abs() + 2 * ys.abs())
    return U8 * y.abs() + (1 + U8) * Ey, xo, Exo


@pytest.mark.parametrize('D,H,mix', CONFIGS, ids = CFG_IDS)
def test_gemm_resid_vs_float64(ops, cluster_mode, D, H, mix):
    g = gen(500 + D + H)
    M, HI = M_ROWS, 64 * H
    inner = int(D * 4 * 2 / 3); Ip = (inner + 63) // 64 * 64
    nc, Wn, w = 5, 6, 3                                   # zgate table [nc, Wn D] (engine layout), this wrapper at column w D, ld Wn D
    cond = cond_runs(M, nc, seed = D + H)
    zg = torch.rand(nc, Wn * D, device = 'cuda', generator = g)
    ls = torch.randn(D, device = 'cuda', generator = g) * 0.3
    x_res = torch.randn(M, D, device = 'cuda', generator = g)
    cr = cond.long().clamp(min = 0)
    sc = torch.where((cond >= 0)[:, None], zg[cr, w * D:(w + 1) * D], ls + 1.).double()
    ck = Checks(f'resid D={D} H={H}')
    xo_buf, xo = guarded(M, D, F32); yb_buf, yb = guarded(M, D, BF16); xb_buf, xb = guarded(M, D, BF16)

    def check_out(tag, y, mag, kb, s, y_out, x32, x16):
        by, ref, Exo = resid_bounds(y, mag, kb, x_res.double(), s)
        if y_out is not None:
            ck(f'resid {tag} y', y_out, y, by)
        if x32 is not None:
            ck(f'resid {tag} x_out', x32, ref, Exo)
            # accumulator error implied by x_out once its fp32 roundings are taken off: the long-K GEMMs of the layer (K up to 5504)
            smag = (1. if s is None else s.abs()) * mag
            acc = (((x32.double() - ref).abs() - (Exo - c_acc(kb) * smag)).clamp_min(0) / smag.clamp_min(1e-300)).max().item()
            show_c_acc(SHOWN, kb, acc)
        if x16 is not None:
            ck(f'resid {tag} x_out_bf16', x16, ref, U8 * ref.abs() + (1 + U8) * Exo)

    # attention out-projection: K = HI, no bias, fp32 x_out, bf16 y saved for backward
    att = torch.randn(M, HI, device = 'cuda', generator = g).to(BF16)
    Wo = (torch.randn(D, HI, device = 'cuda', generator = g) / HI ** 0.5).to(BF16)
    ops.gemm_resid(att, HI, None, 0, 0, Wo, HI, M, D, HI, None, x_res, xo, None, yb, cond, zg[:, w * D:], Wn * D, ls)
    y, mag = gemm64(att, Wo)
    check_out('attn', y, mag, kblocks(att), sc, yb, xo, None)
    ck.true('attn: guard rows untouched', untouched(xo_buf[M]) and untouched(yb_buf[M]) and untouched(xb_buf))
    # text-only model: no condition table, layerscale on every row
    ops.gemm_resid(att, HI, None, 0, 0, Wo, HI, M, D, HI, None, x_res, xo, None, None, None, None, 0, ls)
    check_out('text-only', y, mag, kblocks(att), (ls.double() + 1.).expand(M, D), None, xo, None)
    # FFN out-projection: K = Ip (pad columns of h and W2 are 0), bias; once with fp32 x_out, once with the bf16 copy only
    h = torch.randn(M, Ip, device = 'cuda', generator = g).to(BF16); h[:, inner:] = 0
    W2 = (torch.randn(D, Ip, device = 'cuda', generator = g) / inner ** 0.5).to(BF16); W2[:, inner:] = 0
    b2 = torch.randn(D, device = 'cuda', generator = g) * 0.2
    y, mag = gemm64(h, W2)
    y = y + b2.double()
    ops.gemm_resid(h, Ip, None, 0, 0, W2, Ip, M, D, Ip, b2, x_res, xo, None, yb, cond, zg[:, w * D:], Wn * D, ls)
    check_out('ffn', y, mag, kblocks(h), sc, yb, xo, None)
    yb.fill_(SENT)
    ops.gemm_resid(h, Ip, None, 0, 0, W2, Ip, M, D, Ip, b2, x_res, None, xb, yb, cond, zg[:, w * D:], Wn * D, ls)
    check_out('ffn bf16-only', y, mag, kblocks(h), sc, yb, None, xb)
    ck.true('ffn: guard rows untouched', untouched(xo_buf[M]) and untouched(yb_buf[M]) and untouched(xb_buf[M]))
    # U-Net skip projection: x_a = x_in + [x_in | skip] W_skip^T, the concatenation read as two operands (K1 = D)
    xin_b = torch.randn(M, D, device = 'cuda', generator = g).to(BF16); skip_b = torch.randn(M, D, device = 'cuda', generator = g).to(BF16)
    Wsk = (torch.randn(D, 2 * D, device = 'cuda', generator = g) / (2 * D) ** 0.5).to(BF16)
    xo.fill_(SENT)
    ops.gemm_resid(xin_b, D, skip_b, D, D, Wsk, 2 * D, M, D, 2 * D, None, x_res, xo, None, None, None, None, 0, None)
    y, mag = gemm64(torch.cat((xin_b, skip_b), 1), Wsk)
    check_out('skip', y, mag, kblocks(Wsk), None, None, xo, None)
    ck.true('skip: guard row untouched', untouched(xo_buf[M]))
    ck.done()


# ================================================================================================ resid_bwd
@pytest.mark.parametrize('D', DISPATCH_D)
def test_resid_bwd_vs_float64(ops, D):
    g = gen(600 + D)
    M, nc, Wn, w = M_ROWS, 5, 6, 3
    cond = cond_runs(M, nc, seed = 7 * D)
    zg = torch.rand(nc, Wn * D, device = 'cuda', generator = g)
    ls = torch.randn(D, device = 'cuda', generator = g) * 0.3
    dx = torch.randn(M, D, device = 'cuda', generator = g)
    y = torch.randn(M, D, device = 'cuda', generator = g).to(BF16)
    dx64, y64 = dx.double(), y.double()
    ck = Checks(f'resid_bwd D={D}')
    for form in ('ffn', 'attn', 'text-only', 'skip'):
        use_cond = form in ('ffn', 'attn')
        dy_buf, dy = guarded(M, D, BF16)
        dzg = torch.randn(nc, Wn * D, device = 'cuda', generator = g) * 0.1
        dls_buf, dls = guarded(1, D, F32); dls.normal_(generator = g)
        db_buf, db = guarded(1, D, F32); db.normal_(generator = g)
        dzg0, dls0, db0 = dzg.clone(), dls.clone(), db.clone()
        if form == 'skip':
            ops.resid_bwd(dx, None, None, None, 0, None, dy, None, 0, None, None, M, D)
            ck('resid_bwd skip dy', dy, dx64, U8 * dx64.abs())
            ck.true('skip: guard row untouched', untouched(dy_buf[M]))
            continue
        ops.resid_bwd(dx, y, cond if use_cond else None, zg[:, w * D:] if use_cond else None, Wn * D, ls, dy,
                      dzg[:, w * D:] if use_cond else None, Wn * D, dls[0], db[0] if form != 'attn' else None, M, D)
        isM = (cond >= 0) if use_cond else torch.zeros(M, dtype = torch.bool, device = 'cuda')
        cr = cond.long().clamp(min = 0)
        s = torch.where(isM[:, None], zg[cr, w * D:(w + 1) * D], ls + 1.).double()
        dref = dx64 * s
        ck(f'resid_bwd {form} dy', dy, dref, U8 * dref.abs() + (1 + U8) * 2 * U24 * dref.abs())
        prod = dx64 * y64
        if use_cond:
            rows = torch.nonzero(isM).squeeze(1)
            want = torch.zeros(nc, D, dtype = F64, device = 'cuda').index_add_(0, cr[rows], prod[rows])
            scale = torch.zeros(nc, D, dtype = F64, device = 'cuda').index_add_(0, cr[rows], prod[rows].abs())
            sl = slice(w * D, (w + 1) * D)
            ck(f'resid_bwd {form} dzgate', dzg[:, sl], dzg0[:, sl].double() + want, REL_SUM * (scale + dzg0[:, sl].double().abs()))
            ck.true(f'{form}: other wrappers\' dzgate columns untouched', same_bits(dzg[:, :w * D], dzg0[:, :w * D]) and same_bits(dzg[:, (w + 1) * D:], dzg0[:, (w + 1) * D:]))
        text = ~isM
        ck(f'resid_bwd {form} dlayerscale', dls[0], dls0[0].double() + prod[text].sum(0), REL_SUM * (prod[text].abs().sum(0) + dls0[0].double().abs()))
        if form != 'attn':
            ck(f'resid_bwd {form} dbias', db[0], db0[0].double() + dref.sum(0), REL_SUM * (dref.abs().sum(0) + db0[0].double().abs()))
        else:
            ck.true('attn: dbias untouched without a bias', same_bits(db, db0))
        ck.true(f'{form}: guard rows untouched', untouched(dy_buf[M]) and untouched(dls_buf[1]) and untouched(db_buf[1]))
    ck.done()


# ================================================================================================ GEGLU forward
def phi_cdf(g):
    return 0.5 * torch.erfc(-g / 2 ** 0.5), torch.exp(-0.5 * g * g) / (2 * np.pi) ** 0.5


def gelu_err(g):
    """bounds of the kernel's errors in Phi(g) and phi(g) (gelu_parts): the A-S polynomial, and __expf's ~|g^2| 2^-24 relative error
    on the small tail term"""
    Phi, phi = phi_cdf(g)
    tail = torch.minimum(Phi, 1 - Phi)
    return PHI_ABS + tail * (g * g + 16) * U24, phi * (g * g + 8) * U24


def packed_w1(D, inner, g):
    src = torch.from_numpy(E.w1_row_src(inner)).cuda()
    valid = src >= 0
    W1 = torch.randn(2 * inner, D, device = 'cuda', generator = g) / D ** 0.5
    b1 = torch.randn(2 * inner, device = 'cuda', generator = g) * 0.3
    Wp = torch.zeros(src.numel(), D, device = 'cuda'); bp = torch.zeros(src.numel(), device = 'cuda')
    Wp[valid] = W1[src[valid]]; bp[valid] = b1[src[valid]]
    return Wp.to(BF16), bp, src


def split_vg(t, Ip):
    """[M, 2 Ip] tile-interleaved -> value [M, Ip], gate [M, Ip]"""
    t = t.reshape(t.shape[0], Ip // 64, 2, 64)
    return t[:, :, 0].reshape(-1, Ip), t[:, :, 1].reshape(-1, Ip)


def merge_vg(v, g):
    """value [M, Ip], gate [M, Ip] -> [M, 2 Ip] tile-interleaved"""
    M, Ip = v.shape
    return torch.stack((v.reshape(M, Ip // 64, 64), g.reshape(M, Ip // 64, 64)), 2).reshape(M, 2 * Ip)


_MASKS = {}


def ffn_keep(key, p, layer, M, cols):
    k = (key, p, layer, M, cols)
    if k not in _MASKS:
        _MASKS.clear()
        _MASKS[k] = torch.from_numpy(keep_mask(key, p, SITE_FFN, layer, 0, np.arange(M), np.arange(cols))).cuda()
    return _MASKS[k]


DROP_KEY, DROP_P, DROP_LAYER = (0x2468ACE, 0x1357BDF), 0.1, 3


def dev_key(k):
    return torch.from_numpy(np.array(k, dtype = np.uint32).view(np.int32)).cuda()


@pytest.mark.parametrize('D,H,mix', CONFIGS, ids = CFG_IDS)
def test_gemm_geglu_vs_float64(ops, cluster_mode, D, H, mix):
    g = gen(700 + D + H)
    M = M_ROWS
    inner = int(D * 4 * 2 / 3); Ip = (inner + 63) // 64 * 64
    Wp, bp, src = packed_w1(D, inner, g)
    u = torch.randn(M, D, device = 'cuda', generator = g).to(BF16)
    ck = Checks(f'geglu D={D} inner={inner}')
    keep = ffn_keep(DROP_KEY, DROP_P, DROP_LAYER, M, Ip)
    sc = drop_scale(DROP_P)
    out = {}
    for drop in (False, True):
        vg_buf, vg = guarded(M, 2 * Ip, BF16); h_buf, h = guarded(M, Ip, BF16)
        if drop:
            ops.gemm_geglu_drop(u, D, Wp, D, bp, M, 2 * Ip, D, vg, h, dev_key(DROP_KEY), DROP_P, DROP_LAYER)
        else:
            ops.gemm_geglu(u, D, Wp, D, bp, M, 2 * Ip, D, vg, h)
        out[drop] = vg_buf, vg, h_buf, h
    # the float64 reference in row chunks of at most REF_VALUES entries of [rows, 2 Ip]
    n_chunks = -(-M * 2 * Ip // REF_VALUES)
    step = -(-M // n_chunks)
    for r0 in range(0, M, step):
        rs = slice(r0, min(r0 + step, M))
        y, mag = gemm64(u[rs], Wp)
        y = y + bp.double()
        Ey = c_acc(kblocks(u)) * mag + U24 * y.abs()
        v, gt = split_vg(y, Ip)
        Ev, Eg = split_vg(Ey, Ip)
        Phi, phi = phi_cdf(gt)
        dPhi, _ = gelu_err(gt)
        href = v * gt * Phi
        Eh = v.abs() * (Phi + gt.abs() * phi) * Eg + (gt * Phi).abs() * Ev + v.abs() * gt.abs() * dPhi + 4 * U24 * href.abs()
        for drop in (False, True):
            _, vg, _, h = out[drop]
            tag = 'geglu_drop' if drop else 'geglu'
            ck(f'{tag} vg', vg[rs], y, U8 * y.abs() + (1 + U8) * Ey, row0 = r0)
            want, Ew = (href * keep[rs] * sc, (Eh + U24 * href.abs()) * sc) if drop else (href, Eh)
            ck(f'{tag} h', h[rs, :inner], want[:, :inner], U8 * want[:, :inner].abs() + (1 + U8) * Ew[:, :inner], row0 = r0)
    for drop in (False, True):
        vg_buf, vg, h_buf, h = out[drop]
        tag = 'geglu_drop' if drop else 'geglu'
        ck.true(f'{tag}: pad columns of h exactly 0', bool((h[:, inner:].view(torch.int16) == 0).all()))
        if drop:
            ck.true('dropped h entries exactly 0', bool((h[:, :inner][~keep[:, :inner]].view(torch.int16) == 0).all()))
        ck.true(f'{tag}: guard rows untouched', untouched(vg_buf[M]) and untouched(h_buf[M]))
    ck.done()


# ================================================================================================ GEGLU backward + bias column sums
@pytest.mark.parametrize('D', DISPATCH_D)
def test_geglu_bwd_vs_float64(ops, D):
    g = gen(800 + D)
    M = M_ROWS
    rpb = ops.lib.tfx_geglu_bwd_rows_per_block()
    assert M % rpb != 0
    nblk = (M + rpb - 1) // rpb
    inner = int(D * 4 * 2 / 3); Ip = (inner + 63) // 64 * 64
    src = torch.from_numpy(E.w1_row_src(inner)).cuda()
    OFF = 37                                               # the layer's bias inside the flat gradient buffer
    cols = torch.where(src >= 0, src + OFF, torch.full_like(src, -1)).to(I32)
    vals = torch.randn(M, 2 * Ip, device = 'cuda', generator = g) * 1.5
    vals[:, (src < 0).nonzero().squeeze(1)] = 0            # the packed W1 / bias pad rows are 0, so is vg there
    vg = vals.to(BF16)
    dh = torch.randn(M, Ip, device = 'cuda', generator = g).to(BF16); dh[:, inner:] = 0
    v, gt = (t.double() for t in split_vg(vg, Ip))
    Phi, phi = phi_cdf(gt)
    dPhi, dphi = gelu_err(gt)
    keep = ffn_keep(DROP_KEY, DROP_P, DROP_LAYER, M, Ip)
    ck = Checks(f'geglu_bwd D={D} inner={inner}')
    for drop in (False, True):
        dvg_buf, dvg = guarded(M, 2 * Ip, BF16)
        part_buf, part = guarded(nblk, 2 * Ip, F32)
        if drop:
            ops.geglu_bwd_drop(dh, vg, dvg, M, Ip, None, None, part, dev_key(DROP_KEY), DROP_P, DROP_LAYER)
        else:
            ops.geglu_bwd(dh, vg, dvg, M, Ip, None, None, part)
        out = torch.full((OFF + 2 * inner + 9,), SENT, device = 'cuda')
        out[OFF:OFF + 2 * inner] = torch.randn(2 * inner, device = 'cuda', generator = g)
        out0 = out.clone()
        ops.colsum_f32(part, 2 * Ip, nblk, 2 * Ip, cols, out)
        tag = 'geglu_bwd_drop' if drop else 'geglu_bwd'
        d = dh.double() * (keep * drop_scale(DROP_P) if drop else 1.)
        dv_ref, dg_ref = d * gt * Phi, d * v * (Phi + gt * phi)
        Edv = d.abs() * gt.abs() * dPhi + 4 * U24 * dv_ref.abs()
        Edg = d.abs() * v.abs() * (dPhi + gt.abs() * dphi) + 6 * U24 * d.abs() * v.abs() * (Phi + (gt * phi).abs())
        got_v, got_g = split_vg(dvg, Ip)
        ck(f'{tag} d value', got_v, dv_ref, U8 * dv_ref.abs() + (1 + U8) * Edv)
        ck(f'{tag} d gate', got_g, dg_ref, U8 * dg_ref.abs() + (1 + U8) * Edg)
        ck.true(f'{tag}: guard rows untouched', untouched(dvg_buf[M]) and untouched(part_buf[nblk]))
        # bias gradient: the fp32 column sums of the kernel's terms, through the engine's b1 column map
        terms, errs = merge_vg(dv_ref, dg_ref), merge_vg(Edv, Edg)
        valid = src >= 0
        want = torch.zeros(2 * inner, dtype = F64, device = 'cuda'); want[src[valid]] = terms.sum(0)[valid]
        scale = torch.zeros_like(want); scale[src[valid]] = (terms.abs() + errs).sum(0)[valid]
        syst = torch.zeros_like(want); syst[src[valid]] = errs.sum(0)[valid]
        ck(f'{tag} dbias (colsum_f32)', out[OFF:OFF + 2 * inner], out0[OFF:OFF + 2 * inner].double() + want,
           REL_SUM * (scale + out0[OFF:OFF + 2 * inner].double().abs()) + syst)
        ck.true(f'{tag}: entries outside the column map untouched', untouched(out[:OFF]) and untouched(out[OFF + 2 * inner:]))
    ck.done()
