"""GPU: the AttentionResidual kernels against float64, at every model width and across the chunk boundaries of the deferred backward.

    attn_residual_fwd_h16  x_out = sum_l a_l h_l,  a = softmax_l(sim),  sim_l = <h_l, w> / max(|h_l|, 1e-12),  w = (gamma + 1) pq,
                           over bf16 hiddens h_0 .. h_{L1-1}; x_out fp32, its bf16 copy and the log-sum-exp of the softmax (both optional)
    attn_residual_bwd2     the deferred backward of a stack of AttentionResiduals (layer i mixes h_0 .. h_{i+1}, loss sum_i <x_i, R_i>): per
                           layer the scalars (a, c1, c2) of its earlier hiddens, the complete gradient of its newest hidden, and d gamma / d pq
                           through the per-block partial sums that attn_res_bwd_finish_k folds; then the gradient of h_0 by the own = 0 assembly

Each entry point is called through the C ABI as engine.forward / engine.backward call it: the forward with and without x_out_bf16 and lse,
n_later = 0 with the dummy pointer lists, scalars_later pointing at [token 0][k][0] of tables of (depth + 2) * 3 floats per row, and the
x0 assembly with own = 0 and gammas[0] unused.

Reference and bounds (|got - ref| <= bound element-wise; the worst err / bound of each check is printed, run with -s):
  - references are float64 from the same bf16 hiddens and fp32 gamma / pq, the norm clamped as F.normalize clamps it.  The backward
    reference is the closed form of the deferred assembly (a, ds, c1, c2 per layer and hidden, summed over the later layers), evaluated in
    row chunks; test_reference_backward_matches_autograd holds it to float64 autograd of the stacked AttentionResidual.
  - a row reduction of the kernels sums NCH * 4 terms per lane, then 5 butterfly levels: at most NSUM = NCH * 4 + 5 fp32 roundings
    (2^-24 relative each) of the sum of |terms|, one more for the products, two more for the kernel's fp32 w.
  - __expf is within (2 + 1.173 |x|) ulp and flushes results below 2^-126 to zero; __logf is within 2^-21.41 absolute on [0.5, 2] and
    3 ulp elsewhere.  The online softmax multiplies each term by at most L1 rescale factors whose exponents sum to at most the row's
    sim range, and rounds at most twice per step.
  - x_out: sum_l a_l |h_l| times (those exp and rounding terms + the sim error of l + the a-weighted sim error of the row).  lse: absolute.
  - G: relative to the magnitude sum  sum_i' [a |dx| + |c1| |w| + |c2| |h|],  with the error of each scalar carried through.  ds =
    a (<h, dx> - <x_out, dx>) cancels (identical hiddens cancel it exactly), so its error is carried through |h| |dx| + |x_out| |dx|, and
    the exact effect of the forward's x_out and lse (kernel outputs, float64 reference values) is part of the bound.
  - d gamma / d pq: REL_SUM times (the sum of |terms| + |initial value|) plus the carried error of c1; they start from non-zero values.
  - x_out_bf16 is compared bit for bit with torch's round-to-nearest cast of x_out; calls without x_out_bf16 / lse write the same x_out.
  - bytes a kernel must not write (a guard row after every output and scalar table, a guard float after the workspace and the parameter
    gradients, the scalar slots k >= L1 - 1 a layer does not write) are compared bit for bit.  The scalar tables, the workspace and G
    (before its storing launch) start as NaN: a read of anything the kernels did not write turns a result into NaN.
Rows: the forward grid is persistent and holds at most 64 warps per SM, so M is a prime above twice that many warps (every warp walks two
rows or more), and above five times that at L1 <= 3, where the 4-slot cp.async ring then holds items of several rows at once.  The backward
uses M = 2053: prime, 33 blocks of 64 rows (the last warp's 8-row chunk partial), so attn_res_bwd_finish_k folds 16 + 16 + 1 blocks.
Inputs: every hidden has an all-zero row, rows below the 1e-12 clamp (|h| = 0.9e-12, 0.5e-12, 1e-13, and 0.9e-12 mostly aligned with w) and
a row with a large dynamic range; further rows have identical hiddens, every hidden zero, every hidden below the clamp, and one hidden
aligned with w and the others against it (sim differences of 2 |w|: about 100 at D = 128 and the trained-like scale, more at larger
widths).  Parameters are at a trained-like scale (gamma ~ N(0, 0.5^2) with every 17th column exactly -1, pq ~ N(0, 4^2)) and at the
model's initial scale (gamma = 0, pq ~ N(0, 0.02^2): a nearly uniform softmax)."""
import ctypes
import math

import pytest
import torch

from helpers import SENT, Checks as _Checks, gen, guarded, same_bits, untouched
from transfusion_pytorch_b200 import _lib
from transfusion_pytorch_b200.transfusion import MODEL_DIMS

pytestmark = pytest.mark.gpu
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U23, U24 = 2.0 ** -23, 2.0 ** -24
EPS = 1e-12
TINY = 2.0 ** -149                     # absolute rounding error of a subnormal fp32 result
FLUSH = 2.0 ** -125                    # __expf results below 2^-126 are flushed to zero
REL_SUM = 1e-6                         # sums / atomics, relative to sum |terms| + |initial| (the value test_block_epilogues_gpu.py uses)
FWD_RING = 4                           # ARES_FWD_RING of rowops.cu
BWD2_ROWS = 64                         # rows per attn_res_bwd2_k block: 8 warps of 8 rows
FOLD = 16                              # partial-sum rows per attn_res_bwd_finish_k y-block
M_BWD = 2053
CHUNK = 1024                           # rows per float64 reference chunk
# Measured worst err / bound on an H100 80GB HBM3 (700 W power limit), with the constants above: x_out 0.043 (trained scale) and 0.096
# (initial scale), lse 0.090 and 0.095; stored scalars a 0.64, c1 0.30, c2 0.27; G 0.40; d gamma 0.075, d pq 0.020.  The float64 closed
# form against autograd: 1.5e-3 of its 1e-9 bound.

FWD_CASES = [(D, L1) for L1 in (1, 2, 3, 12) for D in MODEL_DIMS] + [
    (256, 11), (1024, 11), (384, 21), (512, 21), (128, 22), (768, 22), (128, 65), (768, 65)]
# every width at depth 11 (layer 0 assembles exactly one chunk of 10 later layers, the x0 assembly 10 -> 11); depth 1 (n_later = 0 and a
# one-layer x0 assembly); depth 21 / 22 (three chunks); depth 64 (seven)
BWD_CASES = [(D, 11) for D in MODEL_DIMS] + [(128, 1), (768, 1), (256, 21), (1024, 22), (128, 64), (384, 64)]

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


def is_prime(n):
    return n > 1 and all(n % p for p in range(2, math.isqrt(n) + 1))


def prime_above(n):
    n += 1
    while not is_prime(n):
        n += 1
    return n


def resident_warps():
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count * (p.max_threads_per_multi_processor // 32)


def fwd_rows(L1):
    return prime_above((5 if L1 < FWD_RING else 2) * resident_warps())


class Ptrs:
    """ctypes pointer arrays kept alive for the duration of a test"""

    def __init__(self):
        self.keep = []

    def __call__(self, ts):
        a = (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
        self.keep.append(a)
        return ctypes.cast(a, ctypes.c_void_p)


def worst_piece(ck, name, pieces):
    """one check over (got, ref, bound) pieces of an output too large for one float64 reference: the worst piece is reported"""
    worst = None
    for got, ref, bound in pieces:
        r = ((got.double() - ref).abs() / bound.clamp_min(1e-300)).nan_to_num(nan = float('inf')).max().item()
        if worst is None or r > worst[0]:
            worst = (r, got, ref, bound)
    ck(name, *worst[1:])


def nan_filled(shape):
    return torch.full(shape, float('nan'), device = 'cuda')


def all_nan(t):
    return same_bits(t, torch.full_like(t, float('nan')))


# ------------------------------------------------------------------------------------------------ inputs
def params(D, initial, g):
    """(gamma, pq) fp32: the model's initial scale, or a trained-like scale with every 17th gamma column exactly -1 (w = 0 there)"""
    if initial:
        return torch.zeros(D, device = 'cuda'), torch.randn(D, device = 'cuda', generator = g) * 0.02
    gamma = torch.randn(D, device = 'cuda', generator = g) * 0.5
    gamma[::17] = -1.
    return gamma, torch.randn(D, device = 'cuda', generator = g) * 4.


def w64(gamma, pq):
    return (gamma.double() + 1.) * pq.double()


def unit(v):
    return v / v.norm()


def make_hiddens(L1, M, D, align, g):
    """L1 bf16 hiddens [M, D]; the special rows of hidden l align with align[l] (a float64 w).  Rows of hidden l: 100 + l all zero,
    200 + 4 l + (0, 1, 2) below the clamp in a random direction, 203 + 4 l below the clamp and mostly aligned, 500 + l with a large dynamic
    range.  Rows of every hidden: 1 identical, 2 / 3 aligned with align[l] for the last / first hidden and against it for the others, 5 zero,
    6 below the clamp, 7 large."""
    hs = []
    s = D ** 0.5
    first = torch.randn(D, device = 'cuda', generator = g)
    for l in range(L1):
        h = torch.randn(M, D, device = 'cuda', generator = g)
        u = unit(align[l].float())
        h[100 + l] = 0.
        for j, nrm in enumerate((0.9e-12, 0.5e-12, 1e-13)):
            h[200 + 4 * l + j] = unit(h[200 + 4 * l + j]) * nrm
        h[203 + 4 * l] = unit(u + 0.1 * D ** -0.5 * torch.randn(D, device = 'cuda', generator = g)) * 0.9e-12
        h[500 + l] *= 10. ** (torch.rand(D, device = 'cuda', generator = g) * 6 - 3)
        h[1] = first
        h[2] = u * s * (1 if l == L1 - 1 else -1)
        h[3] = u * s * (1 if l == 0 else -1)
        h[5] = 0.
        h[6] = unit(h[6]) * 0.7e-12
        h[7] *= 10. ** (torch.rand(D, device = 'cuda', generator = g) * 6 - 3)
        hs.append(h.to(BF16))
    return hs


# ------------------------------------------------------------------------------------------------ float64 reference
class Row:
    """float64 forward quantities of a chunk of rows: H [L1, m, D] the hiddens, w the layer's w"""

    def __init__(self, H, w):
        self.H = H
        self.nrm = H.norm(dim = -1)
        self.n = self.nrm.clamp_min(EPS)
        self.dot = torch.einsum('lmd,d->lm', H, w)
        self.sim = self.dot / self.n
        self.lse = self.sim.logsumexp(0)
        self.a = (self.sim - self.lse).exp()
        self.x = torch.einsum('lm,lmd->md', self.a, H)
        self.habs_w = torch.einsum('lmd,d->lm', H.abs(), w.abs())

    def sim_err(self, D):
        """bound on |sim_kernel - sim| and on the relative error of the kernel's 1 / max(|h|, eps)"""
        ns = nsum(D) + 1
        rho = (ns / 2 + 2) * U24
        return (ns + 2) * U24 * self.habs_w / self.n + self.sim.abs() * (rho + U24), rho


def fwd_reference(H, w, D):
    """x, lse and their bounds for a chunk of rows"""
    r = Row(H, w)
    L1 = H.shape[0]
    delta, _ = r.sim_err(D)
    rng = r.sim.max(0).values - r.sim.min(0).values
    e_exp = U23 * (2 * (L1 + 1) + 3.4 * rng)
    adelta = (r.a * delta).sum(0)
    coef = r.a * (2 * e_exp + (5 * L1 + 4) * U24 + delta + adelta + (r.a < 2 ** -118).double())
    Ex = torch.einsum('lm,lmd->md', coef, H.abs()) + (2 * L1 + 2) * TINY
    El = adelta + e_exp + (2 * L1 + 1) * U24 + 2 ** -21.41 + 3 * math.log(L1) * U23 + 2 * U24 * r.lse.abs()
    return r.x, r.lse, Ex, El


def layer_scalars(H, w, dx, D, xo = None, lse_k = None):
    """a, c1, c2 [L1, m] of one layer over a chunk of rows (c2 = 0 below the clamp, where the clamped norm is a constant), the layer's d w
    contribution, and, given the kernel's x_out / lse for these rows, the bounds on the kernel's a, c1, c2"""
    r = Row(H, w)
    da = torch.einsum('lmd,md->lm', H, dx)
    diff = da - (r.x * dx).sum(-1)
    ds = r.a * diff
    c1 = ds / r.n
    live = r.nrm >= EPS
    c2 = torch.where(live, ds * r.dot / r.n ** 3, torch.zeros_like(ds))
    out = dict(a = r.a, c1 = c1, c2 = c2, dw = torch.einsum('lm,lmd->d', c1, H))
    if xo is not None:
        ns = nsum(D) + 1
        delta, rho = r.sim_err(D)
        arg = (r.sim - r.lse).abs()
        eps_a = delta + (lse_k - r.lse).abs() + (2 + 1.7 * arg) * U23
        flushed = (r.a < FLUSH).double()                                                   # a = 0 in the kernel
        xo = xo.double()
        e_diff = (ns * U24 * (torch.einsum('lmd,md->lm', H.abs(), dx.abs()) + (xo.abs() * dx.abs()).sum(-1)) + ((xo - r.x) * dx).sum(-1).abs()
                  + U24 * diff.abs())
        e_ds = ds.abs() * (eps_a + U24 + flushed) + r.a * e_diff + TINY
        e_c1 = e_ds / r.n + c1.abs() * (rho + U24) + TINY
        e_dot = (ns + 2) * U24 * r.habs_w
        e_c2 = torch.where(live, (e_ds * r.dot.abs() + ds.abs() * e_dot) / r.n ** 3 + c2.abs() * (3 * rho + 4 * U24) + TINY, torch.zeros_like(ds))
        out.update(ea = r.a * eps_a + FLUSH * flushed, ec1 = e_c1, ec2 = e_c2, dw_abs = torch.einsum('lm,lmd->d', c1.abs(), H.abs()),
                   dw_err = torch.einsum('lm,lmd->d', e_c1, H.abs()))
    return out


def stack_reference(hb, ws, R, xo = None, lse_k = None):
    """scalars [depth, depth + 1, M] (a, c1, c2, and their bounds given the kernel forward) and d w per layer of a stack of
    AttentionResiduals, computed in row chunks"""
    depth, (M, D) = len(ws), hb[0].shape
    names = ('a', 'c1', 'c2') + (('ea', 'ec1', 'ec2') if xo is not None else ())
    sc = {k: torch.zeros(depth, depth + 1, M, dtype = F64, device = 'cuda') for k in names}
    dw = {k: torch.zeros(depth, D, dtype = F64, device = 'cuda') for k in (('dw', 'dw_abs', 'dw_err') if xo is not None else ('dw',))}
    for r0 in range(0, M, CHUNK):
        r1 = min(M, r0 + CHUNK)
        Hall = torch.stack([h[r0:r1] for h in hb]).double()
        for i in range(depth):
            kern = (xo[i][r0:r1], lse_k[i][r0:r1].double()) if xo is not None else ()
            out = layer_scalars(Hall[:i + 2], ws[i], R[i][r0:r1].double(), D, *kern)
            for k in names:
                sc[k][i, :i + 2, r0:r1] = out[k]
            for k in dw:
                dw[k][i] += out[k]
    return sc, dw


def assemble(k, hb, ws, R, sc):
    """G_k = sum over the layers that mix hidden k of [a dx + c1 w] - (sum c2) h_k, the magnitude sum of its terms, and (with the scalar
    bounds of sc) the bound on the kernel's G_k"""
    layers = range(max(k - 1, 0), len(ws))
    h = hb[k].double()
    G, T = torch.zeros_like(h), torch.zeros_like(h)
    E = torch.zeros_like(h) if 'ea' in sc else None
    for i in layers:
        dx, w = R[i].double(), ws[i]
        a, c1 = sc['a'][i, k, :, None], sc['c1'][i, k, :, None]
        G += a * dx + c1 * w
        T += a * dx.abs() + c1.abs() * w.abs()
        if E is not None:
            E += sc['ea'][i, k, :, None] * dx.abs() + (sc['ec1'][i, k, :, None] + 2 * U24 * c1.abs()) * w.abs()
    G -= sc['c2'][layers, k].sum(0)[:, None] * h
    T += sc['c2'][layers, k].abs().sum(0)[:, None] * h.abs()
    if E is None:
        return G, T, None
    n = len(layers)
    E += sc['ec2'][layers, k].sum(0)[:, None] * h.abs() + (3 * n + 6) * U24 * T + U24 * G.abs() + (3 * n + 6) * TINY
    return G, T, E


def ares_ref(hs, gam, pq):
    """float64 AttentionResidual (T.py:803-829): x = sum_l softmax_l(<normalize(h_l) sqrt(D) (gam + 1), pq> / sqrt(D)) h_l"""
    vals = torch.stack(hs)
    D = vals.shape[-1]
    keys = torch.nn.functional.normalize(vals, dim = -1, eps = EPS) * D ** 0.5 * (gam + 1)
    sim = torch.einsum('lnd,d->nl', keys, pq) * D ** -0.5
    return torch.einsum('nl,lnd->nd', sim.softmax(-1), vals)


def stack_inputs(depth, M, D, seed):
    """hiddens, fp32 (gamma, pq) per layer (every third layer at the initial scale) and the incoming gradients R of a stack; hidden l's
    special rows align with the w of the layer that produced it (layer l - 1; layer 0 for x0)"""
    g = gen(seed)
    gam, pq = zip(*[params(D, i % 3 == 1, g) for i in range(depth)])
    ws = [w64(a, b) for a, b in zip(gam, pq)]
    hb = make_hiddens(depth + 1, M, D, [ws[max(l - 1, 0)] for l in range(depth + 1)], g)
    R = [torch.randn(M, D, device = 'cuda', generator = g) for _ in range(depth)]
    return hb, list(gam), list(pq), ws, R


# ------------------------------------------------------------------------------------------------ rows
def test_rows_cover_every_warp_and_fold():
    """forward: M prime and above 2 (5 at L1 < 4) times the warps an SM can hold, for every SM; backward: one partial-sum row per block of
    64 rows, three y-blocks of the fold, the last partial"""
    assert resident_warps() >= 64 * torch.cuda.get_device_properties(0).multi_processor_count
    for L1 in (1, 2, 3, 4, 65):
        M = fwd_rows(L1)
        assert is_prime(M) and M > (5 if L1 < FWD_RING else 2) * resident_warps()
    ws_rows = int(_lib.load().tfx_attn_residual_bwd_workspace_floats(M_BWD, 128)) // 128
    assert is_prime(M_BWD) and M_BWD % 8
    assert ws_rows == -(-M_BWD // BWD2_ROWS) == 33 and ws_rows > 2 * FOLD and ws_rows % FOLD


# ================================================================================================ forward
@pytest.mark.parametrize('D,L1', FWD_CASES)
def test_attn_residual_fwd_vs_float64(ops, D, L1):
    ck = Checks(f'attn_residual_fwd D={D} L1={L1}')
    M = fwd_rows(L1)
    P = Ptrs()
    for initial in (False, True):
        tag = 'initial scale' if initial else 'trained scale'
        g = gen(1000 * L1 + D + initial)
        gamma, pq = params(D, initial, g)
        w = w64(gamma, pq)
        hb = make_hiddens(L1, M, D, [w] * L1, g)
        xob, xo = guarded(M, D, F32); xbb, xb = guarded(M, D, BF16); lb, lse = guarded(M, 1, F32)
        ops.attn_residual_fwd_h16(P(hb), L1, gamma, pq, xo, xb, lse, M, D)                 # training
        x2b, xo2 = guarded(M, D, F32); b2b, xb2 = guarded(M, D, BF16)
        ops.attn_residual_fwd_h16(P(hb), L1, gamma, pq, xo2, xb2, None, M, D)              # eval: no lse
        x3b, xo3 = guarded(M, D, F32); l3b, lse3 = guarded(M, 1, F32)
        ops.attn_residual_fwd_h16(P(hb), L1, gamma, pq, xo3, None, lse3, M, D)             # no bf16 copy
        pieces, step = [], max(256, (1 << 25) // (L1 * D))                                  # float64 chunks of at most 256 MB
        for r0 in range(0, M, step):
            r1 = min(M, r0 + step)
            x, l, Ex, El = fwd_reference(torch.stack([h[r0:r1] for h in hb]).double(), w, D)
            pieces.append(((xo[r0:r1], x, Ex), (lse[r0:r1, 0], l, El)))
        worst_piece(ck, f'{tag} x_out', (p[0] for p in pieces))
        worst_piece(ck, f'{tag} lse', (p[1] for p in pieces))
        ck.true(f'{tag}: x_out_bf16 = bf16(x_out)', same_bits(xb, xo.to(BF16)))
        ck.true(f'{tag}: zero row in every hidden: x_out = 0', bool((xo[5] == 0).all()))
        ck.true(f'{tag}: calls without lse / x_out_bf16 write the same x_out, x_out_bf16, lse',
                same_bits(xo2, xo) and same_bits(xb2, xb) and same_bits(xo3, xo) and same_bits(lse3, lse))
        ck.true(f'{tag}: guard rows untouched', all(untouched(b[M]) for b in (xob, xbb, lb, x2b, b2b, x3b, l3b)))
    ck.done()


# ================================================================================================ deferred backward
def run_stack_backward(ops, hb, gam, pq, R, M, D):
    """forward of every layer, then the deferred backward in engine.backward's order and call pattern; returns the outputs (guarded
    buffers) and the initial values of the parameter gradients"""
    depth = len(gam)
    P = Ptrs()
    xo = [torch.empty(M, D, device = 'cuda') for _ in range(depth)]
    lse = [torch.empty(M, device = 'cuda') for _ in range(depth)]
    for i in range(depth):
        ops.attn_residual_fwd_h16(P(hb[:i + 2]), i + 2, gam[i], pq[i], xo[i], None, lse[i], M, D)
    stride = (depth + 2) * 3
    sc = nan_filled((depth, M + 1, depth + 2, 3))
    sc[:, M] = SENT                                                                    # each table's guard row
    Gb = [guarded(M, D, F32)[0] for _ in range(depth + 1)]
    for b in Gb:
        b[:M] = float('nan')
    g0 = gen(7 + depth + D)
    dgb = [torch.randn(D + 1, device = 'cuda', generator = g0) for _ in range(depth)]       # accumulated into; the last float is a guard
    dpb = [torch.randn(D + 1, device = 'cuda', generator = g0) for _ in range(depth)]
    init = ([t.clone() for t in dgb], [t.clone() for t in dpb])
    nws = int(ops.lib.tfx_attn_residual_bwd_workspace_floats(M, D))
    ws = nan_filled((nws + 1,))
    ws[nws] = SENT
    for i in reversed(range(depth)):
        later = list(range(i + 1, depth))
        ops.attn_residual_bwd2(P(hb[:i + 2]), i + 2, 1, P([gam[j] for j in [i] + later]), P([pq[j] for j in [i] + later]),
                               P([R[j] for j in later] or [R[i]]), P([sc[j][0, i + 1] for j in later] or [R[i]]), len(later), R[i], xo[i], lse[i],
                               Gb[i + 1][:M], sc[i], stride, dgb[i][:D], dpb[i][:D], ws[:nws], M, D)
    ops.attn_residual_bwd2(P(hb[:1]), 1, 0, P([gam[0]] + gam), P([pq[0]] + pq), P(R), P([sc[j][0, 0] for j in range(depth)]), depth,
                           None, None, None, Gb[0][:M], None, stride, None, None, None, M, D)
    return dict(xo = xo, lse = lse, sc = sc, G = Gb, dg = dgb, dp = dpb, ws = ws, init = init)


@pytest.mark.parametrize('D,depth', BWD_CASES)
def test_attn_residual_backward_vs_float64(ops, D, depth):
    ck = Checks(f'attn_residual_bwd2 D={D} depth={depth}')
    M = M_BWD
    hb, gam, pq, ws, R = stack_inputs(depth, M, D, 31 * depth + D)
    out = run_stack_backward(ops, hb, gam, pq, R, M, D)
    ref, dw = stack_reference(hb, ws, R, out['xo'], out['lse'])
    # the scalars layer i stores for its earlier hiddens h_0 .. h_i (slots k = 0 .. i)
    for j, (name, e) in enumerate((('a', 'ea'), ('c1', 'ec1'), ('c2', 'ec2'))):
        worst_piece(ck, f'scalars {name}', ((out['sc'][i][:M, :i + 1, j], ref[name][i, :i + 1].T, ref[e][i, :i + 1].T) for i in range(depth)))

    def G_pieces():
        for k in range(depth + 1):
            G, _, E = assemble(k, hb, ws, R, ref)
            yield out['G'][k][:M], G, E
    worst_piece(ck, 'G', G_pieces())
    for name, bufs, inits, fac in (('d gamma', out['dg'], out['init'][0], [t.double() for t in pq]),
                                   ('d pq', out['dp'], out['init'][1], [t.double() + 1. for t in gam])):
        worst_piece(ck, name, ((bufs[i][:D], inits[i][:D].double() + fac[i] * dw['dw'][i],
                                REL_SUM * (fac[i].abs() * dw['dw_abs'][i] + inits[i][:D].double().abs()) + fac[i].abs() * dw['dw_err'][i])
                               for i in range(depth)))
        ck.true(f'{name}: guards untouched', all(same_bits(b[D:], b0[D:]) for b, b0 in zip(bufs, inits)))
    ck.true('G guard rows untouched', all(untouched(b[M]) for b in out['G']))
    ck.true('scalar table guard rows untouched', untouched(out['sc'][:, M]))
    ck.true('scalar slots k >= L1 - 1 unwritten', all(all_nan(out['sc'][i][:M, i + 1:]) for i in range(depth)))
    ck.true('workspace guard untouched', untouched(out['ws'][-1:]))
    ck.done()


def test_reference_backward_matches_autograd():
    """the closed form the backward test holds the kernels to, against float64 autograd of the stacked AttentionResidual, on inputs with
    zero rows and rows below the clamp (where autograd treats the clamped norm as a constant)"""
    depth, M = 3, 613
    ck = Checks('float64 closed form vs autograd')
    for D in (128, 384):
        hb, gam, pq, ws, R = stack_inputs(depth, M, D, 5 + D)
        hid = [h.double().requires_grad_(True) for h in hb]
        ga = [t.double().requires_grad_(True) for t in gam]
        pa = [t.double().requires_grad_(True) for t in pq]
        loss = sum((ares_ref(hid[:i + 2], ga[i], pa[i]) * R[i].double()).sum() for i in range(depth))
        loss.backward()
        sc, dw = stack_reference(hb, ws, R)
        for k in range(depth + 1):
            G, T, _ = assemble(k, hb, ws, R, sc)
            ck(f'D={D} G', G, hid[k].grad, 1e-9 * T + 1e-300)
        for i in range(depth):
            T = torch.einsum('lm,lmd->d', sc['c1'][i, :i + 2].abs(), torch.stack(hb[:i + 2]).double().abs())
            ck(f'D={D} d gamma', pq[i].double() * dw['dw'][i], ga[i].grad, 1e-9 * pq[i].double().abs() * T + 1e-300)
            ck(f'D={D} d pq', (gam[i].double() + 1) * dw['dw'][i], pa[i].grad, 1e-9 * (gam[i].double() + 1).abs() * T + 1e-300)
        clamped = torch.stack([h.double().norm(dim = -1) for h in hb]) < EPS
        ck.true(f'D={D}: rows below the clamp present in every hidden', bool(clamped.sum(1).ge(4).all()))
    ck.done()
