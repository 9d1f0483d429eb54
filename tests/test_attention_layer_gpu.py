"""GPU: the attention layer against a float64 reference, called the way engine.forward / engine.backward call it.

* the bounded-logit fast path (attention_sm90.cu) and the general kernels (attention.cu) over the whole accepted gamma range, H = 8 and 2,
  ragged layouts with every awkward length and span shape, dv written into the packed dqkvg matrix;
* exact invariants: keys a query cannot see, and queries that cannot see a key tile, leave the results bit for bit unchanged;
* cached prefill (keys and values in a slab cache, kv_limit in cache-row coordinates);
* the LASER / learned-value-residual row kernels (attn_variants.cu) one by one, and the whole layer chain in engine order.
The helpers and the invariant, cache, row-kernel and chain bodies take the head width (dh, default 64); tests/test_dh128_kernels_gpu.py
runs them at 128.

Errors are per (token, head) row: |ours - ref|_inf / max(|ref row|_inf, 1e-3 max|ref|, |mag row|_inf) where `mag` (for outputs that are
sums) holds the magnitudes of the summed terms, e.g. |dS| |K| for dq: the scale of a floating-point sum's rounding error, which does not
shrink where the terms cancel (the first query of a sequence has dq = 0 exactly, as dP = D there; D itself is a sum that cancels).
lse is an absolute error."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from transfusion_pytorch_b200 import _lib
from helpers import guarded, untouched
from test_ops_gpu import make_rb

pytestmark = pytest.mark.gpu
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
SCALE, CAP = 0.125, 50.
SENT = -77.5                                          # fills the dqkvg columns a kernel must not write (exact in bf16)

# Bounds: at most ~3x the largest error measured over the whole parametrisation on an H100 80GB HBM3 (measured value in the comment).
TOL = dict(
    o = 2e-2,              # measured 6.6e-3
    lse = 5e-5,            # measured 1.8e-5 (absolute)
    dq = 4e-3,             # measured 1.5e-3
    dk = 4e-3,             # measured 1.3e-3
    dv = 2.5e-2,           # measured 9.4e-3 (bf16 output)
    dgate = 7e-3,          # measured 2.5e-3
    pair_o = 2e-2,         # fast path vs general kernel; measured 7.7e-3
    pair_lse = 6e-5,       # measured 2.1e-5 (absolute)
    pair_dq = 4e-3,        # measured 1.6e-3
    pair_dk = 6e-3,        # measured 2.1e-3
    pair_dv = 2.5e-2,      # measured 8.7e-3
    cache_o = 1.8e-2,      # measured 6.4e-3
    cache_lse = 4.5e-5,    # measured 1.5e-5 (absolute)
    var_bf16 = 1e-2,       # a bf16-rounded output of a row kernel; measured 3.9e-3
    var_sum = 3.5e-3,      # a row kernel's per-head sums (D, gate sums, d mix) and the fp32 dv0; measured 1.2e-3
    chain_dq = 4.5e-3,     # measured 1.5e-3
    chain_dk = 8e-2,       # measured 2.9e-2 (LASER: P V' with V' up to e^15 in bf16, dO = dAtt sg / o)
    chain_dv = 5.5e-2,     # measured 1.9e-2
    chain_dv0 = 6e-2,      # measured 2.0e-2
    chain_dmix = 7e-2,     # measured 2.2e-2 (H = 32; 1.2e-2 at H = 8)
    chain_dgate = 1.1e-2,  # measured 3.8e-3
)
# dim_head = 128 (the general kernels and the _d128 row kernels, tests/test_dh128_kernels_gpu.py): ~3x the worst error measured there, same card
TOL_D128 = dict(
    o = 1.4e-2,            # measured 4.6e-3
    lse = 4.5e-5,          # measured 1.4e-5 (absolute)
    dq = 2.5e-3,           # measured 8.0e-4
    dk = 3.5e-3,           # measured 1.2e-3
    dv = 3e-2,             # measured 1.0e-2 (bf16 output)
    dgate = 4.5e-3,        # measured 1.5e-3
    cache_o = 1.4e-2,      # measured 3.9e-3
    cache_lse = 4.5e-5,    # measured 1.2e-5 (absolute)
    var_bf16 = 1.2e-2,     # measured 3.9e-3
    var_sum = 2.6e-3,      # measured 8.7e-4
    chain_dq = 2.8e-3,     # measured 9.1e-4
    chain_dk = 4e-2,       # measured 1.4e-2
    chain_dv = 6.5e-2,     # measured 2.2e-2
    chain_dv0 = 7e-2,      # measured 2.3e-2
    chain_dmix = 5.5e-2,   # measured 1.9e-2
    chain_dgate = 5e-3,    # measured 1.7e-3
)
TOLS = {64: TOL, 128: TOL_D128}
INSIDE = {64: 1.1, 128: 0.76}      # gamma whose largest logit sqrt(dh) (gamma + 1)^2 is ~0.7 CAP (inside the bounded path's range at 64)


WORST = {}                         # (dh, name) -> worst error seen in this session (printed by tests/test_dh128_kernels_gpu.py)


def check(name, err_where, dh = 64):
    err, where = err_where
    bound = TOLS[dh][name]
    WORST[dh, name] = max(WORST.get((dh, name), 0.), err)
    assert err <= bound, f'{name}: worst error {err:.3e} at (token, head) {where}, bound {bound:.1e}'


def row_err(ours, ref, H, width = 64, mag = None):
    a, r = ours.double().reshape(-1, H, width), ref.double().reshape(-1, H, width)
    den = r.abs().amax(-1).clamp(min = 1e-3 * r.abs().max().item())
    if mag is not None:
        den = torch.maximum(den, mag.double().reshape(-1, H, width).abs().amax(-1))
    e = (a - r).abs().amax(-1) / den
    i = int(e.argmax())
    return e.max().item(), (i // H, i % H)


def lse_err(ours, ref):                                # [H, M], absolute
    e = (ours.double() - ref.double()).abs()
    i = int(e.argmax())
    return e.max().item(), (i % e.shape[1], i // e.shape[1])


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


TABLES = ('kv_limit', 'tile_q0', 'tile_qend', 'tile_kv0', 'tile_kvend', 'kt_kv0', 'kt_kvend', 'kt_q0', 'kt_qend',
          't2_q0', 't2_qend', 't2_kv0', 't2_kvend', 'k2_kv0', 'k2_kvend', 'k2_q0', 'k2_qend', 'k2_order')


def tables(rb):
    return {n: dev(getattr(rb, n)) for n in TABLES}


def seqs_of(rb):
    return [(int(rb.cu[b]), int(rb.cu[b + 1]), int(rb.cu[b]), int(rb.cu[b + 1])) for b in range(rb.B)]


# ================================================================================================ float64 reference
def ref_attention(q, k, v, gates, kv_limit, seqs, H, dh = 64):
    """span-masked, soft-capped attention in float64 with dh-wide heads (scale dh^-1/2).  seqs: (q_start, q_end, k_start, k_end) row ranges;
    query i sees key j iff k_start <= j <= kv_limit[i].  Returns o [Mq, H dh] (times sigmoid(gate) when gates are given) and the natural-log
    lse [H, Mq]."""
    outs, lses = [], []
    for qs, qe, ks, ke in seqs:
        qq, kk, vv = (t.reshape(-1, H, dh).transpose(0, 1) for t in (q[qs:qe], k[ks:ke], v[ks:ke]))
        s = torch.tanh(torch.einsum('hid,hjd->hij', qq, kk) * (dh ** -0.5 / CAP)) * CAP
        vis = torch.arange(ks, ke, device = q.device)[None, :] <= kv_limit[qs:qe, None]
        s = s.masked_fill(~vis[None], float('-inf'))
        lse = torch.logsumexp(s, -1)
        o = torch.einsum('hij,hjd->hid', torch.exp(s - lse[..., None]), vv)
        if gates is not None:
            o = o * torch.sigmoid(gates[qs:qe].t())[..., None]
        outs.append(o.transpose(0, 1).reshape(qe - qs, H * dh)); lses.append(lse)
    return torch.cat(outs), torch.cat(lses, 1)


HEAD_GROUP = 8     # heads the float64 reference evaluates at once: its [heads, n, n] score tensors stay at an 8-head model's size at any H


def head_groups(H):
    return [(h0, min(h0 + HEAD_GROUP, H)) for h0 in range(0, H, HEAD_GROUP)]


def head_cols(t, h0, h1, width):
    """columns of heads [h0, h1) of a [rows, H width] matrix (None stays None)"""
    return None if t is None else t[:, h0 * width:h1 * width]


@torch.no_grad()
def ref_magnitudes(q, k, v, gates, dog, kv_limit, seqs, H, dh = 64):
    """magnitudes of the terms each output row sums: |P| |V| for o, |dS| |K| for dq, |dS|^T |Q| for dk, |P|^T |dO| for dv, |dO| |o| for the gate
    sums (dO: the gradient at the un-gated attention output).  |dS| = P (|dO| |V|^T + |dO| . |P| |V|) (1 - tanh^2) scale bounds the terms of
    dS = P (dO V^T - dO . o) (1 - tanh^2) scale before dP - D and the sum D = dO . o cancel.  Heads are independent: evaluated in groups of
    at most HEAD_GROUP heads."""
    groups = [_ref_magnitudes(*(head_cols(t, h0, h1, dh) for t in (q, k, v)), head_cols(gates, h0, h1, 1), head_cols(dog, h0, h1, dh),
                              kv_limit, seqs, h1 - h0, dh) for h0, h1 in head_groups(H)]
    return {name: torch.cat([m[name] for m in groups], 1) for name in groups[0]}


def _ref_magnitudes(q, k, v, gates, dog, kv_limit, seqs, H, dh):
    HI, scale = H * dh, dh ** -0.5
    mag = dict(o = torch.zeros(q.shape[0], HI, device = q.device, dtype = F64), dq = torch.zeros(q.shape[0], HI, device = q.device, dtype = F64),
               dk = torch.zeros(k.shape[0], HI, device = q.device, dtype = F64), dv = torch.zeros(k.shape[0], HI, device = q.device, dtype = F64),
               dgate = torch.zeros(q.shape[0], H, device = q.device, dtype = F64))
    for qs, qe, ks, ke in seqs:
        qq, kk, vv = (t.double().reshape(-1, H, dh).transpose(0, 1) for t in (q[qs:qe], k[ks:ke], v[ks:ke]))
        tt = torch.tanh(torch.einsum('hid,hjd->hij', qq, kk) * (scale / CAP))
        vis = torch.arange(ks, ke, device = q.device)[None, :] <= kv_limit[qs:qe, None].long()
        s = (tt * CAP).masked_fill(~vis[None], float('-inf'))
        p = torch.exp(s - torch.logsumexp(s, -1, keepdim = True))
        mag['o'][qs:qe] = (p @ vv.abs()).transpose(0, 1).reshape(-1, HI)
        if dog is None:
            continue
        do = dog[qs:qe].double().reshape(-1, H, dh).transpose(0, 1)
        o = p @ vv
        if gates is not None:
            sg = torch.sigmoid(gates[qs:qe].double().t())[..., None]
            mag['dgate'][qs:qe] = ((do.abs() * (o * sg).abs()).sum(-1) * (1 - sg[..., 0])).t()
            do = do * sg
        ds = p * (do.abs() @ vv.abs().transpose(1, 2) + (do.abs() * (p @ vv.abs())).sum(-1, keepdim = True)) * (1 - tt * tt) * scale
        mag['dq'][qs:qe] = (ds.abs() @ kk.abs()).transpose(0, 1).reshape(-1, HI)
        mag['dk'][ks:ke] = (ds.abs().transpose(1, 2) @ qq.abs()).transpose(0, 1).reshape(-1, HI)
        mag['dv'][ks:ke] = (p.transpose(1, 2) @ do.abs()).transpose(0, 1).reshape(-1, HI)
    return mag


def reference(q, k, v, gates, dog, kv_limit, seqs, H, dh = 64):
    """forward and autograd gradients of ref_attention from the bf16 / fp32 inputs the kernels get, and the magnitudes of the summed terms.
    One float64 graph per group of at most HEAD_GROUP heads (heads are independent), freed before the next"""
    parts = []
    for h0, h1 in head_groups(H):
        qf, kf, vf = (head_cols(t, h0, h1, dh).double().requires_grad_(True) for t in (q, k, v))
        gf = head_cols(gates, h0, h1, 1).double().requires_grad_(True) if gates is not None else None
        o, lse = ref_attention(qf, kf, vf, gf, kv_limit.long(), seqs, h1 - h0, dh)
        o.backward(head_cols(dog, h0, h1, dh).double())
        parts.append(dict(o = o.detach(), lse = lse.detach(), dq = qf.grad, dk = kf.grad, dv = vf.grad, dgate = gf.grad if gf is not None else None))
    cat = lambda name, dim: torch.cat([p[name] for p in parts], dim)
    return dict(o = cat('o', 1), lse = cat('lse', 0), dq = cat('dq', 1), dk = cat('dk', 1), dv = cat('dv', 1),
                dgate = cat('dgate', 1) if gates is not None else None, mag = ref_magnitudes(q, k, v, gates, dog, kv_limit, seqs, H, dh))


# ================================================================================================ inputs
def fast_params(ops, gamma):
    fp = torch.zeros(8, device = 'cuda')
    gam = torch.full((64,), gamma, device = 'cuda')
    ops.attn_fast_params(gam, gam, 64, SCALE, CAP, fp)
    return fp


def unit_rows(x, gamma):
    """q / k as the QKVG epilogue writes them from x [M, H, dh]: per-head RMSNorm, times sqrt(dh) (gamma + 1).  gamma None: 4 x, not normalised
    (the RoPE-only epilogue of qk_rmsnorm = False leaves the logits unbounded: q = k rows reach |s| ~ 16 dh scale, > 3 CAP at dh = 128)"""
    M, H, dh = x.shape
    if gamma is None:
        return (4. * x).reshape(M, H * dh).to(BF16)
    return (Fn.normalize(x, dim = -1) * dh ** 0.5 * (1. + gamma)).reshape(M, H * dh).to(BF16)


def qk_inputs(cu, H, gamma, g, dh = 64):
    """rows 3i: q = k (the diagonal logit at the +bound), rows 3i + 1: q = -k (-bound); the causal queries of the first half of the first
    sequence see only logits near the -bound, where the fixed softmax maximum of the fast path is farthest from the row's own maximum.
    A causal query's diagonal key is the last it sees, so the rows 3i past a sequence's first 64 find their largest logit in a later key
    tile than their first: the running maximum of the general forward rises by about the whole logit range there."""
    M = int(cu[-1])
    rnd = lambda *s: torch.randn(*s, device = 'cuda', generator = g, dtype = F64)
    qd, kd = rnd(M, H, dh), rnd(M, H, dh)
    r = torch.arange(M, device = 'cuda')
    qd[r % 3 == 0] = kd[r % 3 == 0]
    qd[r % 3 == 1] = -kd[r % 3 == 1]
    s = int(cu[0]); e = s + (int(cu[1]) - s + 1) // 2         # (the first half of it)
    u = rnd(1, H, dh)
    kd[s:e] = u + 0.1 * rnd(e - s, H, dh)
    qd[s:e] = -(u + 0.1 * rnd(e - s, H, dh))
    return unit_rows(qd, gamma), unit_rows(kd, gamma)


def assert_sentinel(buf, written):
    """every column of the bf16 [M, NQ] buffer outside the `written` column ranges still holds SENT, bit for bit"""
    keep = torch.ones(buf.shape[1], dtype = torch.bool, device = 'cuda')
    for c0, c1 in written:
        keep[c0:c1] = False
    sent = torch.tensor(SENT, dtype = BF16).view(torch.int16).item()
    assert (buf[:, keep].view(torch.int16) == sent).all(), 'a kernel wrote outside its columns of the packed matrix'


def attn_forward(ops, T, q, k, v, gates, H, fp, o, lse, general_only = False, dh = 64):
    """the attention forward as engine.forward enqueues it.  dh = 64: both kernels are enqueued and the one whose precondition (read from fp
    on the device) fails returns at once (general_only: the general kernel alone, no fast-path flag); dh = 128: the general kernel alone"""
    M, HI = q.shape[0], H * dh
    if dh == 128:
        ops.attn_fwd_d128(q, k, v, HI, HI, HI, gates, H, T['kv_limit'], T['tile_q0'], T['tile_qend'], T['tile_kv0'], T['tile_kvend'], len(T['tile_q0']),
                          o, HI, lse, M, dh ** -0.5, CAP)
        return
    if not general_only:
        ops.attn_fwd_tc(q, k, v, HI, HI, HI, gates, H, T['kv_limit'], T['t2_q0'], T['t2_qend'], T['t2_kv0'], T['t2_kvend'], len(T['t2_q0']),
                        o, HI, lse, M, 0, SCALE, CAP, fp)
    ops.attn_fwd(q, k, v, HI, HI, HI, gates, H, T['kv_limit'], T['tile_q0'], T['tile_qend'], T['tile_kv0'], T['tile_kvend'], len(T['tile_q0']),
                 o, HI, lse, M, SCALE, CAP, None if general_only else fp)


def attn_backward(ops, T, q, k, v, dop, lse, dsum, dq, dk, dqkvg, H, fp, general_only = False, dh = 64):
    """the attention backward after its prep kernel, as engine.backward enqueues it (see attn_forward); dv goes into the v columns of dqkvg"""
    M, HI = q.shape[0], H * dh
    NQ = dqkvg.shape[1]
    if dh == 128:
        ops.attn_bwd_d128(q, k, v, dop, HI, HI, HI, HI, lse, dsum, T['kv_limit'], T['kt_kv0'], T['kt_kvend'], T['kt_q0'], T['kt_qend'], len(T['kt_kv0']),
                          dq, dk, dqkvg[:, 2 * HI:], NQ, M, H, dh ** -0.5, CAP)
        return
    if not general_only:
        ops.attn_bwd_tc(q, k, v, dop, HI, HI, HI, HI, lse, dsum, T['kv_limit'], T['k2_kv0'], T['k2_kvend'], T['k2_q0'], T['k2_qend'], T['k2_order'],
                        len(T['k2_kv0']), dq, dk, dqkvg[:, 2 * HI:], NQ, M, H, SCALE, CAP, fp)
    ops.attn_bwd(q, k, v, dop, HI, HI, HI, HI, lse, dsum, T['kv_limit'], T['kt_kv0'], T['kt_kvend'], T['kt_q0'], T['kt_qend'], len(T['kt_kv0']),
                 dq, dk, dqkvg[:, 2 * HI:], NQ, M, H, SCALE, CAP, None if general_only else fp)


def attention_pass(ops, T, q, k, v, gates, dog, H, fp, general_only = False, dh = 64, pad = 128, dsum_mh_none = False):
    """one layer's attention forward + backward as the engine launches it (attn_forward, the prep kernel, attn_backward); dv goes into the
    v columns of a dqkvg-shaped matrix (ld = 3 HI + pad: pad = 128 with the gate / mix tile, 0 for an ungated model without the value
    residual) whose other columns and a guard row below it hold SENT; dq and dk start non-zero.  dsum_mh_none: the prep kernel gets no
    gate-sum buffer, as an ungated model launches it (dsum_mh is then None)."""
    M, HI = q.shape[0], H * dh
    NQ = 3 * HI + pad
    o = torch.zeros(M, HI, device = 'cuda', dtype = BF16); lse = torch.zeros(H, M, device = 'cuda')
    attn_forward(ops, T, q, k, v, gates, H, fp, o, lse, general_only, dh)
    dop = torch.zeros_like(dog); dsum = torch.zeros(H, M, device = 'cuda')
    dsum_mh = None if dsum_mh_none else torch.zeros(M, H, device = 'cuda')
    dq = torch.full((M, HI), 7., device = 'cuda')                   # cleared by the prep kernel
    if dh == 128:
        ops.attn_bwd_prep_d128(dog, o, gates, dop, dsum, dsum_mh, dq, M, H)
    else:
        ops.attn_bwd_prep(dog, o, gates, dop, dsum, dsum_mh, dq, M, H)
    dk = torch.full((M, HI), 3., device = 'cuda')                   # every row is overwritten
    dqkvg_buf, dqkvg = guarded(M, NQ, BF16)
    attn_backward(ops, T, q, k, v, dop, lse, dsum, dq, dk, dqkvg, H, fp, general_only, dh)
    torch.cuda.synchronize()
    assert_sentinel(dqkvg, [(2 * HI, 3 * HI)])
    assert untouched(dqkvg_buf[M:]), 'a kernel wrote below the last row of the packed matrix'
    return dict(o = o, lse = lse, dq = dq, dk = dk, dv = dqkvg[:, 2 * HI:3 * HI], dsum_mh = dsum_mh)


# ================================================================================================ layouts
SPAN_KINDS = ('one', 'start', 'whole', 'adjacent', 'end64', 'end128', 'skip16')


def span_pattern(kind, n, rng):
    """(offset, length) spans of one kind inside a sequence of n tokens; None when the sequence is too short for it"""
    ri = lambda a, b: int(rng.integers(a, b))               # [a, b)
    if kind == 'one':
        return [(ri(0, n), 1)]
    if kind == 'start':
        return [(0, ri(1, n + 1))]
    if kind == 'whole':
        return [(0, n)]
    if kind == 'adjacent' and n >= 3:
        a = ri(0, n - 2); l1 = ri(1, n - a - 1)
        return [(a, l1), (a + l1, ri(1, n - a - l1 + 1))]
    if kind in ('end64', 'end128') and n >= int(kind[3:]):  # the span's last token is the last row of a 64- / 128-row tile
        w = int(kind[3:])
        end = w * ri(1, n // w + 1)
        off = ri(0, end)
        return [(off, end - off)]
    if kind == 'skip16' and n >= 145:
        # last token one row before the last key of a 16-key warp slice of a backward key tile, first token 64-aligned: the queries of a
        # whole 64-row step see every key of that slice but its last
        end = 143 + 16 * ri(0, (n - 144) // 16 + 1)
        off = 64 * ri(0, 2)
        return [(off, end - off)]
    return None


def random_layout(seed):
    """ragged batch with three of the lengths 1, 63, 64, 65, 127, 128, 129 among random ones, M = seed (mod 4); each sequence gets one
    span pattern, cycled with the seed so that every pattern appears in the set"""
    rng = np.random.default_rng(1000 + seed)
    lens = [int(x) for x in rng.choice([1, 63, 64, 65, 127, 128, 129], size = 3, replace = False)] + [int(x) for x in rng.integers(150, 700, size = 3)]
    rng.shuffle(lens)
    lens.append(int(rng.integers(2, 300)))
    lens[-1] += (seed - sum(lens)) % 4
    spans = []
    for b, n in enumerate(lens):
        pat = span_pattern(SPAN_KINDS[(seed + b) % len(SPAN_KINDS)], n, rng) or span_pattern('one', n, rng)
        spans += [(b, off, ln) for off, ln in pat]
    return lens, spans


LAYOUTS = {
    'two1024': ([1024, 1024], [(0, 206, 256), (0, 668, 256), (1, 100, 700)]),
    'mixed4': ([77, 130, 5, 300], [(0, 10, 40), (1, 64, 64), (1, 128, 2), (3, 120, 150)]),
    'one64': ([64], []),
    'tiles128': ([128, 129, 127], [(1, 0, 129)]),
    'nine': ([640] * 6 + [385, 1000, 257], [(b, 100, 300) for b in range(6)] + [(7, 100, 800)]),
    'seven': ([385, 1000, 257, 640, 129, 900, 31], [(1, 100, 800), (3, 0, 640), (5, 300, 77), (5, 500, 300)]),
    **{f'random{s}': random_layout(s) for s in range(8)},
}
RINGS = {
    'ring4096': ([4096], [(0, 1000, 300), (0, 2500, 700)]),               # 64 query steps for the first key tile
    'ring4000': ([4000, 1000], [(0, 100, 2000), (1, 300, 500)]),          # 63 / 16 steps: odd counts
}
GAMMAS = {'gamma0': 0.0, 'inside': 1.1, 'outside': 1.2}                  # y_max = 0.16, 0.71 (fast path), 0.78 (general kernel)


def fast_vs_fp64(ops, lens, spans, H, gamma, seed, gated = None, pad = 128):
    """gated: None gates iff H == 8.  gamma None: unnormed logits (|s / cap| > 3, as a qk_rmsnorm = False model gives them), on the general
    kernels alone with no fast-path parameters, as such a model launches them.  pad: the dqkvg pitch is 3 HI + pad (attention_pass)"""
    rb = make_rb(lens, spans)
    M, T = rb.M, tables(rb)
    g = torch.Generator(device = 'cuda').manual_seed(seed)
    general_only = gamma is None
    fp = None if general_only else fast_params(ops, gamma)
    torch.cuda.synchronize()
    if not general_only:
        assert fp[0].item() == (1. if gamma <= 1.1 else 0.)
    q, k = qk_inputs(rb.cu, H, gamma, g)
    y = (q.double() * k.double()).reshape(M, H, 64).sum(-1) * SCALE / CAP
    if gamma == 1.1:                                    # the soft-cap argument reaches ~0.7 at both signs
        assert y.max().item() > 0.69 and y.min().item() < -0.69
    elif general_only:
        assert y.max().item() > 3 and y.min().item() < -3
    v = (torch.randn(M, H * 64, device = 'cuda', generator = g) * 2).to(BF16)
    gates = torch.randn(M, H, device = 'cuda', generator = g) if (H == 8 if gated is None else gated) else None
    dog = torch.randn(M, H * 64, device = 'cuda', generator = g).to(BF16)
    runs = [] if general_only else [attention_pass(ops, T, q, k, v, gates, dog, H, fp, pad = pad)]
    runs.append(attention_pass(ops, T, q, k, v, gates, dog, H, fp, general_only = True, pad = pad))
    eng, gen = runs[0], runs[-1]
    if not general_only and fp[0].item() == 0.:         # outside the bound the general kernel did the work
        assert torch.equal(eng['o'], gen['o']) and torch.equal(eng['lse'], gen['lse'])
    ref = reference(q, k, v, gates, dog, T['kv_limit'], seqs_of(rb), H)
    mag = ref['mag']
    for out in runs:
        check('o', row_err(out['o'], ref['o'], H, mag = mag['o']))
        check('lse', lse_err(out['lse'], ref['lse']))
        for name in ('dq', 'dk', 'dv'):
            check(name, row_err(out[name], ref[name], H, mag = mag[name]))
        if gates is not None:
            check('dgate', row_err((1 - torch.sigmoid(gates)) * out['dsum_mh'], ref['dgate'], H, 1, mag = mag['dgate']))
    if general_only:
        return
    check('pair_o', row_err(eng['o'], gen['o'], H, mag = mag['o']))
    check('pair_lse', lse_err(eng['lse'], gen['lse']))
    for name in ('dq', 'dk', 'dv'):
        check('pair_' + name, row_err(eng[name], gen[name], H, mag = mag[name]))


@pytest.mark.parametrize('gamma', list(GAMMAS), ids = list(GAMMAS))
@pytest.mark.parametrize('H', [8, 2])
@pytest.mark.parametrize('layout', list(LAYOUTS))
def test_attention_vs_fp64(ops, layout, H, gamma):
    """bounded-logit fast path (engine launch pattern) and general kernels against float64 autograd, and against each other"""
    fast_vs_fp64(ops, *LAYOUTS[layout], H, GAMMAS[gamma], seed = 20 + H)


@pytest.mark.parametrize('gamma', list(GAMMAS), ids = list(GAMMAS))
@pytest.mark.parametrize('layout', list(RINGS))
def test_attention_vs_fp64_long_sequences(ops, layout, gamma):
    fast_vs_fp64(ops, *RINGS[layout], 8, GAMMAS[gamma], seed = 30)


# ================================================================================================ exact invariants
INV_LAYOUT = ([385, 1000, 257, 640, 129], [(1, 100, 800), (3, 0, 640), (4, 5, 1)])


def _inv_setup(ops, H, dh = 64):
    rb = make_rb(*INV_LAYOUT)
    g = torch.Generator(device = 'cuda').manual_seed(40)
    fp = fast_params(ops, 1.1) if dh == 64 else None
    q, k = qk_inputs(rb.cu, H, INSIDE[dh], g, dh)
    v = (torch.randn(rb.M, H * dh, device = 'cuda', generator = g) * 2).to(BF16)
    gates = torch.randn(rb.M, H, device = 'cuda', generator = g)
    dog = torch.randn(rb.M, H * dh, device = 'cuda', generator = g).to(BF16)
    return rb, tables(rb), g, fp, q, k, v, gates, dog


def _same_key_tiles(rb, a, b, names, seen, dh = 64):
    """dk / dv rows of every backward key tile (128 keys of the k2 tables at dh = 64, where the fast path's tiles are the coarser; the 64 keys
    of the kt tables at dh = 128) that no query in `seen` (bool [M]) can see are bit-identical between runs a and b"""
    kvl, cu = rb.kv_limit, rb.cu
    n = 0
    kv0s, kves = (rb.k2_kv0, rb.k2_kvend) if dh == 64 else (rb.kt_kv0, rb.kt_kvend)
    for kv0, kve in zip(kv0s.tolist(), kves.tolist()):
        bq = int(np.searchsorted(cu, kv0, side = 'right') - 1)
        s, e = int(cu[bq]), int(cu[bq + 1])
        if (seen[s:e] & (kvl[s:e] >= kv0)).any():
            continue
        n += 1
        for name in names:
            assert torch.equal(a[name][kv0:kve], b[name][kv0:kve]), (name, kv0)
    return n


@pytest.mark.parametrize('H', [8, 2])
def test_invisible_keys_do_not_matter(ops, H, dh = 64):
    """new K rows (inside the RMS-norm bound) and V rows of +-1e3 where a set of queries cannot see them: those queries' o / lse and the
    dk / dv of key tiles no changed query sees stay bit-identical; their dq moves by reduction-order noise only"""
    rb, T, g, fp, q, k, v, gates, dog = _inv_setup(ops, H, dh)
    M, cu = rb.M, rb.cu
    base = attention_pass(ops, T, q, k, v, gates, dog, H, fp, dh = dh)
    changed = np.zeros(M, dtype = bool)
    changed[cu[2]:cu[3]] = True                          # a whole sequence: the steps of the previous sequence's last key tile run into it
    changed[cu[4] + 100:cu[5]] = True                    # the tail of a causal sequence: its first 100 queries cannot see it
    rows = torch.from_numpy(np.nonzero(changed)[0]).cuda()
    k2, v2 = k.clone(), v.clone()
    k2[rows] = unit_rows(torch.randn(len(rows), H, dh, device = 'cuda', generator = g, dtype = F64), INSIDE[dh])
    v2[rows] = (torch.randint(0, 2, (len(rows), H * dh), device = 'cuda', generator = g) * 2000. - 1000.).to(BF16)
    new = attention_pass(ops, T, q, k2, v2, gates, dog, H, fp, dh = dh)
    kvl = rb.kv_limit
    seq = np.repeat(np.arange(rb.B), rb.seq_lens)
    first_changed = np.array([np.argmax(changed[cu[b]:cu[b + 1]]) + cu[b] if changed[cu[b]:cu[b + 1]].any() else 1 << 30 for b in range(rb.B)])
    blind = kvl < first_changed[seq]                     # queries that see none of the changed keys
    assert blind.sum() > 0.6 * M and (~blind).sum() > 250
    bq = torch.from_numpy(np.nonzero(blind)[0]).cuda()
    assert torch.equal(new['o'][bq], base['o'][bq]) and torch.equal(new['lse'][:, bq], base['lse'][:, bq])
    d = (new['dq'][bq] - base['dq'][bq]).abs().reshape(-1, H, dh).amax(-1)
    assert (d <= 1e-5 * base['dq'][bq].abs().reshape(-1, H, dh).amax(-1)).all()
    assert _same_key_tiles(rb, base, new, ('dk', 'dv'), ~blind, dh) >= 8


@pytest.mark.parametrize('H', [8, 2])
def test_invisible_queries_do_not_matter(ops, H, dh = 64):
    """new Q / dO rows for queries that cannot see a key tile: that tile's dk / dv stay bit-identical (masked steps, masked rows of a step,
    and steps that run past the end of the sequence into the changed rows)"""
    rb, T, g, fp, q, k, v, gates, dog = _inv_setup(ops, H, dh)
    M, cu = rb.M, rb.cu
    base = attention_pass(ops, T, q, k, v, gates, dog, H, fp, dh = dh)
    changed = np.zeros(M, dtype = bool)
    changed[cu[1]:cu[1] + 100] = True                    # causal queries before the span: they cannot see the key tiles from row 128 on
    changed[cu[2]:cu[3]] = True
    rows = torch.from_numpy(np.nonzero(changed)[0]).cuda()
    q2, dog2 = q.clone(), dog.clone()
    q2[rows] = unit_rows(torch.randn(len(rows), H, dh, device = 'cuda', generator = g, dtype = F64), INSIDE[dh])
    dog2[rows] = torch.randn(len(rows), H * dh, device = 'cuda', generator = g).to(BF16)
    new = attention_pass(ops, T, q2, k, v, gates, dog2, H, fp, dh = dh)
    assert _same_key_tiles(rb, base, new, ('dk', 'dv'), changed, dh) >= 12


# ================================================================================================ cached prefill
@pytest.mark.parametrize('H', [8, 2])
def test_cached_prefill_vs_fp64(ops, H, dh = 64):
    """q rows in their own matrix, keys / values in a zero-initialised slab cache (M_kv = n_slabs cap); slabs hold a prefix of earlier rows
    (always visible) and are filled to lengths that are not multiples of 64.  Finite rows past a slab's filled length change nothing."""
    n_slabs, cap = 4, 700
    lens, base = [300, 129, 1, 250], [0, 57, 200, 3]
    slab = [2, 0, 3, 1]
    spans = [(0, 0, 40), (1, 60, 69), (3, 100, 150)]
    rb = make_rb(lens, spans)
    M, HI, cu = rb.M, H * dh, rb.cu
    g = torch.Generator(device = 'cuda').manual_seed(50)
    seq = np.repeat(np.arange(rb.B), rb.seq_lens)
    off = np.asarray(slab) * cap + np.asarray(base) - cu[:-1]        # as pack_incremental builds it
    kv_row = np.arange(M) + off[seq]
    kvl = rb.kv_limit + off[seq]
    tabs = {}
    for pre in ('tile', 't2'):
        q0 = getattr(rb, f'{pre}_q0')
        ts = np.searchsorted(cu, q0, side = 'right') - 1
        tabs.update({f'{pre}_q0': dev(q0), f'{pre}_qend': dev(getattr(rb, f'{pre}_qend')),
                     f'{pre}_kv0': dev((np.asarray(slab)[ts] * cap).astype(np.int32)), f'{pre}_kvend': dev((getattr(rb, f'{pre}_kvend') + off[ts]).astype(np.int32))})
    kvl_d = dev(kvl.astype(np.int32))
    fp = fast_params(ops, 1.1) if dh == 64 else None
    q, knew = qk_inputs(cu, H, INSIDE[dh], g, dh)
    rows_all = n_slabs * cap
    kc = torch.zeros(rows_all, HI, device = 'cuda', dtype = BF16); vc = torch.zeros_like(kc)
    filled = np.zeros(rows_all, dtype = bool)
    for b in range(rb.B):
        s0 = slab[b] * cap
        kc[s0:s0 + base[b]] = unit_rows(torch.randn(base[b], H, dh, device = 'cuda', generator = g, dtype = F64), INSIDE[dh])
        vc[s0:s0 + base[b]] = (torch.randn(base[b], HI, device = 'cuda', generator = g) * 2).to(BF16)
        filled[s0:s0 + base[b] + lens[b]] = True
    kr = torch.from_numpy(kv_row).cuda()
    kc[kr] = knew
    vc[kr] = (torch.randn(M, HI, device = 'cuda', generator = g) * 2).to(BF16)
    gates = torch.randn(M, H, device = 'cuda', generator = g)
    seqs = [(int(cu[b]), int(cu[b + 1]), slab[b] * cap, slab[b] * cap + base[b] + lens[b]) for b in range(rb.B)]

    def run(kc, vc):
        res = []
        for fast in ((True, False) if dh == 64 else (False,)):
            o = torch.zeros(M, HI, device = 'cuda', dtype = BF16); lse = torch.zeros(H, M, device = 'cuda')
            if dh == 128:
                ops.attn_fwd_d128(q, kc, vc, HI, HI, HI, gates, H, kvl_d, tabs['tile_q0'], tabs['tile_qend'], tabs['tile_kv0'], tabs['tile_kvend'],
                                  len(tabs['tile_q0']), o, HI, lse, M, dh ** -0.5, CAP)
            elif fast:
                ops.attn_fwd_tc(q, kc, vc, HI, HI, HI, gates, H, kvl_d, tabs['t2_q0'], tabs['t2_qend'], tabs['t2_kv0'], tabs['t2_kvend'], len(tabs['t2_q0']),
                                o, HI, lse, M, rows_all, SCALE, CAP, fp)
            else:
                ops.attn_fwd(q, kc, vc, HI, HI, HI, gates, H, kvl_d, tabs['tile_q0'], tabs['tile_qend'], tabs['tile_kv0'], tabs['tile_kvend'], len(tabs['tile_q0']),
                             o, HI, lse, M, SCALE, CAP, None)
            res.append((o, lse))
        torch.cuda.synchronize()
        return res

    out = run(kc, vc)
    with torch.no_grad():
        ref_o, ref_lse = ref_attention(q.double(), kc.double(), vc.double(), gates.double(), kvl_d.long(), seqs, H, dh)
    mag_o = ref_magnitudes(q, kc, vc, None, None, kvl_d, seqs, H, dh)['o'] * torch.sigmoid(gates.double()).repeat_interleave(dh, 1)
    for o, lse in out:
        check('cache_o', row_err(o, ref_o, H, dh, mag = mag_o), dh)
        check('cache_lse', lse_err(lse, ref_lse), dh)
    rest = torch.from_numpy(np.nonzero(~filled)[0]).cuda()
    kc2, vc2 = kc.clone(), vc.clone()
    kc2[rest] = unit_rows(torch.randn(len(rest), H, dh, device = 'cuda', generator = g, dtype = F64), INSIDE[dh])
    vc2[rest] = (torch.randint(0, 2, (len(rest), HI), device = 'cuda', generator = g) * 2000. - 1000.).to(BF16)
    for (o, lse), (o2, lse2) in zip(out, run(kc2, vc2)):
        assert torch.equal(o, o2) and torch.equal(lse, lse2)


# ================================================================================================ attn_variants.cu, kernel by kernel
VAR_M = 333


def _rand(g, *shape, scale = 1.):
    return torch.randn(*shape, device = 'cuda', generator = g) * scale


def laser_ref(x, c):
    return torch.exp(c * torch.tanh(x / c))


@pytest.mark.parametrize('clamp', [15., 5.])
@pytest.mark.parametrize('H', [2, 6, 8])
def test_laser_v_fwd_vs_fp64(ops, H, clamp, dh = 64):
    """v' = exp(c tanh(v / c)), plain and scattered to cache rows (the other rows stay zero).  Elementwise: a dh-wide head is dh / 64
    64-wide heads to it, as engine.forward passes it"""
    M, HI = VAR_M, H * dh
    g = torch.Generator(device = 'cuda').manual_seed(60 + H)
    v = _rand(g, M, HI, scale = 8.).to(BF16)
    vl = torch.zeros(M, HI, device = 'cuda', dtype = BF16)
    ops.laser_v_fwd(v, HI, None, vl, HI, M, HI // 64, clamp)
    rows = torch.randperm(3 * M, device = 'cuda', generator = g)[:M].to(torch.int32)
    vc = torch.zeros(3 * M, HI, device = 'cuda', dtype = BF16); vc[rows.long()] = v
    vlc = torch.zeros_like(vc)
    ops.laser_v_fwd(vc, HI, rows, vlc, HI, M, HI // 64, clamp)
    torch.cuda.synchronize()
    want = laser_ref(v.double(), clamp)
    check('var_bf16', row_err(vl, want, H, dh), dh)
    assert torch.equal(vlc[rows.long()], vl)
    untouched = torch.ones(3 * M, dtype = torch.bool, device = 'cuda'); untouched[rows.long()] = False
    assert (vlc[untouched] == 0).all()


@pytest.mark.parametrize('gated', [True, False])
@pytest.mark.parametrize('H', [2, 6, 8])
def test_laser_out_fwd_vs_fp64(ops, H, gated, dh = 64):
    M, HI = VAR_M, H * dh
    g = torch.Generator(device = 'cuda').manual_seed(70 + H)
    o = torch.exp(_rand(g, M, HI, scale = 4.)).to(BF16)
    gates = _rand(g, M, H) if gated else None
    att = torch.zeros(M, HI, device = 'cuda', dtype = BF16)
    if dh == 128:
        ops.laser_out_fwd_d128(o, gates, att, M, H)
    else:
        ops.laser_out_fwd(o, gates, att, M, H)
    torch.cuda.synchronize()
    want = torch.log(o.double()).reshape(M, H, dh)
    if gated:
        want = want * torch.sigmoid(gates.double())[..., None]
    check('var_bf16', row_err(att, want, H, dh), dh)


@pytest.mark.parametrize('H', [2, 6, 8])
def test_laser_bwd_prep_vs_fp64(ops, H, dh = 64, gated = True, dsum_mh_none = False):
    """att = log(o) sigmoid(gate): dO = dAtt sg / o, D = sum dAtt sg, which must equal sum dO o (what the attention backward takes it for),
    d gate = (1 - sg) sum dAtt att, and dq is cleared.  Ungated (gates None): att = log(o), and the gate-sum buffer gets sum dAtt log(o);
    dsum_mh_none: no gate-sum buffer, as an ungated model launches it"""
    M, HI = VAR_M, H * dh
    g = torch.Generator(device = 'cuda').manual_seed(80 + H)
    o = torch.exp(_rand(g, M, HI, scale = 4.)).to(BF16)
    gates = _rand(g, M, H)
    datt = _rand(g, M, HI).to(BF16)
    of, gf = o.double().requires_grad_(True), gates.double().requires_grad_(True)
    sg = torch.sigmoid(gf) if gated else torch.ones_like(gf)
    (torch.log(of).reshape(M, H, dh) * sg[..., None]).reshape(M, HI).backward(datt.double())
    dop = torch.zeros_like(datt); dsum = torch.zeros(H, M, device = 'cuda')
    dsum_mh = None if dsum_mh_none else torch.zeros(M, H, device = 'cuda')
    dq = torch.full((M, HI), 7., device = 'cuda')
    if dh == 128:
        ops.laser_bwd_prep_d128(datt, o, gates if gated else None, dop, dsum, dsum_mh, dq, M, H)
    else:
        ops.laser_bwd_prep(datt, o, gates if gated else None, dop, dsum, dsum_mh, dq, M, H)
    torch.cuda.synchronize()
    check('var_bf16', row_err(dop, of.grad, H, dh), dh)
    D_ref = (of.grad * o.double()).reshape(M, H, dh).sum(-1)
    check('var_sum', row_err(dsum.t(), D_ref, H, 1), dh)
    if gated:
        check('var_sum', row_err((1 - torch.sigmoid(gates)) * dsum_mh, gf.grad, H, 1), dh)
    elif not dsum_mh_none:
        terms = (datt.double() * torch.log(o.double())).reshape(M, H, dh)
        check('var_sum', row_err(dsum_mh, terms.sum(-1), H, 1, mag = terms.abs().sum(-1)), dh)
    assert (dq == 0).all()


@pytest.mark.parametrize('H', [2, 6, 8])
def test_laser_v_bwd_vs_fp64(ops, H, dh = 64):
    """dv = dv' d/dv exp(c tanh(v / c)), in place on the v columns of the packed dqkvg matrix (ld = 3 HI + 128)"""
    M, HI = VAR_M, H * dh
    NQ = 3 * HI + 128
    g = torch.Generator(device = 'cuda').manual_seed(90 + H)
    v = _rand(g, M, HI, scale = 8.).to(BF16)
    dvl = _rand(g, M, HI).to(BF16)
    dqkvg = torch.full((M, NQ), SENT, device = 'cuda', dtype = BF16)
    dqkvg[:, 2 * HI:3 * HI] = dvl
    ops.laser_v_bwd(dqkvg[:, 2 * HI:], NQ, v, HI, M, HI // 64, 15.)
    torch.cuda.synchronize()
    vf = v.double().requires_grad_(True)
    laser_ref(vf, 15.).backward(dvl.double())
    check('var_bf16', row_err(dqkvg[:, 2 * HI:3 * HI], vf.grad, H, dh), dh)
    assert_sentinel(dqkvg, [(2 * HI, 3 * HI)])


@pytest.mark.parametrize('H', [2, 6, 8])
def test_vmix_fwd_vs_fp64(ops, H, dh = 64):
    """v = v mix + v0 (1 - mix), mix = sigmoid(mix_pre + bias), in place on the token's cache rows of v and v0; other rows untouched"""
    M, HI = VAR_M, H * dh
    g = torch.Generator(device = 'cuda').manual_seed(100 + H)
    R = 2 * M + 17
    rows = torch.randperm(R, device = 'cuda', generator = g)[:M].to(torch.int32)
    vc = _rand(g, R, HI, scale = 2.).to(BF16); v0c = _rand(g, R, HI, scale = 2.).to(BF16)
    mixpre, bias = _rand(g, M, H, scale = 2.), _rand(g, H)
    before = vc.clone()
    if dh == 128:
        ops.vmix_fwd_d128(vc, HI, rows, v0c, HI, mixpre, bias, M, H)
    else:
        ops.vmix_fwd(vc, HI, rows, v0c, HI, mixpre, bias, M, H)
    torch.cuda.synchronize()
    r = rows.long()
    mix = torch.sigmoid(mixpre.double() + bias.double())[..., None]
    want = (before[r].double().reshape(M, H, dh) * mix + v0c[r].double().reshape(M, H, dh) * (1 - mix))
    check('var_bf16', row_err(vc[r], want, H, dh), dh)
    untouched = torch.ones(R, dtype = torch.bool, device = 'cuda'); untouched[r] = False
    assert torch.equal(vc[untouched], before[untouched])


@pytest.mark.parametrize('H', [2, 6, 8])
def test_vmix_bwd_vs_fp64(ops, H, dh = 64):
    """dv_raw = dvm mix in place on the v columns of dqkvg, dv_first += dvm (1 - mix) on a non-zero start, d mix_pre into its dqkvg columns
    (from 3 HI + H rounded up to even, as engine.MIX)"""
    M, HI = VAR_M, H * dh
    NQ, MIX = 3 * HI + 128, 3 * HI + (H + 1) // 2 * 2
    g = torch.Generator(device = 'cuda').manual_seed(110 + H)
    vraw, v0 = _rand(g, M, HI, scale = 2.).to(BF16), _rand(g, M, HI, scale = 2.).to(BF16)
    mixpre, bias = _rand(g, M, H, scale = 2.), _rand(g, H)
    vm = torch.zeros_like(vraw)
    vm.copy_(vraw)
    if dh == 128:
        ops.vmix_fwd_d128(vm, HI, None, v0, HI, mixpre, bias, M, H)
    else:
        ops.vmix_fwd(vm, HI, None, v0, HI, mixpre, bias, M, H)
    dvm = _rand(g, M, HI).to(BF16)
    dqkvg = torch.full((M, NQ), SENT, device = 'cuda', dtype = BF16)
    dqkvg[:, 2 * HI:3 * HI] = dvm
    dv0_start = _rand(g, M, HI)
    dv0 = dv0_start.clone()
    if dh == 128:
        ops.vmix_bwd_d128(dqkvg[:, 2 * HI:], NQ, vm, HI, v0, HI, mixpre, bias, dv0, dqkvg[:, MIX:], NQ, M, H)
    else:
        ops.vmix_bwd(dqkvg[:, 2 * HI:], NQ, vm, HI, v0, HI, mixpre, bias, dv0, dqkvg[:, MIX:], NQ, M, H)
    torch.cuda.synchronize()
    vf, v0f, mf = vraw.double().requires_grad_(True), v0.double().requires_grad_(True), mixpre.double().requires_grad_(True)
    mix = torch.sigmoid(mf + bias.double())[..., None]
    (vf.reshape(M, H, dh) * mix + v0f.reshape(M, H, dh) * (1 - mix)).reshape(M, HI).backward(dvm.double())
    check('var_bf16', row_err(dqkvg[:, 2 * HI:3 * HI], vf.grad, H, dh), dh)
    check('var_sum', row_err(dv0 - dv0_start, v0f.grad, H, dh), dh)
    # d mix_pre sums dvm (v_mixed - v0) (1 - mix): v_mixed is the bf16 the forward wrote, so its rounding scales with |v_mixed| + |v0|
    mag = (dvm.double().abs() * (vm.double().abs() + v0.double().abs())).reshape(M, H, dh).sum(-1) * (1 - mix[..., 0].detach())
    check('var_sum', row_err(dqkvg[:, MIX:MIX + H], mf.grad, H, 1, mag = mag), dh)
    assert_sentinel(dqkvg, [(2 * HI, 3 * HI), (MIX, MIX + H)])


@pytest.mark.parametrize('H', [2, 6, 8])
def test_add_f32_into_bf16_vs_fp64(ops, H):
    M, HI = VAR_M, H * 64
    NQ = 3 * HI + 128
    g = torch.Generator(device = 'cuda').manual_seed(120 + H)
    dst = _rand(g, M, HI).to(BF16)
    src = _rand(g, M, HI)
    dqkvg = torch.full((M, NQ), SENT, device = 'cuda', dtype = BF16)
    dqkvg[:, 2 * HI:3 * HI] = dst
    ops.add_f32_into_bf16(dqkvg[:, 2 * HI:], NQ, src, HI, M, HI)
    torch.cuda.synchronize()
    check('var_bf16', row_err(dqkvg[:, 2 * HI:3 * HI], dst.double() + src.double(), H))
    assert_sentinel(dqkvg, [(2 * HI, 3 * HI)])


# ================================================================================================ the layer chain in engine order
@pytest.mark.parametrize('laser', [True, False], ids = ['laser', 'plain'])
@pytest.mark.parametrize('H', [8, 2])
def test_layer_chain_vs_fp64(ops, H, laser, dh = 64, gated = True):
    """v_mixed = v mix + v0 (1 - mix) -> [v' = exp(15 tanh(v_mixed / 15))] -> o = attention(q, k, v') -> att = log(o) sigmoid(gate)
    (without LASER: att = attention(q, k, v_mixed) sigmoid(gate)), forward and backward launched as engine.forward / engine.backward do,
    against one float64 autograd graph.  Pins the D that laser_bwd_prep hands to the attention backward.  Ungated (gate_values = False):
    no sigmoid(gate) factor; gates = None into every attention, LASER and prep call, and no gate-sum buffer (dsum_mh = None)."""
    rb = make_rb([300, 129, 64, 500], [(0, 10, 90), (1, 0, 129), (3, 200, 143)])
    M, HI, T = rb.M, H * dh, tables(rb)
    NQ, MIX = 3 * HI + 128, 3 * HI + (H + 1) // 2 * 2
    g = torch.Generator(device = 'cuda').manual_seed(130 + H)
    fp = fast_params(ops, 1.1) if dh == 64 else None
    q, k = qk_inputs(rb.cu, H, INSIDE[dh], g, dh)
    vraw = _rand(g, M, HI, scale = 3.)
    vraw[torch.rand(M, HI, device = 'cuda', generator = g) < 0.02] = 30.       # values at the top of the soft clamp: v' up to ~e^15
    vraw = vraw.to(BF16)
    v0 = _rand(g, M, HI, scale = 3.).to(BF16)
    mixpre, bias, gates = _rand(g, M, H, scale = 2.), _rand(g, H), _rand(g, M, H)
    dog = _rand(g, M, HI).to(BF16)
    kgates = gates if gated else None                                       # the gates the kernels get
    # ---- forward
    v = vraw.clone()
    if dh == 128:
        ops.vmix_fwd_d128(v, HI, None, v0, HI, mixpre, bias, M, H)
    else:
        ops.vmix_fwd(v, HI, None, v0, HI, mixpre, bias, M, H)
    if laser:
        v_att = torch.zeros_like(v)
        ops.laser_v_fwd(v, HI, None, v_att, HI, M, HI // 64, 15.)
    else:
        v_att = v
    att_gates = None if laser else kgates
    o_l = torch.zeros(M, HI, device = 'cuda', dtype = BF16); lse = torch.zeros(H, M, device = 'cuda')
    attn_forward(ops, T, q, k, v_att, att_gates, H, fp, o_l, lse, dh = dh)
    if laser:
        att = torch.zeros_like(o_l)
        if dh == 128:
            ops.laser_out_fwd_d128(o_l, kgates, att, M, H)
        else:
            ops.laser_out_fwd(o_l, kgates, att, M, H)
    else:
        att = o_l
    # ---- backward
    dop = torch.zeros_like(dog); dsum = torch.zeros(H, M, device = 'cuda'); dsum_mh = torch.zeros(M, H, device = 'cuda') if gated else None
    dq = torch.full((M, HI), 7., device = 'cuda'); dk = torch.zeros(M, HI, device = 'cuda')
    if laser and dh == 128:
        ops.laser_bwd_prep_d128(dog, o_l, kgates, dop, dsum, dsum_mh, dq, M, H)
    elif laser:
        ops.laser_bwd_prep(dog, o_l, kgates, dop, dsum, dsum_mh, dq, M, H)
    elif dh == 128:
        ops.attn_bwd_prep_d128(dog, att, kgates, dop, dsum, dsum_mh, dq, M, H)
    else:
        ops.attn_bwd_prep(dog, att, kgates, dop, dsum, dsum_mh, dq, M, H)
    dqkvg = torch.full((M, NQ), SENT, device = 'cuda', dtype = BF16)
    attn_backward(ops, T, q, k, v_att, dop, lse, dsum, dq, dk, dqkvg, H, fp, dh = dh)
    if laser:
        ops.laser_v_bwd(dqkvg[:, 2 * HI:], NQ, v, HI, M, HI // 64, 15.)
    dv0_start = _rand(g, M, HI)
    dv0 = dv0_start.clone()
    if dh == 128:
        ops.vmix_bwd_d128(dqkvg[:, 2 * HI:], NQ, v, HI, v0, HI, mixpre, bias, dv0, dqkvg[:, MIX:], NQ, M, H)
    else:
        ops.vmix_bwd(dqkvg[:, 2 * HI:], NQ, v, HI, v0, HI, mixpre, bias, dv0, dqkvg[:, MIX:], NQ, M, H)
    torch.cuda.synchronize()
    assert_sentinel(dqkvg, [(2 * HI, 3 * HI), (MIX, MIX + H)])
    # ---- float64 graph
    qf, kf, vf, v0f = (t.double().requires_grad_(True) for t in (q, k, vraw, v0))
    mf, gf = mixpre.double().requires_grad_(True), gates.double().requires_grad_(True)
    mix = torch.sigmoid(mf + bias.double())[..., None]
    vm = (vf.reshape(M, H, dh) * mix + v0f.reshape(M, H, dh) * (1 - mix)).reshape(M, HI)
    vm.retain_grad()
    v_in = laser_ref(vm, 15.) if laser else vm
    o, _ = ref_attention(qf, kf, v_in, None if laser or not gated else gf, T['kv_limit'].long(), seqs_of(rb), H, dh)
    o.retain_grad()
    sgf = torch.sigmoid(gf) if gated else torch.ones_like(gf)
    out = (torch.log(o).reshape(M, H, dh) * sgf[..., None]).reshape(M, HI) if laser else o
    out.backward(dog.double())
    # magnitudes of the summed terms, carried through the elementwise steps
    mag = ref_magnitudes(q, k, v_in.detach(), None if laser else kgates, o.grad if laser else dog, T['kv_limit'], seqs_of(rb), H, dh)
    with torch.no_grad():
        t = torch.tanh(vm / 15.)
        dvatt_dvm = (torch.exp(15. * t) * (1 - t * t)).reshape(M, H, dh) if laser else 1.
        mag_dvm = mag['dv'].reshape(M, H, dh) * dvatt_dvm
        mix = mix.detach()
        sg = torch.sigmoid(gates.double())
        # d mix_pre sums dvm (v_mixed - v0) (1 - mix) over the bf16 dvm the backward wrote, whose error scales with the terms dvm sums (mag_dvm),
        # not with |dvm|: where dvm cancels, |dvm| alone understates it (the worst row grows with the number of rows: 0.46 at H = 32)
        mag_dmix = (torch.maximum(vm.grad.abs().reshape(M, H, dh), mag_dvm) * (vm.abs() + v0.double().abs()).reshape(M, H, dh)).sum(-1) * (1 - mix[..., 0])
        mag_dgate = (dog.double().abs() * torch.log(o).abs()).reshape(M, H, dh).sum(-1) * sg * (1 - sg) if laser else mag['dgate']
    check('chain_dq', row_err(dq, qf.grad, H, dh, mag = mag['dq']), dh)
    check('chain_dk', row_err(dk, kf.grad, H, dh, mag = mag['dk']), dh)
    check('chain_dv', row_err(dqkvg[:, 2 * HI:3 * HI], vf.grad, H, dh, mag = mag_dvm * mix), dh)
    check('chain_dv0', row_err(dv0 - dv0_start, v0f.grad, H, dh, mag = mag_dvm * (1 - mix)), dh)
    check('chain_dmix', row_err(dqkvg[:, MIX:MIX + H], mf.grad, H, 1, mag = mag_dmix), dh)
    if gated:
        check('chain_dgate', row_err((1 - torch.sigmoid(gates)) * dsum_mh, gf.grad, H, 1, mag = mag_dgate), dh)
