"""GPU: the kv-cache sampler kernels (csrc/decode.cu) against float64 and exact restatements, called through the C ABI with the arguments
decode.TextDecoder and decode.ode_solve pass.

    attn_decode     one query row per (sample, head) against its cache slab: keys [tile_kv0, min(tile_kvend, kv_limit[row] + 1))
    sample_tokens   greedy argmax / min-p + Gumbel-max draw (oracle/sampler_draw.py restates the draw), then the state machine update
    decode_prep     sampler state -> the eight metadata vectors of the next text step
    ode_pre / ode_post / counter_inc    one evaluation of the fixed-grid midpoint solver with classifier-free guidance

References and bounds (|got - ref| <= bound element-wise; the worst err / bound of each check is printed, run with -s):
  - attn_decode: float64 soft-capped softmax attention over the visible keys of each slab, from the same bf16 inputs.  Per (sample, head)
    the bound is the bf16 rounding of the output (2^-8 |ref|) plus E * sum_j P_j |V_j| * sigmoid(gate), where E collects the fp32 terms:
    each score is a dh-term fp32 dot product (dh * 2^-24 of sum |q k| scale, damped by the tanh's slope) plus the soft-cap's tanh
    (2^-20 absolute, times cap), twice (a score and the softmax normaliser); the __expf weights and rescales (3 * 2^-21 plus 2^-23 per unit
    of the exponent, which spans at most 2 cap, twice); and the fp32 sums of P V and of P over a warp's keys (n_w + 10 roundings, twice).
  - sample_tokens: the kernel's token must be the float64 argmax over the kept ids; a different id is accepted only when its float64
    value is within draw_error (oracle/sampler_draw.py: the fp32 error of logit / T and of the Gumbel value) of the maximum, of both.
    Greedy picks, the six state rows, the token history and counters[0] are compared exactly.
  - decode_prep and the state machine: bit for bit.  ode_pre: 1 ulp (2^-23 |ref|) of float64 y + c f_prev; f = u + cfg (c - u): 2^-24
    (2.01 |cfg (c - u)| + 1.01 |f|); y + h f: |h| times that plus 2^-24 1.01 |ref|.  The whole solve: see test_ode_solve_*.
  - bytes a kernel must not write hold a sentinel and are compared bit for bit.
Measured worst err / bound on an H100 80GB HBM3 (700 W power limit): attn_decode o 0.96, and 0.96 at dh = 128 (the bf16 rounding);
ode_post f_prev 0.98 and y 0.99 (single fp32 roundings, which the bounds state exactly); ode_pre x_eval 0.5; the whole solve 0.0075.  No tempered draw needed the
near-tie allowance.
Known difference, not tested: when min-p removes every id below vlimit the kernel returns token 0, the reference's argmax returns vlimit."""
import math

import numpy as np
import pytest
import torch

from helpers import SENT, Checks as _Checks, gen, guarded, same_bits, untouched
from oracle import sampler_draw as sd
from transfusion_pytorch_b200 import _lib
from transfusion_pytorch_b200.decode import midpoint_table
from transfusion_pytorch_b200.transfusion import MAX_HEADS, MIN_HEADS

pytestmark = pytest.mark.gpu
BF16, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
U8, U24 = 2.0 ** -8, 2.0 ** -24
CAP, LASER_C = 50., 15.
HEADS = (2, 6, 8, 16, 32)
SLAB = 1040                            # rows per cache slab: not a multiple of the 128 keys one pass of the 4 warps covers
SLAB0 = 3
FILLS = (1, 2, 31, 32, 33, 96, 127, 128, 129, 255, 256, 257, 1000, SLAB - 1)
N_DRAW = 130                           # samples of the decode-attention tests: more than 128
ISENT = -12345                         # int32 sentinel
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


def i32(a):
    return torch.as_tensor(np.asarray(a, dtype = np.int32)).cuda()


def test_heads_cover_the_accepted_range():
    assert set(HEADS) >= {MIN_HEADS, MAX_HEADS} and all(h % 2 == 0 for h in HEADS)


# ================================================================================================ tfx_attn_decode
def rms_rows(x, gamma):
    """q / k as the QKVG epilogue writes them: per-head RMSNorm times (gamma + 1), gamma per head dimension"""
    return (x / x.pow(2).mean(-1, keepdim = True).sqrt() * (gamma + 1.)).reshape(x.shape[0], -1)


# padded row pitches (q, k, v, o) per head width: the 128-wide kernel reads keys as 16-byte and values / writes outputs as 8-byte vectors
PITCH_PAD = {64: (3, 72, 6, 10), 128: (3, 72, 12, 20)}


def decode_case(H, case, seed, dh = 64):
    """slabs, query rows, tile tables and pitches of one decode-attention launch with dh-wide heads"""
    g = gen(seed)
    rng = np.random.default_rng(seed)
    HI, S = H * dh, N_DRAW
    M_q = S + 6                                           # six query rows no tile names: untouched
    pitched = case != 'gated'
    ld_q, ld_k, ld_v, ld_o = (HI + p for p in PITCH_PAD[dh]) if pitched else (HI, HI, HI, HI)
    n_rows = (SLAB0 + S + 1) * SLAB
    fill = np.array([FILLS[i % len(FILLS)] for i in range(S)])
    slab = SLAB0 + rng.permutation(S)                     # sample s owns slab slab[s]: not slab order
    rows = np.sort(rng.choice(M_q, S, replace = False))   # query row of sample s
    order = rng.permutation(S)                            # tile t holds sample order[t]
    kv0 = slab * SLAB
    mode = np.arange(S) % 3
    # mode 0: kv_limit = tile_kvend - 1 (the engine); 1: kv_limit binds, tile_kvend reaches further; 2: tile_kvend binds
    kvend = kv0 + np.where(mode == 1, np.minimum(fill + rng.integers(1, 300, S), SLAB), fill)
    kvlim_s = np.where(mode == 2, kv0 + SLAB + 500, kv0 + fill - 1)
    kv_limit = np.full(M_q, -1, dtype = np.int64); kv_limit[rows] = kvlim_s
    if case == 'saturated':                               # unnormalised: |s / cap| > 3 on most keys
        q = torch.randn(M_q, HI, device = 'cuda', generator = g) * 16.
        k = torch.randn(n_rows, HI, device = 'cuda', generator = g) * 16.
    else:
        gq, gk = (torch.randn(dh, device = 'cuda', generator = g) * 0.2 for _ in range(2))
        q = rms_rows(torch.randn(M_q, H, dh, device = 'cuda', generator = g), gq)
        k = rms_rows(torch.randn(n_rows, H, dh, device = 'cuda', generator = g), gk)
    v = torch.randn(n_rows, HI, device = 'cuda', generator = g) * 2.
    if case == 'laser':                                   # the LASER slab holds exp(c tanh(v / c))
        v = torch.exp(LASER_C * torch.tanh(v * 4. / LASER_C))
    gates = None if case == 'laser' else torch.randn(M_q, H, device = 'cuda', generator = g) * 2.
    visible = torch.zeros(n_rows, dtype = torch.bool, device = 'cuda')
    for s in range(S):
        visible[kv0[s]: min(kvend[s], kvlim_s[s] + 1)] = True
    qb = torch.full((M_q, ld_q), SENT, device = 'cuda', dtype = BF16); qb[:, :HI] = q.to(BF16)
    kb = torch.full((n_rows, ld_k), float('nan'), device = 'cuda', dtype = BF16); kb[visible, :HI] = k[visible].to(BF16)
    vb = torch.full((n_rows, ld_v), float('nan'), device = 'cuda', dtype = BF16); vb[visible, :HI] = v[visible].to(BF16)
    return dict(H = H, dh = dh, S = S, M_q = M_q, ld = (ld_q, ld_k, ld_v, ld_o), q = qb, k = kb, v = vb, gates = gates, rows = rows, order = order,
                kv0 = kv0, kvend = kvend, kv_limit = kv_limit, vis_end = np.minimum(kvend, kvlim_s + 1))


def ref_decode(c):
    """float64 output [S, H, dh] and bound per sample (row order of c['rows'])"""
    H, dh = c['H'], c['dh']
    HI = H * dh
    out, bnd = [], []
    for s in range(c['S']):
        r, a, e = int(c['rows'][s]), int(c['kv0'][s]), int(c['vis_end'][s])
        q = c['q'][r, :HI].double().reshape(H, dh) * dh ** -0.5
        k = c['k'][a:e, :HI].double().reshape(e - a, H, dh)
        v = c['v'][a:e, :HI].double().reshape(e - a, H, dh)
        d = torch.einsum('hd,jhd->hj', q, k)
        t = torch.tanh(d / CAP)
        p = torch.softmax(CAP * t, -1)
        o = torch.einsum('hj,jhd->hd', p, v)
        pv = torch.einsum('hj,jhd->hd', p, v.abs())
        dot_err = dh * U24 * torch.einsum('hd,jhd->hj', q.abs(), k.abs()) * (1 - t * t) + CAP * 2.0 ** -20
        n_w = math.ceil((e - a) / 128) * 32
        E = 2 * dot_err.amax(-1) + 3 * 2.0 ** -21 * 2 + 2 * (2 * CAP) * 2.0 ** -23 + 2 * (n_w + 10) * U24
        sg = torch.sigmoid(c['gates'][r].double()) if c['gates'] is not None else torch.ones(H, dtype = F64, device = 'cuda')
        o = o * sg[:, None]
        out.append(o); bnd.append(U8 * o.abs() + (E + 2.0 ** -20)[:, None] * pv * sg[:, None])
    return torch.stack(out), torch.stack(bnd)


@pytest.mark.parametrize('case', ['gated', 'laser', 'saturated'])
@pytest.mark.parametrize('H', HEADS)
def test_attn_decode_vs_fp64(ops, H, case, dh = 64):
    """every fill length at the edges of the 4 warps x 32 keys split, up to a full slab; samples in an order other than slab order, tiles
    in a third order; kv_limit and tile_kvend each binding; NaN in every cache row a query may not see"""
    c = decode_case(H, case, 100 + H + 7 * len(case), dh)
    ld_q, ld_k, ld_v, ld_o = c['ld']
    HI, S, M_q = H * dh, c['S'], c['M_q']
    ob, o = guarded(M_q, ld_o, BF16)
    order = c['order']
    args = (c['q'], c['k'], c['v'], ld_q, ld_k, ld_v, c['gates'], H, i32(c['kv_limit']), i32(c['rows'][order]), i32(c['kv0'][order]),
            i32(c['kvend'][order]), S, o, ld_o, dh ** -0.5, CAP)
    if dh == 128:
        ops.attn_decode_d128(*args)
    else:
        ops.attn_decode(*args)
    torch.cuda.synchronize()
    ref, bnd = ref_decode(c)
    chk = Checks(f'attn_decode dh={dh} H={H} {case}' if dh != 64 else f'attn_decode H={H} {case}')
    rows = torch.as_tensor(c['rows']).cuda()
    chk('o' if dh == 64 else f'o dh={dh}', o[rows, :HI].reshape(S, H, dh), ref, bnd)
    free = torch.ones(M_q, dtype = torch.bool, device = 'cuda'); free[rows] = False
    chk.true('rows without a tile untouched', untouched(o[free]))
    chk.true('guard row untouched', untouched(ob[M_q:]))
    chk.true('columns past H*dh untouched', untouched(o[:, HI:]))
    chk.done()


# ================================================================================================ tfx_sample_tokens
def new_state(S, rng, hist_cap = 4):
    st = np.zeros((6, S), dtype = np.int64)
    st[0] = rng.integers(0, 500, S); st[1] = rng.integers(0, 900, S); st[2] = rng.integers(0, 50, S); st[4] = rng.integers(0, 10, S)
    hb = torch.full((S + 1, hist_cap), ISENT, device = 'cuda', dtype = I32)
    return st, hb


def run_draw(ops, lg, ld, rows, V, vlimit, S, T, min_p, seed, counters, advance = 1, st = None, hist = None, hist_cap = 4, eos = -1, som = None,
             max_length = 10 ** 6):
    """one tfx_sample_tokens launch on a fresh (or given) state; returns the device state"""
    if st is None:
        st = torch.zeros(6, S, device = 'cuda', dtype = I32)
    if hist is None:
        hist = torch.full((S + 1, hist_cap), ISENT, device = 'cuda', dtype = I32)
    som_t = i32(som if som else [-1])
    ops.sample_tokens(lg, ld, rows, V, vlimit, st, S, hist, hist_cap, eos, som_t, len(som or []), max_length, T, min_p, seed, counters, advance)
    return st, hist


def keep_off_the_threshold(x, T, min_p, vlimit, rng):
    """float32 logits [R, V] with no id within 1e-4 of the min-p threshold (the kernel decides those in fp32), and at least one kept id
    below vlimit (see the known difference in the module docstring)"""
    x = x.copy()
    if min_p > 0:
        d = x.astype(np.float64) / np.float64(np.float32(T))
        d = d - d.max(1, keepdims = True) - np.log(np.float64(np.float32(min_p)))
        near = (np.abs(d) < 1e-4) & (d != -np.log(np.float64(np.float32(min_p))))
        x[near] -= np.float32(1e-2)
    if vlimit:
        for r in range(x.shape[0]):
            if not sd.kept(x[r], T, min_p, vlimit)[:vlimit].any():
                x[r, r % vlimit] = x[r].max()
    return x


def check_draws(chk, name, tok, logits, rows, T, min_p, vlimit, seed, step):
    """kernel tokens [S] against the float64 argmax of the restated draw"""
    S = len(tok)
    lg = logits[rows]
    keep = sd.kept(lg, T, min_p, vlimit)
    y, g = sd.draw_values(lg, T, seed, step, np.arange(S))
    y = np.where(keep, y, -np.inf)
    err = sd.draw_error(lg.astype(np.float64) / np.float64(np.float32(T)), g)
    best = y.argmax(1)
    i = np.arange(S)
    ok = keep[i, tok] & (y[i, tok] >= y[i, best] - err[i, tok] - err[i, best])
    chk.true(f'{name}: {int((~ok).sum())} draws are not the float64 argmax, e.g. sample {int(np.argmin(ok))}: token '
             f'{int(tok[np.argmin(ok)])} (y {y[np.argmin(ok), tok[np.argmin(ok)]]:.6g}), argmax {int(best[np.argmin(ok)])} '
             f'(y {y[np.argmin(ok), best[np.argmin(ok)]]:.6g})', ok.all())
    return int((tok != best).sum())


@pytest.mark.parametrize('V,vlimit', [(17, 0), (17, 9), (390, 0), (390, 200), (4099, 0), (4099, 2500)])
def test_tempered_draws_are_the_float64_argmax(ops, V, vlimit):
    """V below one warp's 32 lanes and not a multiple of 32, ld > V, -inf logits, the rows indirection of sample_first, several steps"""
    S, R, ld = 37, 48, V + 5
    rng = np.random.default_rng(V + vlimit)
    chk = Checks(f'sample_tokens V={V} vlimit={vlimit}')
    near = 0
    for ti, T in enumerate((0.7, 1.0, 1.3)):
        for mi, min_p in enumerate((0.0, 0.1, 1.0)):
            x = (rng.standard_normal((R, V)) * 3).astype(np.float32)
            x[rng.random((R, V)) < 0.03] = -np.inf
            x[:, 0] = np.where(rng.random(R) < 0.5, x[:, 0], -np.inf)
            x = keep_off_the_threshold(x, T, min_p, vlimit, rng)
            lgb = torch.full((R, ld), float('nan'), device = 'cuda'); lgb[:, :V] = torch.from_numpy(x).cuda()
            seed = int(rng.integers(0, 2 ** 63))
            for k, step in enumerate((None, 1, 6)):
                rows = rng.permutation(R)[:S] if (ti + mi + k) % 2 else np.arange(S)
                cnt = None if step is None else i32([0, step])
                st, _ = run_draw(ops, lgb, ld, i32(rows) if (ti + mi + k) % 2 else None, V, vlimit, S, T, min_p, seed, cnt)
                tok = st[2].cpu().numpy().astype(np.int64)
                near += check_draws(chk, f'T={T} min_p={min_p} step={step}', tok, x, rows, T, min_p, vlimit, seed, step or 0)
    print(f'sample_tokens V={V} vlimit={vlimit}: {near} draws resolved as near ties')
    chk.done()


def extreme_hashes(V, S, step):
    """(seed, sample, id) whose hash gives the largest and the smallest u, searched over seeds (vectorised)"""
    s, c = np.arange(S, dtype = np.uint64)[None, :, None], np.arange(V, dtype = np.uint64)[None, None, :]
    found = {}
    for base in range(0, 1 << 14, 32):
        seeds = np.arange(base, base + 32, dtype = np.uint64)[:, None, None]
        top = sd.draw_hash(seeds, step, s, c) >> np.uint64(40)          # the top 24 bits: 2^24 - 1 also has the largest 23
        for name, val in (('largest', (1 << 24) - 1), ('smallest', 0)):
            w = np.argwhere(top == val)
            if len(w) and name not in found:
                found[name] = (base + int(w[0][0]), int(w[0][1]), int(w[0][2]))
        if len(found) == 2:
            return found
    raise AssertionError('no extreme hash found')


def test_extreme_uniforms_draw_the_float64_argmax(ops):
    """the ids whose u is the largest (1 - 2^-24) and the smallest (2^-24) the mapping gives, planted 40 below the row maximum with
    min_p = 0: the float64 draw picks another id.  A u that rounds to 1 gives that id an infinite Gumbel value and it wins."""
    V, S, STEP = 4099, 8, 3
    found = extreme_hashes(V, S, STEP)
    chk = Checks('sample_tokens extreme u')
    for name, (seed, s, c) in found.items():
        u = sd.uniform(sd.draw_hash(seed, STEP, s, c))
        chk.true(f'{name}: restated u {u!r}', u == (1 - 2.0 ** -24 if name == 'largest' else 2.0 ** -24))
        rng = np.random.default_rng(seed)
        x = (rng.standard_normal((S, V)) * 2).astype(np.float32)
        x[s, c] = x[s].max() - 40
        st, _ = run_draw(ops, torch.from_numpy(x).cuda(), V, None, V, 0, S, 1.0, 0.0, seed, i32([0, STEP]))
        tok = st[2].cpu().numpy().astype(np.int64)
        chk.true(f'{name} u: sample {s} drew the planted id {c} (logit {x[s].max() - x[s, c]:.0f} below the maximum)', tok[s] != c)
        check_draws(chk, f'{name} u (seed {seed}, sample {s}, id {c})', tok, x, np.arange(S), 1.0, 0.0, 0, seed, STEP)
    chk.done()


def test_greedy_is_the_exact_argmax(ops):
    """ties inside one lane (ids c, c + 32 k) and across lanes resolve to the lowest id; an all -inf row gives 0 as torch.argmax does"""
    chk = Checks('sample_tokens greedy')
    for V in (17, 390, 4099):
        R, S, ld = 40, 32, V + 3
        rng = np.random.default_rng(V)
        x = rng.integers(-4, 4, (R, V)).astype(np.float32)             # many ties at the maximum
        x[0] = 0; x[0, [5, 5 + 32 * ((V - 6) // 32)]] = 9                # one lane (equal when V < 38)
        x[1] = 0; x[1, [3, V - 1]] = 9                                  # across lanes
        x[2] = -np.inf
        x[3] = -np.inf; x[3, V - 1] = -1e30
        x[4, :] = -7; x[4, V // 2] = np.inf
        want_t = torch.from_numpy(x).argmax(1).numpy()
        lgb = torch.full((R, ld), 1e9, device = 'cuda'); lgb[:, :V] = torch.from_numpy(x).cuda()       # columns past V are never read
        for rows in (None, rng.permutation(R)[:S]):
            st, _ = run_draw(ops, lgb, ld, None if rows is None else i32(rows), V, 0, S, 0.0, 0.1, 1, None)
            r = np.arange(S) if rows is None else rows
            tok = st[2].cpu().numpy()
            want = x[r].argmax(1)
            chk.true(f'V={V} rows={"given" if rows is not None else "none"}: {int((tok != want).sum())} greedy tokens differ from argmax',
                     (tok == want).all() and (want == want_t[r]).all())
    chk.done()


def restate_update(st, hist, hist_cap, tok, eos, som, max_length, advance):
    """OracleTextDecoder._update (oracle/torch_reference.py) on arrays, with the history bounded by hist_cap"""
    st, hist = st.copy(), hist.copy()
    left = 0
    for s in range(st.shape[1]):
        if st[3, s] != 0:
            continue
        t = int(tok[s])
        if st[5, s] < hist_cap:
            hist[s, st[5, s]] = t
        st[5, s] += 1; st[2, s] = t
        if advance:
            st[0, s] += 1; st[1, s] += 1
        st[4, s] += 1
        if t == eos: st[3, s] = 2
        elif st[4, s] > max_length: st[3, s] = 2
        elif t in som: st[3, s] = 1
        left += int(st[3, s] == 0)
    return st, hist, left


@pytest.mark.parametrize('advance,counters', [(1, True), (0, True), (1, False)])
@pytest.mark.parametrize('S', [1, 7, 8, 9, 4097])
def test_state_machine_matches_the_restatement(ops, S, advance, counters):
    """phases 1 and 2 untouched; [eos] and three [som] ids; num_tokens reaching max_length and max_length + 1; hist_cap overflow"""
    V, HC, EOS, SOM, MAXLEN = 390, 5, 257, [259, 300, 388], 40
    rng = np.random.default_rng(S + 10 * advance + counters)
    st0, _ = new_state(S, rng)
    st0[3] = rng.choice([0, 0, 0, 1, 2], S)
    st0[4] = rng.choice([MAXLEN - 1, MAXLEN, 3, 20], S)
    st0[5] = rng.choice([0, 2, HC - 1, HC, HC + 3], S)
    x = rng.standard_normal((S, V)).astype(np.float32)
    pick = rng.choice([EOS] + SOM + [0, 17, V - 1, 256, 258], S)
    x[np.arange(S), pick] = 10.
    hist0 = rng.integers(-1000, -1, (S, HC))
    st = torch.from_numpy(st0.astype(np.int32)).cuda()
    hb = torch.full((S + 1, HC), ISENT, device = 'cuda', dtype = I32); hb[:S] = torch.from_numpy(hist0.astype(np.int32)).cuda()
    cnt = i32([3, 5]) if counters else None
    run_draw(ops, torch.from_numpy(x).cuda(), V, None, V, 0, S, 0.0, 0.0, 9, cnt, advance = advance, st = st, hist = hb[:S], hist_cap = HC, eos = EOS,
             som = SOM, max_length = MAXLEN)
    want_st, want_hist, left = restate_update(st0, hist0, HC, pick, EOS, SOM, MAXLEN, advance)
    chk = Checks(f'sample_tokens state S={S} advance={advance} counters={counters}')
    got = st.cpu().numpy()
    for r, nm in enumerate(('len', 'tokens_seen', 'last_token', 'phase', 'num_tokens', 'hist_len')):
        chk.true(f'state row {nm}: {int((got[r] != want_st[r]).sum())} samples differ', (got[r] == want_st[r]).all())
    chk.true('hist differs', (hb[:S].cpu().numpy() == want_hist).all())
    chk.true('hist guard row written', (hb[S] == ISENT).all().item())
    if counters:
        chk.true(f'counters {cnt.tolist()}, want [{3 + left}, 5]', cnt.tolist() == [3 + left, 5])
    chk.done()


def test_draw_frequencies_follow_the_filtered_softmax(ops):
    """the uniformity of the hash, which the restatement takes as given: frequencies over 16k draws of a 12-id vocabulary follow
    softmax(min-p filtered logits / T) restricted to ids < vlimit, where the two largest logits lie past vlimit"""
    Vs, T, minp, N = 12, 0.7, 0.2, 4096
    base = torch.tensor([2.0, 1.5, 1.0, 0.0, -1.0, -3.0, 0.5, 1.8, -0.5, 0.2, 3.0, 2.5], device = 'cuda')
    lg = torch.zeros(N, 16, device = 'cuda'); lg[:, :Vs] = base
    counts = torch.zeros(Vs, device = 'cuda')
    for step in range(4):
        st, _ = run_draw(ops, lg, 16, None, Vs, 10, N, T, minp, 777, i32([0, step]), hist_cap = 2)
        counts += torch.bincount(st[2].long(), minlength = Vs).float()[:Vs]
    p = (base / T).softmax(-1)
    keep = p >= minp * p.max()
    keep[10:] = False
    want = torch.where(keep, p, torch.zeros_like(p)); want = want / want.sum()
    freq = counts / counts.sum()
    assert (counts[~keep] == 0).all()
    assert (freq - want).abs().max().item() < 0.02, (freq, want)


def test_captured_text_step_replays_like_eager_steps(ops):
    """decode_prep + a tempered sample_tokens, captured once and replayed K times = K eager steps (state, history, counters, metadata)"""
    S, V, cap, K, HC = 9, 390, 50, 6, 8
    rng = np.random.default_rng(5)
    st0, _ = new_state(S, rng)
    st0[0] = [0, 3, 48, 49, 50, 70, 10, 20, 30]
    x = torch.from_numpy((rng.standard_normal((S, V)) * 2).astype(np.float32)).cuda()
    som = i32([259])

    def fresh():
        return (torch.from_numpy(st0.astype(np.int32)).cuda(), torch.zeros(S, HC, device = 'cuda', dtype = I32), i32([0, 0]),
                torch.zeros(8, S, device = 'cuda', dtype = I32))

    def step(st, hist, cnt, meta):
        ops.decode_prep(st, S, cap, 2, meta[0], meta[1], meta[2], meta[3], meta[4], meta[5], meta[6], meta[7], cnt)
        ops.sample_tokens(x, V, None, V, 0, st, S, hist, HC, 7, som, 1, 12, 1.0, 0.05, 4242, cnt, 1)

    eager = fresh()
    for _ in range(K):
        step(*eager)
    graph = fresh()
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        step(*graph)
    for _ in range(K):
        gr.replay()
    torch.cuda.synchronize()
    for a, b, nm in zip(eager, graph, ('state', 'hist', 'counters', 'meta')):
        assert torch.equal(a, b), nm
    assert eager[2][1].item() == K


# ================================================================================================ tfx_decode_prep
@pytest.mark.parametrize('counters', [True, False])
@pytest.mark.parametrize('S', [1, 127, 128, 129, 1000])
def test_decode_prep_matches_the_restatement(ops, S, counters):
    """the metadata OracleTextDecoder.step builds: len 0 and len >= cap clamp to a row inside the slab; counters[1] advances once per
    launch over several blocks"""
    cap, slab0 = 77, 5
    rng = np.random.default_rng(S)
    st = np.zeros((6, S), dtype = np.int64)
    st[0] = rng.choice([0, 1, cap - 2, cap - 1, cap, cap + 9, 40], S); st[1] = rng.integers(0, 3000, S); st[2] = rng.integers(0, 390, S)
    st[3] = rng.integers(0, 3, S); st[4] = rng.integers(0, 9, S); st[5] = rng.integers(0, 9, S)
    outs = [torch.full((S + 3,), ISENT, device = 'cuda', dtype = I32) for _ in range(8)]
    cnt = i32([17, 41]) if counters else None
    ops.decode_prep(i32(st), S, cap, slab0, *[o[:S] for o in outs], cnt)
    ln = np.minimum(st[0], cap - 1)
    base = (slab0 + np.arange(S)) * cap
    want = [st[2], st[1], base + ln, base + ln, np.arange(S), np.arange(S) + 1, base, base + ln + 1]
    names = ('text_id', 'rope_pos', 'kv_row', 'kv_limit', 'tile_q0', 'tile_qend', 'tile_kv0', 'tile_kvend')
    chk = Checks(f'decode_prep S={S}')
    for o, w, nm in zip(outs, want, names):
        got = o.cpu().numpy()
        chk.true(f'{nm}: {int((got[:S] != w).sum())} entries differ', (got[:S] == w).all())
        chk.true(f'{nm}: guard entries written', (got[S:] == ISENT).all())
    chk.true('a cache row outside its slab', ((base + ln >= base) & (base + ln < base + cap)).all())
    if counters:
        chk.true(f'counters {cnt.tolist()}, want [0, 42]', cnt.tolist() == [0, 42])
    chk.done()


# ================================================================================================ ODE kernels
BIG_N = 132 * 8 * 256 * 2 + 77        # more than one grid-stride pass of ew_grid_d (at most 8 blocks of 256 threads per SM)
ODE_N = (1, 255, 257, BIG_N)


def test_big_n_needs_two_grid_stride_passes():
    assert BIG_N > torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256


def fsent(n):
    return torch.full((n,), SENT, device = 'cuda')


@pytest.mark.parametrize('dup', [1, 2, 3])
@pytest.mark.parametrize('n', ODE_N)
def test_ode_pre(ops, n, dup):
    """evaluation 0 (c = 0) reads no f_prev (it is NaN); evaluation 1 (c = dt / 2) gives fp32(y + c f_prev); cond_times[0 .. n_cond) = t"""
    g = gen(n + dup)
    tab = midpoint_table(5, 'cuda')
    y = torch.randn(n, device = 'cuda', generator = g) * 3
    f = torch.randn(n, device = 'cuda', generator = g) * 2
    chk = Checks(f'ode_pre n={n} dup={dup}')
    for e, fprev, n_cond in ((0, torch.full_like(f, float('nan')), 0), (1, f, n + 300 if n < 1000 else 300), (3, f, None)):
        xb = fsent(dup * n + 64)
        ct = fsent(max(n_cond or 0, 1) + 16)
        idx = i32([e])
        ops.ode_pre(y, fprev, xb, n, dup, tab, idx, None if n_cond is None else ct, n_cond or 0)
        torch.cuda.synchronize()
        t, c = tab[e, 0], tab[e, 1].item()
        x = xb[:dup * n].reshape(dup, n)
        if c == 0:
            chk.true(f'eval {e}: x_eval is not y bit for bit', all(same_bits(x[d], y) for d in range(dup)))
        else:
            ref = y.double() + c * f.double()
            for d in range(dup):
                chk(f'x_eval copy {d}', x[d], ref, 2.0 ** -23 * ref.abs())
        chk.true(f'eval {e}: x_eval tail written', untouched(xb[dup * n:]))
        k = n_cond or 0
        chk.true(f'eval {e}: cond_times[:{k}] != t', (ct[:k] == t).all().item())
        chk.true(f'eval {e}: cond_times past n_cond written', untouched(ct[k:]))
    chk.done()


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('n', ODE_N)
def test_ode_post(ops, n, mode):
    """mode 0 writes f_prev only, mode 1 y only; f = u + cfg (c - u), or pred_cond itself without guidance"""
    g = gen(3 * n + mode)
    tab = midpoint_table(5, 'cuda')
    e = mode                                          # evaluations 0 and 1 of the table have modes 0 and 1
    h = tab[e, 2].item()
    pc = torch.randn(n, device = 'cuda', generator = g) * 2
    pu = torch.randn(n, device = 'cuda', generator = g) * 2
    y0 = torch.randn(n, device = 'cuda', generator = g) * 3
    fp0 = torch.randn(n, device = 'cuda', generator = g)
    chk = Checks(f'ode_post n={n} mode={mode}')
    for cfg, guided in ((2.5, True), (1.0, False)):
        yb, fb = fsent(n + 64), fsent(n + 64)
        yb[:n] = y0; fb[:n] = fp0
        ops.ode_post(yb[:n], fb[:n], pc, pu if guided else None, cfg, n, tab, i32([e]))
        torch.cuda.synchronize()
        c64, u64 = pc.double(), pu.double()
        f = u64 + cfg * (c64 - u64) if guided else c64
        fb_err = U24 * (2.01 * (cfg * (c64 - u64)).abs() + 1.01 * f.abs()) if guided else torch.zeros_like(f)
        tag = 'guided' if guided else 'unguided'
        if mode == 0:
            chk.true(f'{tag}: y written', same_bits(yb[:n], y0))
            if guided:
                chk(f'f_prev {tag}', fb[:n], f, fb_err)
            else:
                chk.true('f_prev is not pred_cond bit for bit', same_bits(fb[:n], pc))
        else:
            chk.true(f'{tag}: f_prev written', same_bits(fb[:n], fp0))
            ref = y0.double() + h * f
            chk(f'y {tag}', yb[:n], ref, abs(h) * fb_err + U24 * 1.01 * ref.abs())
        chk.true(f'{tag}: tails written', untouched(yb[n:]) and untouched(fb[n:]))
    chk.done()


@pytest.mark.parametrize('steps', [2, 3, 9, 33])
def test_ode_solve_matches_float64_midpoint(ops, steps):
    """2 (steps - 1) evaluations driven by the device index and tfx_counter_inc, the model dy/dt = (1/2 - t) y + 1/10 + t a torch op
    reading t from cond_times, guidance cfg = 0.6 over pred_cond = f + d, pred_uncond = f - 1.5 d (combines to f).  Against the float64
    midpoint of oracle/shims/torchdiffeq on the same grid; a captured evaluation replayed 2 (steps - 1) - 1 times equals the eager loop.
    Bound: at most 32 fp32 roundings per evaluation of values below 2 (|y0| + 2) (|y| stays below e^(1/2) (|y0| + 1.1), |d| <= 1/4)."""
    from oracle.shims.torchdiffeq import odeint
    n, dup, cfg, n_evals = 4097, 2, 0.6, 2 * (steps - 1)
    g = gen(steps)
    tab = midpoint_table(steps, 'cuda')
    y0 = torch.randn(n, device = 'cuda', generator = g) * 2
    delta = torch.sin(torch.arange(n, device = 'cuda', dtype = F32)) * 0.25

    def run(use_graph):
        y, fprev, x = y0.clone(), torch.zeros(n, device = 'cuda'), torch.zeros(dup * n, device = 'cuda')
        ct, idx = torch.zeros(3, device = 'cuda'), torch.zeros(1, device = 'cuda', dtype = I32)

        def one_eval():
            ops.ode_pre(y, fprev, x, n, dup, tab, idx, ct, 3)
            t = ct[0]
            pc = (0.5 - t) * x[:n] + (0.1 + t) + delta
            pu = (0.5 - t) * x[n:] + (0.1 + t) - 1.5 * delta
            ops.ode_post(y, fprev, pc, pu, cfg, n, tab, idx)
            ops.counter_inc(idx)

        one_eval()
        if use_graph:
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                one_eval()
            for _ in range(n_evals - 1):
                gr.replay()
        else:
            for _ in range(n_evals - 1):
                one_eval()
        torch.cuda.synchronize()
        return y, idx.item(), ct.clone()

    ye, ie, cte = run(False)
    yg, ig, _ = run(True)
    grid = torch.linspace(0, 1, steps).double()
    ref = odeint(lambda t, v: (0.5 - t) * v + 0.1 + t, y0.double().cpu(), grid, method = 'midpoint')[-1].cuda()
    chk = Checks(f'ode solve steps={steps}')
    chk('y', ye, ref, U24 * 32 * n_evals * 2 * (y0.double().abs() + 2))
    chk.true('the captured replay differs from the eager loop', same_bits(yg, ye))
    chk.true(f'index {ie}, {ig} after {n_evals} evaluations', ie == ig == n_evals)
    chk.true('cond_times of the last evaluation', (cte == tab[n_evals - 1, 0]).all().item())
    chk.done()
