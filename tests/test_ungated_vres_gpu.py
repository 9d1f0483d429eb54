"""GPU: ungated attention (`attn_kwargs = dict(gate_values = False)`) and the learned value residual above 16 heads, end to end.

Kernels: the QKVG epilogue against float64 (bounds of tests/test_block_epilogues_gpu.py and tests/test_noqknorm_gpu.py) with and without the gate,
with the value-residual mix at 18 - 32 heads (the mix then runs into the second 32-column slice of the gate tile), in both norm modes and at both
head widths; a launch with neither gates nor mix_pre reads a weight without the gate tile.  The q / k backward pack without gates.
Model: the train step against the reference's own outputs (tests/golden/*ungated*.pt, small_vres_h32, small_wide1536_vres) on the bounded-logit
path and on the general kernels, the 128-wide heads against the fp32 checker, graph replay, `sample_many`, and the launches of an ungated step.
Model tolerances are those of tests/test_parity_gpu.py and tests/test_sampling_gpu.py."""
import copy

import pytest
import torch

from helpers import SENT, Checks as _Checks, c_acc, gen, golden_noise, grad_fingerprint, guarded, load_golden, same_bits, unpack_rows, untouched, compare_sampling
from test_block_epilogues_gpu import gammas, gemm64, kblocks, pair_sum, qk_forward_ref, rope64, rope_tables, N_POS, ZERO_ROW
from transfusion_pytorch_b200 import Transfusion, _lib, synth
from oracle.ungated_reference import UngatedOracleEngine

pytestmark = pytest.mark.gpu
BF16, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
U8, U24 = 2.0 ** -8, 2.0 ** -24
M_ROWS = 9011                        # not a multiple of 128 (nor of 32): the last GEMM tile and its last warp slab are partial
LOSS_REL, HID_REL, GRAD_REL = 1e-3, 2e-2, 6e-2
MARGIN_BOUND, LATENT_TOL = 0.1, 5e-2
SHOWN = {}

# (model dim D, heads H, head width, qk-RMSNorm, gated, value-residual mix): the mix past the first 32-column slice at H = 18, 24, 30, 32, the
# widths of the 1536- and 2048-wide models, both norm modes, and ungated launches with and without the mix (without: no gate tile at all)
CONFIGS = [(128, 18, 64, True, True, True), (1536, 24, 64, True, False, True), (2048, 32, 64, True, True, True), (768, 30, 64, False, True, True),
           (2048, 32, 64, False, False, True), (1536, 24, 64, False, True, False), (512, 8, 64, True, False, False), (256, 16, 64, True, False, True),
           (1024, 20, 64, False, False, False), (2048, 16, 128, True, False, True), (384, 3, 128, False, False, False), (256, 5, 128, True, True, True)]
CFG_IDS = [f'd{d}h{h}dh{dh}' + ('' if n else 'rope') + ('g' if g else 'nog') + ('mix' if m else '') for d, h, dh, n, g, m in CONFIGS]


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


@pytest.fixture(scope = 'module', autouse = True)
def _report():
    yield
    for name, r in sorted(SHOWN.items()):
        print(f'worst over the file: {name:28s} {r:.3g}')


def Checks(what):
    return _Checks(what, SHOWN)


def inputs(D, H, dh, norm, gated, mix, seed):
    g = gen(seed)
    HI = dh * H
    NQ = 3 * HI + (128 if gated or mix else 0)           # the weight has a gate tile iff the launch uses it
    u = torch.randn(M_ROWS, D, device = 'cuda', generator = g).to(BF16)
    u[ZERO_ROW] = 0
    W = (torch.randn(NQ, D, device = 'cuda', generator = g) / D ** 0.5).to(BF16)
    pos = torch.randint(0, N_POS, (M_ROWS,), device = 'cuda', generator = g, dtype = I32)
    pos[::97] = N_POS - 1
    return dict(D = D, H = H, dh = dh, HI = HI, NQ = NQ, norm = norm, gated = gated, mix = mix, u = u, W = W, gq = gammas(seed + 1, dh),
                gk = gammas(seed + 2, dh), pos = pos)


def run(ops, x, tt, gated = None, mix = None):
    """the QKVG entry point of x's head width and norm mode into fresh guarded outputs; gates / mix_pre passed as x (or the overrides) say"""
    H, HI, D = x['H'], x['HI'], x['D']
    gated = x['gated'] if gated is None else gated
    mix = x['mix'] if mix is None else mix
    out = {}
    for n, c, dt in (('q', HI, BF16), ('k', HI, BF16), ('v', HI, BF16), ('gates', H, F32), ('inv', 2 * H, F32), ('mix', H, F32)):
        out[n + '_buf'], out[n] = guarded(M_ROWS, c, dt)
    g, m = (out['gates'] if gated else None), (out['mix'] if mix else None)
    sfx = '_d128' if x['dh'] == 128 else ''
    if x['norm']:
        getattr(ops, 'gemm_qkvg' + sfx)(x['u'], D, x['W'], D, M_ROWS, H, D, out['q'], out['k'], out['v'], g, out['inv'], x['gq'], x['gk'], x['pos'], tt, N_POS, None, m)
    else:
        getattr(ops, 'gemm_qkvg_rope' + sfx)(x['u'], D, x['W'], D, M_ROWS, H, D, out['q'], out['k'], out['v'], g, x['pos'], tt, N_POS, None, m)
    return out


@pytest.mark.parametrize('D,H,dh,norm,gated,mix', CONFIGS, ids = CFG_IDS)
def test_gemm_qkvg_gate_tile_vs_float64(ops, D, H, dh, norm, gated, mix):
    x = inputs(D, H, dh, norm, gated, mix, seed = 900 + D + H + dh)
    HI, M = x['HI'], M_ROWS
    t, tt = rope_tables(ops, dh)
    o = run(ops, x, tt)
    ck = Checks(f'qkvg dh={dh} D={D} H={H} norm={int(norm)} gated={int(gated)} mix={int(mix)}')
    y, mag = gemm64(x['u'], x['W'])
    kb = kblocks(x['u'])
    ca = c_acc(kb)
    cs = t[x['pos'].long()].double()
    c, s = cs[:, None, :, 0], cs[:, None, :, 1]
    for which, gam in ((0, x['gq']), (1, x['gk'])):
        sec = slice(which * HI, (which + 1) * HI)
        ys, ms = y[:, sec].reshape(M, H, dh), mag[:, sec].reshape(M, H, dh)
        name = 'qk'[which]
        if norm:
            ref, bound, inv, rel_inv = qk_forward_ref(ys, ms, gam, c, s, kb)
            ck(f'qkvg inv_{name}', o['inv'][:, which * H:(which + 1) * H], inv[..., 0], inv[..., 0] * rel_inv[..., 0] * (1 + U8))
        else:
            ref = rope64(ys, c, s)
            bound = U8 * ref.abs() + (1 + U8) * pair_sum(ca * ms + 3 * U24 * ys.abs())
        ck(f'qkvg {name}', o[name].reshape(M, H, dh), ref, bound)
    ck('qkvg v', o['v'], y[:, 2 * HI:3 * HI], U8 * y[:, 2 * HI:3 * HI].abs() + (1 + U8) * ca * mag[:, 2 * HI:3 * HI])
    m0 = 3 * HI + (H + 1) // 2 * 2
    gsl, msl = slice(3 * HI, 3 * HI + H), slice(m0, m0 + H)
    if gated:
        ck('qkvg gates', o['gates'], y[:, gsl], ca * mag[:, gsl])
    else:
        ck.true('null gates: sentinel gate buffer untouched', untouched(o['gates_buf']))
    if mix:
        ck('qkvg mix', o['mix'], y[:, msl], ca * mag[:, msl])
    else:
        ck.true('mix buffer untouched without mix_pre', untouched(o['mix_buf']))
    if not norm:
        ck.true('qk_inv buffer untouched', untouched(o['inv_buf']))
    for n in ('q', 'k', 'v', 'gates', 'mix'):
        ck.true(f'{n}: guard row untouched', untouched(o[n + '_buf'][M]))
    # q, k, v come from the same accumulators whatever the gate tile carries: a gated launch with the mix writes the same bytes (and, where this
    # launch has them, the same gates and mix)
    if x['NQ'] > 3 * HI:
        full = run(ops, x, tt, gated = True, mix = True)
        for n in ('q', 'k', 'v') + (('gates',) if gated else ()) + (('mix',) if mix else ()):
            ck.true(f'{n} = gated mix launch bytes', same_bits(o[n], full[n]))
    ck.done()


def test_gemm_qkvg_without_gate_tile_reads_no_weight_past_v(ops):
    """with neither gates nor mix_pre the GEMM's N is 3 H DH: the weight rows behind to_v are not read (here: NaN rows behind a 3 H DH view)"""
    D, H = 512, 8
    x = inputs(D, H, 64, True, False, False, seed = 31)
    HI = x['HI']
    t, tt = rope_tables(ops, 64)
    ref = run(ops, x, tt)
    Wn = torch.full((3 * HI + 128, D), float('nan'), device = 'cuda', dtype = BF16)
    Wn[:3 * HI] = x['W']
    o = run(ops, dict(x, W = Wn), tt)
    for n in ('q', 'k', 'v', 'inv'):
        assert same_bits(o[n], ref[n]), n
    assert untouched(o['gates_buf']) and untouched(o['mix_buf'])


@pytest.mark.parametrize('H,dh,norm', [(18, 64, True), (32, 64, False), (8, 64, True), (3, 128, True), (16, 128, False)])
def test_qk_bwd_pack_without_gates(ops, H, dh, norm):
    """gates = None: the q / k columns are the gated pack's bytes (float64-checked in tests/test_block_epilogues_gpu.py and
    tests/test_noqknorm_gpu.py) and, for the RoPE-only pack, R(pos)^T d against float64 here; no gate column is written and dsum is not read"""
    D = 512
    x = inputs(D, H, dh, norm, True, False, seed = 1200 + H + dh)
    HI, NQ, M = x['HI'], x['NQ'], M_ROWS
    t, tt = rope_tables(ops, dh)
    o = run(ops, x, tt)
    g = gen(1300 + H)
    dq = torch.randn(M, HI, device = 'cuda', generator = g); dk = torch.randn(M, HI, device = 'cuda', generator = g)
    dsum = torch.randn(M, H, device = 'cuda', generator = g)
    sfx = '_d128' if dh == 128 else ''
    outs = {}
    for gated in (True, False):
        buf, out = guarded(M, NQ, BF16)
        dgam = torch.zeros(2, dh, device = 'cuda')
        gg, ds = (o['gates'], dsum) if gated else (None, None)
        if norm:
            getattr(ops, 'qk_bwd_pack' + sfx)(dq, dk, o['q'], o['k'], o['inv'], x['gq'], x['gk'], x['pos'], t, gg, ds, out, NQ, dgam[0], dgam[1], M, H)
        else:
            getattr(ops, 'qk_bwd_pack_rope' + sfx)(dq, dk, x['pos'], t, gg, ds, out, NQ, M, H)
        outs[gated] = (buf, out, dgam)
    ck = Checks(f'qk_bwd_pack dh={dh} H={H} norm={int(norm)} ungated')
    (_, og, dgg), (nbuf, on, dgn) = outs[True], outs[False]
    ck.true('q / k columns = gated pack bytes', same_bits(on[:, :2 * HI], og[:, :2 * HI]))
    # dgamma is summed with atomics (order-dependent last bits): equal up to fp32 reorderings of the gated pack's sum
    ck('dgamma = gated pack (atomic sum order)', dgn, dgg.double(), 1e-5 * dgg.double().abs().max())
    ck.true('gate, dv and pad columns untouched', untouched(on[:, 2 * HI:]))
    ck.true('guard row untouched', untouched(nbuf[M]))
    if not norm:
        cs = t[x['pos'].long()].double()
        c, s = cs[:, None, None, :, 0], cs[:, None, None, :, 1]
        xx = torch.zeros(M, 2, H, dh, device = 'cuda', dtype = F64, requires_grad = True)
        d64 = torch.stack((dq, dk), 1).double().reshape(M, 2, H, dh)
        (rope64(xx, c, s) * d64).sum().backward()
        ck('qk_bwd_rope dx (ungated)', on[:, :2 * HI].reshape(M, 2, H, dh), xx.grad, U8 * xx.grad.abs() + (1 + U8) * 3 * U24 * pair_sum(d64.abs()))
    ck.done()


# ================================================================================================ model
def build(fx_or_ctor, seed = None):
    ctor, seed = (fx_or_ctor['ctor'], fx_or_ctor['seed']) if seed is None else (fx_or_ctor, seed)
    torch.manual_seed(0)
    model = Transfusion(**ctor).cuda()
    synth.fill_parameters_(model, seed = seed)
    return model.eval()


def rel_max(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp(min = 1e-9)).item()


def check_grads(model, fx):
    fp = grad_fingerprint((n, p.grad) for n, p in model.named_parameters() if p.grad is not None)
    assert set(fx['grads']) <= set(fp)
    for k, v in fx['grads'].items():
        ref_n = max(v['stats'][3].item(), 1e-12)
        assert abs(fp[k]['stats'][2].item() - v['stats'][2].item()) / ref_n < GRAD_REL, k
        assert abs(fp[k]['stats'][3].item() - v['stats'][3].item()) / ref_n < GRAD_REL, k


@pytest.mark.parametrize('name', ['small_ungated', 'small_ungated_laser_vres', 'small_ungated_noqknorm', 'small_vres_h32', 'small_wide1536_vres'])
def test_train_step_matches_reference(name):
    """depth 4 (two U-Net skips) or, at width 1536, 2; two modality types.  small_ungated and small_ungated_laser_vres run the bounded-logit
    kernels (64-wide normed heads), small_ungated_noqknorm the general ones; small_vres_h32 (32 heads) and small_wide1536_vres (24) mix values
    from the second 32-column slice of the gate tile"""
    fx = load_golden(name)
    model = build(fx)
    batch = synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = golden_noise(fx, batch, model.dim_latents))
    rb = model._last_batch
    assert rb.modality_positions == fx['modality_positions'] and rb.total_tokens == fx['total_tokens']
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < LOSS_REL
    assert abs(bd.text.item() - fx['text_loss'].item()) / fx['text_loss'].item() < LOSS_REL
    assert all(abs(a.item() - b.item()) / b.item() < LOSS_REL for a, b in zip(bd.flow, fx['flow_losses']))
    st = model.engine.state
    rows = fx['hidden_rows']
    cols = fx.get('hidden_cols')
    for l, h in enumerate(fx['hiddens'] + [fx['embed']]):
        ours = unpack_rows(st['hid'][l] if l < len(fx['hiddens']) else st['out'], rb)
        if cols is not None:
            ours = ours[..., cols.to(ours.device)]
        for b in range(rb.B):
            k = rows < int(rb.seq_lens[b])
            assert rel_max(ours[b, rows[k]], h[b, k]) < HID_REL, f'hidden {l} sample {b}'
    loss.backward()
    assert sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None) == fx['no_grad']
    check_grads(model, fx)


def test_dh128_ungated_matches_checker():
    """128-wide heads (general kernels) without the gate: loss and gradients against the fp32 checker on the host"""
    ctor = dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)), prob_uncond = 0.,
                transformer = dict(dim = 256, depth = 4, heads = 3, dim_head = 128, attn_kwargs = dict(gate_values = False)))
    batch = synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)
    fx = load_golden('small_ungated')                   # the same batch: its times and noise
    out = {}
    for dev in ('cuda', 'cpu'):
        torch.manual_seed(0)
        model = Transfusion(**ctor)
        synth.fill_parameters_(model, seed = 3)
        model = model.to(dev).eval()
        if dev == 'cpu':
            model._engine = UngatedOracleEngine(model)
        loss = model(batch, times = fx['times'], noise = golden_noise(fx, batch, model.dim_latents))
        loss.backward()
        out[dev] = (loss.item(), {n: p.grad.detach().float().cpu().clone() for n, p in model.named_parameters() if p.grad is not None})
    (lc, gc), (lo, go) = out['cuda'], out['cpu']
    assert abs(lc - lo) / abs(lo) < LOSS_REL, (lc, lo)
    assert set(gc) == set(go) and not any('to_gates' in n for n in gc)
    for n in gc:
        if any(k in n for k in ('to_qk', 'to_v', 'to_out', 'net.0.weight')):
            assert (gc[n] - go[n]).norm() / go[n].norm().clamp(min = 1e-12) < GRAD_REL, n


def _small_batch():
    batch = synth.small_batch(4, seed = 3, dim_latent = 32, text_vocab = 64)
    nm = max(sum(torch.is_tensor(p) and p.is_floating_point() for p in s) for s in batch)
    times = torch.rand(4, nm, generator = torch.Generator().manual_seed(1))
    rows = sum(p.shape[0] for s in batch for p in s if torch.is_tensor(p) and p.is_floating_point())
    return batch, times, rows


CTOR_SMALL = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0.,
                  transformer = dict(dim = 128, depth = 2, heads = 2, attn_kwargs = dict(gate_values = False)))


def test_graph_replay_follows_eager_trajectory():
    from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
    batch, times, rows = _small_batch()
    results = []
    for use_graph in (False, True):
        model = build(CTOR_SMALL, 7).train()
        tr = DataParallelTrainer(model, lr = 1e-3, cuda_graph = use_graph)
        losses = []
        for step in range(6):
            noise = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(500 + step))]
            losses.append(tr.step(batch, times = times, noise = noise).item())
        results.append((losses, model.engine.flat.clone()))
        if use_graph:
            assert any(g.graph is not None for g in tr._graphs.values()), 'the step was never captured'
    (l0, p0), (l1, p1) = results
    assert all(abs(a - b) / abs(a) < 2e-3 for a, b in zip(l0, l1)), (l0, l1)
    assert (p1 - p0).abs().max().item() < 2e-3 * p0.abs().max().item() + 2e-4


def test_sample_many_vs_reference_with_margins():
    fx = load_golden('sampling_ungated')
    model = build(fx)
    out = model.sample_many(copy.deepcopy(fx['prompts']), init_modality_noise = fx['noise'], **fx['kw'])
    rep = compare_sampling(model, out, fx, bound = MARGIN_BOUND, lat_tol = LATENT_TOL)
    assert len(rep) == len(fx['samples']) and all(len(r['latent_err']) >= 1 for r in rep)
    eager = model.sample_many(copy.deepcopy(fx['prompts']), init_modality_noise = fx['noise'], use_cuda_graph = False, **fx['kw'])
    for a, b in zip(out, eager):
        for p, q in zip(a, b):
            assert torch.equal(p.cpu(), q.cpu()) if torch.is_tensor(p) else torch.equal(p[1].cpu(), q[1].cpu())


def _calls(model, batch, times, noise):
    """entry point -> list of argument tuples of one eager train step"""
    eng = model.engine
    eng.ensure_attached()
    eng.ops.timing = {}
    loss = model(batch, times = times, noise = noise)
    loss.backward()
    torch.cuda.synchronize()
    calls = {n: [a for _, _, a in v] for n, v in eng.ops.timing.items()}
    eng.ops.timing = None
    return calls


@pytest.mark.parametrize('vres', [False, True])
def test_ungated_step_launches_no_gate_work(vres):
    """no gate buffer reaches any kernel; without the value residual every QKVG GEMM is given the 3 HI-row weight (N = 3 HI) and the packed
    gradient has 3 HI columns; with it, only the layers that have a mix Linear pass mix_pre (the first layer's launch then has no gate tile)"""
    batch, times, rows = _small_batch()
    ctor = copy.deepcopy(CTOR_SMALL)
    ctor['transformer'].update(depth = 3, use_value_residual = vres)
    model = build(ctor, 7).train()
    eng = model.engine
    noise = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(5))]
    calls = _calls(model, batch, times, noise)
    HI = eng.HI
    assert eng.NQ == 3 * HI + (128 if vres else 0)
    qk = calls['gemm_qkvg']
    assert len(qk) == 3
    for i, a in enumerate(qk):
        assert a[10] is None, 'gates passed to gemm_qkvg'
        assert a[2].shape[0] == eng.NQ and (a[18] is not None) == (vres and i > 0)
    for name, gi in (('attn_fwd_tc', 6), ('attn_fwd', 6), ('attn_bwd_prep', 2), ('qk_bwd_pack', 9)):
        assert all(a[gi] is None for a in calls[name]), name
    assert all(a[5] is None for a in calls['attn_bwd_prep'])           # no gate sums
    assert all(a[11].shape[1] == eng.NQ for a in calls['qk_bwd_pack'])
    if not vres:
        assert eng.packed['qkvg0'].shape == (3 * HI, eng.D)
