"""GPU: `Transformer(qk_rmsnorm = False)` end to end - the RoPE-only QKVG epilogue (tfx_gemm_qkvg_rope) and its backward (tfx_qk_bwd_pack_rope)
against float64, the engine's routing (general running-maximum attention kernels only, no bounded-logit launches), parity with the reference's
own outputs (tests/golden/*noqknorm*.pt), a layer whose logits leave the bounded path's range, graph replay, and the q / k norm gammas that no
optimizer may touch.

Kernel bounds follow tests/test_block_epilogues_gpu.py (same constants): q / k = RoPE(y) with y the float64 GEMM of the same bf16 operands; the
accumulator error C_ACC |u| |W|^T of both elements of a rope pair reaches each output, plus a few fp32 roundings and the bf16 cast.  The backward
is float64 autograd of RoPE from the same fp32 gradients: two fp32 products and a sum per element, then the bf16 cast.
Model tolerances are those of tests/test_parity_gpu.py and tests/test_sampling_gpu.py."""
import copy

import pytest
import torch

from helpers import SENT, Checks as _Checks, gen, golden_noise, grad_fingerprint, guarded, load_golden, same_bits, unpack_rows, untouched, compare_sampling
from transfusion_pytorch_b200 import Transfusion, _lib, synth
from oracle.noqknorm_reference import NoQkNormOracleEngine

pytestmark = pytest.mark.gpu
BF16, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
U8, U24 = 2.0 ** -8, 2.0 ** -24
C_ACC = 1.6e-6                       # fp32 accumulation of the wgmma GEMMs relative to |u| @ |W|^T (tests/test_block_epilogues_gpu.py)
M_ROWS = 9011                        # not a multiple of 128 (nor of 32): the last GEMM tile and its last warp slab are partial
N_POS = 16384
LOSS_REL, HID_REL, GRAD_REL = 1e-3, 2e-2, 6e-2
MARGIN_BOUND, LATENT_TOL = 0.1, 5e-2
HEADS = list(range(2, 33, 2))
DISPATCH_D = (128, 256, 384, 512, 768, 1024)
SHOWN = {}


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


def Checks(what):
    return _Checks(what, SHOWN)


def rope_tables(ops, dh = 64):
    freqs = 1. / (10000 ** (torch.arange(0, dh, 2, device = 'cuda').float() / dh))
    t = torch.empty(N_POS, dh // 2, 2, device = 'cuda'); tt = torch.empty(dh // 2, N_POS, 2, device = 'cuda')
    ops.rope_table(freqs, t, tt, N_POS, dh // 2)
    return t, tt


def rope64(y, c, s):
    y0, y1 = y[..., 0::2], y[..., 1::2]
    return torch.stack((y0 * c - y1 * s, y1 * c + y0 * s), -1).flatten(-2)


def pair_sum(x):
    return (x[..., 0::2] + x[..., 1::2]).repeat_interleave(2, -1)


def inputs(H, seed, dh = 64):
    D = DISPATCH_D[(H // 2) % len(DISPATCH_D)]
    g = gen(seed)
    HI, NQ = dh * H, 3 * dh * H + 128
    u = torch.randn(M_ROWS, D, device = 'cuda', generator = g).to(BF16)
    W = (torch.randn(NQ, D, device = 'cuda', generator = g) / D ** 0.5).to(BF16)
    gq, gk = (torch.rand(dh, device = 'cuda', generator = g) * 1.9 - 0.9 for _ in range(2))
    pos = torch.randint(0, N_POS, (M_ROWS,), device = 'cuda', generator = g, dtype = I32)
    pos[::97] = N_POS - 1
    return dict(D = D, H = H, dh = dh, HI = HI, NQ = NQ, mix = H <= 16, u = u, W = W, gq = gq, gk = gk, pos = pos)


def run(ops, x, tt, rope_only, M = M_ROWS, kv = None):
    """gemm_qkvg_rope or gemm_qkvg (their _d128 twins for 128-wide heads) into fresh guarded outputs"""
    H, HI, D = x['H'], x['HI'], x['D']
    out = {}
    for n, c, dt in (('q', HI, BF16), ('k', HI, BF16), ('v', HI, BF16), ('gates', H, F32), ('inv', 2 * H, F32), ('mix', H, F32)):
        out[n + '_buf'], out[n] = guarded(M, c, dt)
    k, v, rows = kv if kv is not None else (out['k'], out['v'], None)
    mix = out['mix'] if x['mix'] else None
    rope_args = (x['u'], D, x['W'], D, M, H, D, out['q'], k, v, out['gates'], x['pos'], tt, N_POS, rows, mix)
    norm_args = (x['u'], D, x['W'], D, M, H, D, out['q'], k, v, out['gates'], out['inv'], x['gq'], x['gk'], x['pos'], tt, N_POS, rows, mix)
    if rope_only and x['dh'] == 128:
        ops.gemm_qkvg_rope_d128(*rope_args)
    elif rope_only:
        ops.gemm_qkvg_rope(*rope_args)
    elif x['dh'] == 128:
        ops.gemm_qkvg_d128(*norm_args)
    else:
        ops.gemm_qkvg(*norm_args)
    return out


# ================================================================================================ kernels
@pytest.mark.parametrize('H', HEADS)
def test_gemm_qkvg_rope_vs_float64(ops, H, dh = 64):
    x = inputs(H, seed = 500 + H, dh = dh)
    HI, M = x['HI'], M_ROWS
    t, tt = rope_tables(ops, dh)
    o = run(ops, x, tt, rope_only = True)
    ck = Checks(f'qkvg_rope dh={dh} D={x["D"]} H={H}')
    a64, w64 = x['u'].double(), x['W'].double()
    y, mag = a64 @ w64.t(), a64.abs() @ w64.abs().t()
    cs = t[x['pos'].long()].double()
    c, s = cs[:, None, :, 0], cs[:, None, :, 1]
    for which, name in ((0, 'q'), (1, 'k')):
        sec = slice(which * HI, (which + 1) * HI)
        ys, ms = y[:, sec].reshape(M, H, dh), mag[:, sec].reshape(M, H, dh)
        ref = rope64(ys, c, s)
        ck(f'qkvg_rope {name}', o[name].reshape(M, H, dh), ref, U8 * ref.abs() + (1 + U8) * pair_sum(C_ACC * ms + 3 * U24 * ys.abs()))
    # v, gates and mix come from the same accumulators as gemm_qkvg's: identical bytes
    n = run(ops, x, tt, rope_only = False)
    for name in ('v', 'gates') + (('mix',) if x['mix'] else ()):
        ck.true(f'{name} = gemm_qkvg bytes', same_bits(o[name], n[name]))
    if not x['mix']:
        ck.true('mix buffer untouched without mix_pre', untouched(o['mix_buf']))
    ck.true('qk_inv buffer untouched', untouched(o['inv_buf']))
    for name in ('q', 'k', 'v', 'gates'):
        ck.true(f'{name}: guard row untouched', untouched(o[name + '_buf'][M]))
    # kv-cache append: k / v rows land at kv_rows[m] of a larger matrix; everything else is the dense call's bytes
    R = 2 * M + 50
    rows = torch.randperm(R, device = 'cuda', generator = gen(7))[:M].to(I32)
    kc, vc = (torch.full((R, HI), SENT, device = 'cuda', dtype = BF16) for _ in range(2))
    o2 = run(ops, x, tt, rope_only = True, kv = (kc, vc, rows))
    ck.true('kv_rows: q, gates = dense bytes', same_bits(o2['q'], o['q']) and same_bits(o2['gates'], o['gates']))
    ck.true('kv_rows: dense k, v untouched', untouched(o2['k_buf']) and untouched(o2['v_buf']))
    ck.true('kv_rows: cache rows = dense k, v bytes', same_bits(kc[rows.long()], o['k']) and same_bits(vc[rows.long()], o['v']))
    other = torch.ones(R, dtype = torch.bool, device = 'cuda'); other[rows.long()] = False
    ck.true('kv_rows: other cache rows untouched', untouched(kc[other]) and untouched(vc[other]))
    ck.done()


@pytest.mark.parametrize('H', HEADS)
def test_qk_bwd_pack_rope_vs_float64(ops, H, dh = 64):
    x = inputs(H, seed = 700 + H, dh = dh)
    HI, NQ, M = x['HI'], x['NQ'], M_ROWS
    t, tt = rope_tables(ops, dh)
    o = run(ops, x, tt, rope_only = True)
    g = gen(800 + H)
    dq = torch.randn(M, HI, device = 'cuda', generator = g); dk = torch.randn(M, HI, device = 'cuda', generator = g)
    dsum = torch.randn(M, H, device = 'cuda', generator = g)
    out_buf, out = guarded(M, NQ, BF16)
    if dh == 128:
        ops.qk_bwd_pack_rope_d128(dq, dk, x['pos'], t, o['gates'], dsum, out, NQ, M, H)
    else:
        ops.qk_bwd_pack_rope(dq, dk, x['pos'], t, o['gates'], dsum, out, NQ, M, H)
    ck = Checks(f'qk_bwd_pack_rope dh={dh} H={H}')
    cs = t[x['pos'].long()].double()
    c, s = cs[:, None, None, :, 0], cs[:, None, None, :, 1]
    xx = torch.zeros(M, 2, H, dh, device = 'cuda', dtype = F64, requires_grad = True)
    d64 = torch.stack((dq, dk), 1).double().reshape(M, 2, H, dh)
    (rope64(xx, c, s) * d64).sum().backward()
    ref = xx.grad
    ck('qk_bwd_rope dx', out[:, :2 * HI].reshape(M, 2, H, dh), ref, U8 * ref.abs() + (1 + U8) * 3 * U24 * pair_sum(d64.abs()))
    # the gate column is qk_bwd_pack's, bit for bit
    n_buf, n = guarded(M, NQ, BF16)
    on = run(ops, x, tt, rope_only = False)
    dgam = torch.zeros(2, dh, device = 'cuda')
    pack_args = (dq, dk, on['q'], on['k'], on['inv'], x['gq'], x['gk'], x['pos'], t, o['gates'], dsum, n, NQ, dgam[0], dgam[1], M, H)
    if dh == 128:
        ops.qk_bwd_pack_d128(*pack_args)
    else:
        ops.qk_bwd_pack(*pack_args)
    ck.true('gate column = qk_bwd_pack bytes', same_bits(out[:, 3 * HI:3 * HI + H], n[:, 3 * HI:3 * HI + H]))
    ck.true('dv columns untouched', untouched(out[:, 2 * HI:3 * HI]))
    ck.true('pad columns untouched', untouched(out[:, 3 * HI + H:]))
    ck.true('guard row untouched', untouched(out_buf[M]))
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


def gammas(model):
    return {n: p for n, p in model.named_parameters() if n.endswith(('.fn.q_norm.gamma', '.fn.k_norm.gamma'))}


def check_grads(model, fx):
    fp = grad_fingerprint((n, p.grad) for n, p in model.named_parameters() if p.grad is not None)
    assert set(fx['grads']) <= set(fp)
    for k, v in fx['grads'].items():
        ref_n = max(v['stats'][3].item(), 1e-12)
        assert abs(fp[k]['stats'][2].item() - v['stats'][2].item()) / ref_n < GRAD_REL, k
        assert abs(fp[k]['stats'][3].item() - v['stats'][3].item()) / ref_n < GRAD_REL, k


@pytest.mark.parametrize('name', ['small_noqknorm', 'small_noqknorm_laser_vres'])
def test_train_step_matches_reference(name):
    """depth 4 (two U-Net skips), two modality types; 'small_noqknorm_laser_vres' adds `attn_laser = True, use_value_residual = True`"""
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
    rows = fx['hidden_rows']                            # the positions the fixture keeps
    for l, h in enumerate(fx['hiddens'] + [fx['embed']]):
        ours = unpack_rows(st['hid'][l] if l < len(fx['hiddens']) else st['out'], rb)
        for b in range(rb.B):
            k = rows < int(rb.seq_lens[b])
            assert rel_max(ours[b, rows[k]], h[b, k]) < HID_REL, f'hidden {l} sample {b}'
    loss.backward()
    assert sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None) == fx['no_grad']
    check_grads(model, fx)


def test_text_only_loss_grads_greedy_tokens_and_cache():
    fx = load_golden('text_noqknorm')
    model = build(fx)
    text = synth.text_batch(4, 257, seed = 3)
    loss = model(text)
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < LOSS_REL
    loss.backward()
    assert all(p.grad is None for p in gammas(model).values())
    check_grads(model, fx)
    # free-running greedy generation through the kv cache (prefill + captured decode graph): tokens equal up to the first reference near-tie
    gen_ = model.generate_text_only(text[:, :fx['prompt_len']], fx['gen_len'], temperature = 0.).cpu()
    ref, margins = fx['generated'], fx['margins']
    assert gen_.shape == ref.shape
    for b in range(gen_.shape[0]):
        neq = (gen_[b] != ref[b]).nonzero()
        if neq.numel():
            k = int(neq[0])
            assert margins[b, k].item() < MARGIN_BOUND, f'row {b}: token {k} differs although the reference margin is {margins[b, k].item():.4f}'
    assert torch.equal(gen_, model.generate_text_only(text[:, :fx['prompt_len']], fx['gen_len'], temperature = 0., use_cuda_graph = False).cpu())
    # cached forward_text token by token (decode attention) equals one un-cached causal forward (general attention)
    text = synth.text_batch(3, 300, seed = 9).cuda()
    with torch.no_grad():
        full = model.forward_text(text[:, :200], return_loss = False).float()
        lg, cache = model.forward_text(text[:, :150], return_loss = False, return_kv_cache = True)
        outs = [lg.float()]
        for j in range(150, 200):
            lg, cache = model.forward_text(text[:, j:j + 1], return_loss = False, cache = cache, return_kv_cache = True)
            outs.append(lg.float())
    assert (torch.cat(outs, dim = 1) - full).abs().max().item() < 2e-2 * full.abs().max().item()


def test_sample_many_vs_reference_with_margins():
    fx = load_golden('sampling_noqknorm')
    model = build(fx)
    out = model.sample_many(copy.deepcopy(fx['prompts']), init_modality_noise = fx['noise'], **fx['kw'])
    rep = compare_sampling(model, out, fx, bound = MARGIN_BOUND, lat_tol = LATENT_TOL)
    assert len(rep) == len(fx['samples']) and all(len(r['latent_err']) >= 1 for r in rep)     # the forced modality is decoded before any text
    eager = model.sample_many(copy.deepcopy(fx['prompts']), init_modality_noise = fx['noise'], use_cuda_graph = False, **fx['kw'])
    for a, b in zip(out, eager):
        for p, q in zip(a, b):
            assert torch.equal(p.cpu(), q.cpu()) if torch.is_tensor(p) else torch.equal(p[1].cpu(), q[1].cpu())


def vs_checker(ctor, batch, times, noise, seed, scale_qk = 1.):
    """loss, breakdown and a sample of gradients of the CUDA engine against the fp32 checker (NoQkNormOracleEngine) on the host"""
    out = {}
    for dev in ('cuda', 'cpu'):
        torch.manual_seed(0)
        model = Transfusion(**ctor)
        synth.fill_parameters_(model, seed = seed)
        with torch.no_grad():
            for n, p in model.named_parameters():
                if n.endswith('.fn.to_qk.0.weight'):
                    p.mul_(scale_qk)
        model = model.to(dev).eval()
        if dev == 'cpu':
            model._engine = NoQkNormOracleEngine(model)
        loss, bd = model(batch, times = times, noise = noise, return_breakdown = True)
        loss.backward()
        grads = {n: p.grad.detach().float().cpu().clone() for n, p in model.named_parameters()
                 if p.grad is not None and any(k in n for k in ('to_qk', 'to_v', 'to_out', 'net.0.weight', 'text_embed'))}
        out[dev] = (loss.item(), bd.text.item(), [f.item() for f in bd.flow], grads, model)
    (lc, tc, fc, gc, mc), (lo, to_, fo, go, _) = out['cuda'], out['cpu']
    assert abs(lc - lo) / abs(lo) < LOSS_REL and abs(tc - to_) / abs(to_) < LOSS_REL, (lc, lo, tc, to_)
    assert all(abs(a - b) / abs(b) < LOSS_REL for a, b in zip(fc, fo)), (fc, fo)
    assert set(gc) == set(go) and len(gc) >= 8
    for n in gc:
        assert (gc[n] - go[n]).norm() / go[n].norm().clamp(min = 1e-12) < GRAD_REL, n
    return mc


def test_config2_matches_checker():
    ctor = dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), prob_uncond = 0., transformer = dict(dim = 512, depth = 8, qk_rmsnorm = False))
    vs_checker(ctor, synth.config2_batch(2, seed = 4), synth.config2_times(2, seed = 4), [torch.randn(1024, 384, generator = torch.Generator().manual_seed(3))], seed = 4)


def test_logits_past_the_bounded_range_match_float64_attention():
    """to_qk scaled so that |s / cap| reaches 1.2, far past 0.75 (where the bounded kernels' polynomial tanh and fixed softmax maximum stop being
    valid): the general kernel's gated output equals a dense float64 soft-capped attention of the same bf16 q / k / v, and the whole step
    matches the fp32 checker"""
    ctor = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0., transformer = dict(dim = 128, depth = 2, heads = 2, qk_rmsnorm = False))
    batch = synth.small_batch(3, seed = 1, dim_latent = 32, text_vocab = 64)
    nm = max(sum(torch.is_tensor(p) and p.is_floating_point() for p in s) for s in batch)
    times = torch.rand(3, nm, generator = torch.Generator().manual_seed(5))
    rows = sum(p.shape[0] for s in batch for p in s if torch.is_tensor(p) and p.is_floating_point())
    noise = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(4))]
    model = vs_checker(ctor, batch, times, noise, seed = 1, scale_qk = 3.)
    eng, rb = model.engine, model._last_batch
    cap, H = eng.softcap, eng.H
    kv_limit = rb.dev['kv_limit'].long().cpu()
    worst = 0.
    for L in eng.state['layers']:
        q, k, v = (L[n].double().cpu().reshape(-1, H, 64) for n in ('q', 'k', 'v'))
        sg = torch.sigmoid(L['gates'].double().cpu())
        got = L['att'].double().cpu().reshape(-1, H, 64)
        for b in range(rb.B):
            r0, r1 = int(rb.cu[b]), int(rb.cu[b + 1])
            raw = torch.einsum('ihd,jhd->hij', q[r0:r1], k[r0:r1]) * eng.scale
            worst = max(worst, (raw / cap).abs().max().item())
            sim = (raw / cap).tanh() * cap
            j = torch.arange(r0, r1)
            sim = sim.masked_fill(~(j[None, None, :] <= kv_limit[r0:r1, None][None]), float('-inf'))
            p = sim.softmax(-1)
            ref = torch.einsum('hij,jhd->ihd', p, v[r0:r1]) * sg[r0:r1, :, None]
            # bf16 probabilities / output: 2^-8 of sum_j p |v| and of the output, times the gate
            pv = torch.einsum('hij,jhd->ihd', p, v[r0:r1].abs()) * sg[r0:r1, :, None]
            err = (got[r0:r1] - ref).abs()
            assert (err <= 4 * U8 * pv + U8 * ref.abs() + 1e-6).all(), (err / (4 * U8 * pv + U8 * ref.abs() + 1e-6)).max().item()
    assert worst > 1., f'the scaled weights give |s / cap| up to {worst:.2f} only'


def _launches(model, batch, times, noise):
    eng = model.engine
    eng.ensure_attached()
    eng.ops.timing, eng.ops.order = {}, []
    loss = model(batch, times = times, noise = noise)
    loss.backward()
    torch.cuda.synchronize()
    order = eng.ops.order
    eng.ops.timing = eng.ops.order = None
    return order


def test_step_launches_only_the_general_attention_kernels():
    base = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0.)
    batch = synth.small_batch(3, seed = 1, dim_latent = 32, text_vocab = 64)
    nm = max(sum(torch.is_tensor(p) and p.is_floating_point() for p in s) for s in batch)
    times = torch.rand(3, nm, generator = torch.Generator().manual_seed(5))
    rows = sum(p.shape[0] for s in batch for p in s if torch.is_tensor(p) and p.is_floating_point())
    noise = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(4))]
    normed = _launches(build(dict(base, transformer = dict(dim = 128, depth = 2, heads = 2)), 1).train(), batch, times, noise)
    plain = _launches(build(dict(base, transformer = dict(dim = 128, depth = 2, heads = 2, qk_rmsnorm = False)), 1).train(), batch, times, noise)
    assert normed.count('attn_fast_params') == 2 and normed.count('attn_fwd_tc') == 2 and normed.count('attn_bwd_tc') == 2
    assert not {'attn_fast_params', 'attn_fwd_tc', 'attn_bwd_tc', 'gemm_qkvg', 'qk_bwd_pack'} & set(plain)
    assert plain.count('gemm_qkvg_rope') == 2 and plain.count('qk_bwd_pack_rope') == 2 and plain.count('attn_fwd') == 2 and plain.count('attn_bwd') == 2
    rename = dict(gemm_qkvg = 'gemm_qkvg_rope', qk_bwd_pack = 'qk_bwd_pack_rope')
    assert plain == [rename.get(n, n) for n in normed if n not in ('attn_fast_params', 'attn_fwd_tc', 'attn_bwd_tc')]


CTOR_SMALL = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0., transformer = dict(dim = 128, depth = 2, heads = 2, qk_rmsnorm = False))


def _small_batch():
    batch = synth.small_batch(4, seed = 3, dim_latent = 32, text_vocab = 64)
    nm = max(sum(torch.is_tensor(p) and p.is_floating_point() for p in s) for s in batch)
    times = torch.rand(4, nm, generator = torch.Generator().manual_seed(1))
    rows = sum(p.shape[0] for s in batch for p in s if torch.is_tensor(p) and p.is_floating_point())
    return batch, times, rows


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


@pytest.mark.parametrize('opt', ['adam', 'adamw', 'fused'])
def test_gammas_get_no_gradient_and_never_change(opt):
    """as in the reference, the unused q / k norm gammas get no gradient (`.grad is None`): torch.optim skips them (AdamW's weight decay included),
    and the engine keeps them out of its flat buffers, so its fused Adam (with clipping and EMA, eager and replayed) cannot touch them either"""
    from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
    batch, times, rows = _small_batch()
    model = build(CTOR_SMALL, 7).train()
    g0 = {n: p.detach().clone() for n, p in gammas(model).items()}
    assert len(g0) == 4 and all(g.abs().min() > 0 for g in g0.values())
    others0 = {n: p.detach().clone() for n, p in model.named_parameters() if n not in g0}
    ema = model.create_ema(0.9)
    if opt == 'fused':
        tr = DataParallelTrainer(model, lr = 1e-3, weight_decay = 0.1, decoupled_weight_decay = True, max_grad_norm = 0.5, ema_decay = 0.9, cuda_graph = True)
    else:
        o = (torch.optim.Adam(model.parameters(), lr = 1e-3, weight_decay = 0.1) if opt == 'adam' else
             torch.optim.AdamW(model.parameters(), lr = 1e-3, weight_decay = 0.1))
    for step in range(5):
        noise = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(500 + step))]
        if opt == 'fused':
            tr.step(batch, times = times, noise = noise)
        else:
            o.zero_grad()
            loss = model(batch, times = times, noise = noise)
            loss.backward()
            assert all(p.grad is None for p in gammas(model).values())
            torch.nn.utils.clip_grad_norm_(model.parameters(), 0.5)
            o.step()
        ema.update()
    torch.cuda.synchronize()
    if opt == 'fused':
        assert any(g.graph is not None for g in tr._graphs.values()), 'the step was never captured'
    for n, p in gammas(model).items():
        assert p.grad is None, n
        assert same_bits(p.detach(), g0[n]), n
    for n, p in gammas(ema.ema_model).items():
        assert same_bits(p.detach().cuda(), g0[n]), n
    assert not model.engine.offs.keys() & g0.keys()
    moved = [n for n, p in model.named_parameters() if n in others0 and p.requires_grad and not torch.equal(p.detach(), others0[n])]
    assert len(moved) > 10
