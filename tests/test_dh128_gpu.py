"""GPU: `Transformer(dim_head = 128)` end to end - every dim_head = 128 kernel against float64 at every accepted head count (1-16), the engine's
routing (general running-maximum attention only, no bounded-logit launch; a 64-wide model keeps its launch list), parity of whole training
steps and greedy decoding with the fp32 checker (oracle/dh128_reference.py), and graph replay against eager.

Kernel bounds: bf16 operands are exact in float64; the attention kernels round P and dS to bf16 (relative 2^-8 per term), the GEMM epilogues
add the fp32 accumulation error C_ACC |u| |W|^T (tests/test_block_epilogues_gpu.py) and the bf16 output cast."""
import pytest
import torch

import copy

from helpers import compare_sampling, gen, golden_noise, grad_fingerprint, load_golden, unpack_rows
from transfusion_pytorch_b200 import Transfusion, _lib, synth
from oracle.dh128_reference import HeadDimOracleEngine

pytestmark = pytest.mark.gpu
BF16, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
U8, U24 = 2.0 ** -8, 2.0 ** -24
C_ACC = 1.6e-6
DH = 128
HEADS = list(range(1, 17))
CAP = 50.
N_POS = 4096
LOSS_REL, HID_REL, GRAD_REL = 1e-3, 2e-2, 6e-2
MARGIN_BOUND, LATENT_TOL = 0.1, 5e-2


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


def rel_err(got, ref):
    return ((got.double() - ref).norm() / ref.norm().clamp(min = 1e-30)).item()


# ------------------------------------------------------------------------------------------------ attention
SEQS = (150, 77, 64, 13)           # partial 64-row tiles and a sequence of exactly one tile


def layout(seed):
    """packed sequences with a causal mask and, per sequence longer than 20, one modality span whose tokens all see up to its last token:
    kv_limit jumps there, inside a 64-key tile.  Tile tables as the host builds them: 64-row query tiles that never straddle a sequence
    (keys from the sequence start up to the tile's largest kv_limit), and per 64-key tile every query row of its sequence"""
    g = torch.Generator().manual_seed(seed)
    kv_limit, tq0, tqe, tk0, tke, kq0, kqe = [], [], [], [], [], [], []
    s0 = 0
    for n in SEQS:
        lim = [s0 + i for i in range(n)]
        if n > 20:
            a = int(torch.randint(1, n // 2, (1,), generator = g)); b = min(n - 1, a + 37)
            lim[a:b + 1] = [s0 + b] * (b + 1 - a)
        kv_limit += lim
        for t0 in range(s0, s0 + n, 64):
            t1 = min(t0 + 64, s0 + n)
            tq0.append(t0); tqe.append(t1); tk0.append(s0); tke.append(max(kv_limit[t0 - s0 + s0:t1]) + 1)
        for t0 in range(s0, s0 + n, 64):
            kq0.append(s0); kqe.append(s0 + n)
        s0 += n
    t = lambda a: torch.tensor(a, dtype = I32, device = 'cuda')
    kt0 = [t0 for s, n in zip([0] + list(torch.tensor(SEQS).cumsum(0)[:-1].tolist()), SEQS) for t0 in range(s, s + n, 64)]
    kte = [min(t0 + 64, s + n) for s, n in zip([0] + list(torch.tensor(SEQS).cumsum(0)[:-1].tolist()), SEQS) for t0 in range(s, s + n, 64)]
    return s0, t(kv_limit), [t(a) for a in (tq0, tqe, tk0, tke)], [t(a) for a in (kt0, kte, kq0, kqe)]


def test_layout_has_span_jumps_inside_a_tile():
    M, kv_limit, _, _ = layout(3)
    lim = kv_limit.cpu()
    assert (lim >= torch.arange(M)).all()
    jumps = [int(l) for i, l in enumerate(lim.tolist()) if l > i]
    assert jumps and any((j + 1) % 64 for j in jumps)


def reference_attention(q, k, v, gates, kv_limit, H, scale):
    M = q.shape[0]
    q, k, v = (x.double().reshape(M, H, DH).requires_grad_() for x in (q, k, v))
    s = torch.einsum('ihd,jhd->hij', q, k) * scale
    s = (s / CAP).tanh() * CAP
    vis = torch.arange(M, device = 'cuda')[None, :] <= kv_limit.long()[:, None]
    # keys of other sequences: the packed layout lets a row see only keys of its own sequence
    seq = torch.repeat_interleave(torch.arange(len(SEQS), device = 'cuda'), torch.tensor(SEQS, device = 'cuda'))
    vis = vis & (seq[:, None] == seq[None, :])
    s = s.masked_fill(~vis[None], float('-inf'))
    o = torch.einsum('hij,jhd->ihd', s.softmax(-1), v) * torch.sigmoid(gates.double())[:, :, None]
    return o, (q, k, v)


@pytest.mark.parametrize('H', HEADS)
def test_attention_forward_backward_vs_float64(ops, H):
    M, kv_limit, ft, bt = layout(H)
    g = gen(100 + H)
    HI, scale = H * DH, DH ** -0.5
    q, k, v = (torch.randn(M, HI, device = 'cuda', generator = g).to(BF16) for _ in range(3))
    gates = torch.randn(M, H, device = 'cuda', generator = g)
    o = torch.empty(M, HI, device = 'cuda', dtype = BF16); lse = torch.empty(H, M, device = 'cuda')
    ops.attn_fwd_d128(q, k, v, HI, HI, HI, gates, H, kv_limit, *ft, len(ft[0]), o, HI, lse, M, scale, CAP)
    ref, leaves = reference_attention(q, k, v, gates, kv_limit, H, scale)
    err = (o.double().reshape(M, H, DH) - ref).abs()
    assert (err <= 2 * U8 * ref.abs() + 0.02 * ref.abs().amax(-1, keepdim = True) + 1e-6).all(), err.max().item()
    # backward: dO of the gated output
    dog = torch.randn(M, HI, device = 'cuda', generator = g).to(BF16)
    ref.backward(dog.double().reshape(M, H, DH))
    dop = torch.empty(M, HI, device = 'cuda', dtype = BF16)
    dsum_hm, dsum_mh = torch.empty(H, M, device = 'cuda'), torch.empty(M, H, device = 'cuda')
    dq = torch.full((M, HI), 7., device = 'cuda'); dk = torch.empty(M, HI, device = 'cuda')
    NQ = 3 * HI + 128
    dv_mat = torch.zeros(M, NQ, device = 'cuda', dtype = BF16)
    ops.attn_bwd_prep_d128(dog, o, gates, dop, dsum_hm, dsum_mh, dq, M, H)
    sg = torch.sigmoid(gates.double())
    og = o.double().reshape(M, H, DH)
    assert torch.allclose(dsum_mh.double(), (dog.double().reshape(M, H, DH) * og).sum(-1), rtol = 1e-4, atol = 1e-4)
    assert torch.equal(dsum_hm.t(), dsum_mh)
    assert (dop.double().reshape(M, H, DH) - dog.double().reshape(M, H, DH) * sg[:, :, None]).abs().max() <= U8 * dog.double().abs().max()
    assert (dq == 0).all()
    ops.attn_bwd_d128(q, k, v, dop, HI, HI, HI, HI, lse, dsum_hm, kv_limit, *bt, len(bt[0]), dq, dk, dv_mat[:, 2 * HI:], NQ, M, H, scale, CAP)
    dv = dv_mat[:, 2 * HI:3 * HI]
    for name, got, leaf in (('dq', dq, leaves[0]), ('dk', dk, leaves[1]), ('dv', dv, leaves[2])):
        r = leaf.grad.reshape(M, HI)
        assert rel_err(got, r) < 2e-2, (name, rel_err(got, r))
    assert (dv_mat[:, :2 * HI] == 0).all() and (dv_mat[:, 3 * HI:] == 0).all()


@pytest.mark.parametrize('H', [1, 3, 8, 16])
def test_decode_vs_dense_float64_over_the_slab(ops, H):
    S, cap = 5, 300
    g = gen(300 + H)
    HI, scale = H * DH, DH ** -0.5
    lens = torch.tensor([1, 37, 64, 129, 300], dtype = I32)
    k = torch.randn(S * cap, HI, device = 'cuda', generator = g).to(BF16)
    v = torch.randn(S * cap, HI, device = 'cuda', generator = g).to(BF16)
    q = torch.randn(S, HI, device = 'cuda', generator = g).to(BF16)
    gates = torch.randn(S, H, device = 'cuda', generator = g)
    base = torch.arange(S, dtype = I32) * cap
    kv_limit = (base + lens - 1).cuda(); tq0 = torch.arange(S, dtype = I32, device = 'cuda')
    tk0 = base.cuda(); tke = (base + cap).cuda()
    o = torch.empty(S, HI, device = 'cuda', dtype = BF16)
    ops.attn_decode_d128(q, k, v, HI, HI, HI, gates, H, kv_limit, tq0, tk0, tke, S, o, HI, scale, CAP)
    for s in range(S):
        r = slice(int(base[s]), int(base[s] + lens[s]))
        kk, vv = k[r].double().reshape(-1, H, DH), v[r].double().reshape(-1, H, DH)
        sim = torch.einsum('hd,jhd->hj', q[s].double().reshape(H, DH), kk) * scale
        p = ((sim / CAP).tanh() * CAP).softmax(-1)
        ref = torch.einsum('hj,jhd->hd', p, vv) * torch.sigmoid(gates[s].double())[:, None]
        err = (o[s].double().reshape(H, DH) - ref).abs()
        assert (err <= U8 * ref.abs() + 1e-4 * vv.abs().amax(0) + 1e-6).all(), (s, err.max().item())


# ------------------------------------------------------------------------------------------------ QKVG epilogue + backward packs
def rope_tables(ops):
    freqs = 1. / (10000 ** (torch.arange(0, DH, 2, device = 'cuda').float() / DH))
    t = torch.empty(N_POS, DH // 2, 2, device = 'cuda'); tt = torch.empty(DH // 2, N_POS, 2, device = 'cuda')
    ops.rope_table(freqs, t, tt, N_POS, DH // 2)
    return t, tt


def rope(y, cs):
    c, s = cs[..., 0], cs[..., 1]
    y0, y1 = y[..., 0::2], y[..., 1::2]
    return torch.stack((y0 * c - y1 * s, y1 * c + y0 * s), -1).flatten(-2)


@pytest.mark.parametrize('H', HEADS)
@pytest.mark.parametrize('normed', [True, False])
def test_qkvg_and_qk_backward_pack_vs_float64(ops, H, normed):
    M, D = 1111, (128, 256, 512, 1024)[H % 4]
    g = gen(700 + H)
    HI, NQ = H * DH, 3 * H * DH + 128
    u = torch.randn(M, D, device = 'cuda', generator = g).to(BF16)
    W = (torch.randn(NQ, D, device = 'cuda', generator = g) / D ** 0.5).to(BF16)
    gq, gk = (torch.rand(DH, device = 'cuda', generator = g) * 1.9 - 0.9 for _ in range(2))
    pos = torch.randint(0, N_POS, (M,), device = 'cuda', generator = g, dtype = I32)
    t, tt = rope_tables(ops)
    q, k, v = (torch.empty(M, HI, device = 'cuda', dtype = BF16) for _ in range(3))
    gates = torch.empty(M, H, device = 'cuda'); inv = torch.empty(M, 2 * H, device = 'cuda'); mix = torch.empty(M, H, device = 'cuda')
    if normed:
        ops.gemm_qkvg_d128(u, D, W, D, M, H, D, q, k, v, gates, inv, gq, gk, pos, tt, N_POS, None, mix)
    else:
        ops.gemm_qkvg_rope_d128(u, D, W, D, M, H, D, q, k, v, gates, pos, tt, N_POS, None, mix)
    y = u.double() @ W.double().t()
    mag = u.double().abs() @ W.double().abs().t()
    cs = t[pos.long()].double()[:, None]                                # [M, 1, 64, 2]
    leaves = []
    for which, (name, got, gam) in enumerate((('q', q, gq), ('k', k, gk))):
        ys = y[:, which * HI:(which + 1) * HI].reshape(M, H, DH).clone().requires_grad_()
        x = torch.nn.functional.normalize(ys, dim = -1) * DH ** 0.5 * (gam.double() + 1.) if normed else ys
        ref = rope(x, cs)
        ms = mag[:, which * HI:(which + 1) * HI].reshape(M, H, DH)
        scl = (DH ** 0.5 * (gam.double() + 1.).abs() / ys.detach().norm(dim = -1, keepdim = True)) if normed else 1.
        bound = U8 * ref.detach().abs() + 2 * (scl * (C_ACC * ms + 4 * U24 * ys.detach().abs())).amax(-1, keepdim = True) + 1e-6
        assert ((got.double().reshape(M, H, DH) - ref.detach()).abs() <= bound).all(), name
        leaves.append((ys, ref))
        if normed:
            assert torch.allclose(inv[:, which * H:(which + 1) * H].double(), 1. / ys.detach().norm(dim = -1), rtol = 1e-4)
    assert torch.allclose(v.double(), y[:, 2 * HI:3 * HI], rtol = U8, atol = 4 * C_ACC * mag[:, 2 * HI:3 * HI].max().item())
    assert torch.allclose(gates.double(), y[:, 3 * HI:3 * HI + H], rtol = 1e-5, atol = 2 * C_ACC * mag.max().item())
    m0 = 3 * HI + (H + 1) // 2 * 2                                       # the mix rows start at an even row
    assert torch.allclose(mix.double(), y[:, m0:m0 + H], rtol = 1e-5, atol = 2 * C_ACC * mag.max().item())
    # backward pack: dq, dk (fp32) -> d[q_pre | k_pre | . | gates] (bf16) and the gamma gradients
    dq, dk = (torch.randn(M, HI, device = 'cuda', generator = g) for _ in range(2))
    dsum = torch.randn(M, H, device = 'cuda', generator = g)
    out = torch.zeros(M, NQ, device = 'cuda', dtype = BF16)
    dgq, dgk = torch.zeros(DH, device = 'cuda'), torch.zeros(DH, device = 'cuda')
    if normed:
        ops.qk_bwd_pack_d128(dq, dk, q, k, inv, gq, gk, pos, t, gates, dsum, out, NQ, dgq, dgk, M, H)
    else:
        ops.qk_bwd_pack_rope_d128(dq, dk, pos, t, gates, dsum, out, NQ, M, H)
    gl = [gq, gk]
    if normed:
        gl = [gq.double().requires_grad_(), gk.double().requires_grad_()]
        leaves = []
        for which in range(2):
            ys = y[:, which * HI:(which + 1) * HI].reshape(M, H, DH).clone().requires_grad_()
            leaves.append((ys, rope(torch.nn.functional.normalize(ys, dim = -1) * DH ** 0.5 * (gl[which] + 1.), cs)))
    for which, (ys, ref) in enumerate(leaves):
        ref.backward((dq, dk)[which].double().reshape(M, H, DH))
        r = ys.grad.reshape(M, HI)
        assert rel_err(out[:, which * HI:(which + 1) * HI], r) < 2e-2, (which, rel_err(out[:, which * HI:(which + 1) * HI], r))
    if normed:
        for which, got in enumerate((dgq, dgk)):
            assert rel_err(got, gl[which].grad) < 2e-2, which
    dg = (1 - torch.sigmoid(gates.double())) * dsum.double()
    assert torch.allclose(out[:, 3 * HI:3 * HI + H].double(), dg, rtol = 2 * U8, atol = 1e-6)
    assert (out[:, 2 * HI:3 * HI] == 0).all() and (out[:, 3 * HI + H:] == 0).all()


# ------------------------------------------------------------------------------------------------ LASER / value-residual row kernels
@pytest.mark.parametrize('H', HEADS)
def test_laser_and_vmix_row_kernels_vs_float64(ops, H):
    M = 333
    g = gen(900 + H)
    HI = H * DH
    gates = torch.randn(M, H, device = 'cuda', generator = g)
    sg = torch.sigmoid(gates.double())[:, :, None]
    o = (torch.rand(M, HI, device = 'cuda', generator = g) * 3 + 0.01).to(BF16)
    att = torch.empty(M, HI, device = 'cuda', dtype = BF16)
    ops.laser_out_fwd_d128(o, gates, att, M, H)
    ref = o.double().log().reshape(M, H, DH) * sg
    assert ((att.double().reshape(M, H, DH) - ref).abs() <= U8 * ref.abs() + 1e-5).all()
    datt = torch.randn(M, HI, device = 'cuda', generator = g).to(BF16)
    dop = torch.empty(M, HI, device = 'cuda', dtype = BF16)
    dsum_hm, dsum_mh = torch.empty(H, M, device = 'cuda'), torch.empty(M, H, device = 'cuda')
    dq = torch.full((M, HI), 3., device = 'cuda')
    ops.laser_bwd_prep_d128(datt, o, gates, dop, dsum_hm, dsum_mh, dq, M, H)
    a, oo = datt.double().reshape(M, H, DH), o.double().reshape(M, H, DH)
    assert ((dop.double().reshape(M, H, DH) - a * sg / oo).abs() <= U8 * (a * sg / oo).abs() + 1e-6).all()
    assert torch.allclose(dsum_hm.t().double(), (a * sg).sum(-1), rtol = 1e-4, atol = 1e-4)
    assert torch.allclose(dsum_mh.double(), (a * oo.log() * sg).sum(-1), rtol = 1e-3, atol = 1e-3)
    assert (dq == 0).all()
    # value residual
    v, v0 = (torch.randn(M, HI, device = 'cuda', generator = g).to(BF16) for _ in range(2))
    mixpre, bias = torch.randn(M, H, device = 'cuda', generator = g), torch.randn(H, device = 'cuda', generator = g)
    mx = torch.sigmoid(mixpre.double() + bias.double())[:, :, None]
    vm = v.clone()
    ops.vmix_fwd_d128(vm, HI, None, v0, HI, mixpre, bias, M, H)
    ref = v.double().reshape(M, H, DH) * mx + v0.double().reshape(M, H, DH) * (1 - mx)
    assert ((vm.double().reshape(M, H, DH) - ref).abs() <= U8 * ref.abs() + 1e-6).all()
    dvm = torch.randn(M, HI, device = 'cuda', generator = g).to(BF16)
    dv = dvm.clone(); acc = torch.ones(M, HI, device = 'cuda'); dmix = torch.zeros(M, 32, device = 'cuda', dtype = BF16)
    ops.vmix_bwd_d128(dv, HI, vm, HI, v0, HI, mixpre, bias, acc, dmix, 32, M, H)
    gd = dvm.double().reshape(M, H, DH)
    assert ((dv.double().reshape(M, H, DH) - gd * mx).abs() <= U8 * (gd * mx).abs() + 1e-6).all()
    assert torch.allclose(acc.double().reshape(M, H, DH), 1 + gd * (1 - mx), rtol = 1e-5, atol = 1e-5)
    ref_dm = (gd * (vm.double().reshape(M, H, DH) - v0.double().reshape(M, H, DH))).sum(-1) * (1 - mx[..., 0])
    assert torch.allclose(dmix[:, :H].double(), ref_dm, rtol = 2 * U8, atol = 1e-3)
    assert (dmix[:, H:] == 0).all()


# ------------------------------------------------------------------------------------------------ whole model
def build(ctor, seed, dev = 'cuda'):
    torch.manual_seed(0)
    model = Transfusion(**ctor)
    synth.fill_parameters_(model, seed = seed)
    model = model.to(dev).eval()
    if dev == 'cpu':
        model._engine = HeadDimOracleEngine(model)
    return model


def small_inputs(B = 3, seed = 1):
    batch = synth.small_batch(B, seed = seed, dim_latent = 32, text_vocab = 64)
    nm = max(sum(torch.is_tensor(p) and p.is_floating_point() for p in s) for s in batch)
    times = torch.rand(B, nm, generator = torch.Generator().manual_seed(5))
    rows = sum(p.shape[0] for s in batch for p in s if torch.is_tensor(p) and p.is_floating_point())
    noise = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(4))]
    return batch, times, noise


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


@pytest.mark.parametrize('name', ['small_dh128', 'small_dh128_laser_vres', 'small_dh128_noqknorm'])
def test_train_step_matches_reference(name):
    """the reference's own outputs (oracle/make_golden_dh128.py): loss, breakdown, hidden states, gradient fingerprints"""
    fx = load_golden(name)
    model = build(fx['ctor'], fx['seed'])
    batch = synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = golden_noise(fx, batch, model.dim_latents))
    rb = model._last_batch
    assert rb.modality_positions == fx['modality_positions'] and rb.total_tokens == fx['total_tokens']
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < LOSS_REL
    assert abs(bd.text.item() - fx['text_loss'].item()) / fx['text_loss'].item() < LOSS_REL
    assert all(abs(a.item() - b.item()) / b.item() < LOSS_REL for a, b in zip(bd.flow, fx['flow_losses']))
    st = model.engine.state
    rows = fx['hidden_rows']
    for l, h in enumerate(fx['hiddens'] + [fx['embed']]):
        ours = unpack_rows(st['hid'][l] if l < len(fx['hiddens']) else st['out'], rb)
        for b in range(rb.B):
            k = rows < int(rb.seq_lens[b])
            assert rel_max(ours[b, rows[k]], h[b, k]) < HID_REL, f'hidden {l} sample {b}'
    loss.backward()
    assert sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None) == fx['no_grad']
    check_grads(model, fx)


def test_text_only_loss_grads_and_greedy_tokens_match_reference():
    fx = load_golden('text_dh128')
    model = build(fx['ctor'], fx['seed'])
    text = synth.text_batch(4, 257, seed = 3)
    loss = model(text)
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < LOSS_REL
    loss.backward()
    check_grads(model, fx)
    gen_ = model.generate_text_only(text[:, :fx['prompt_len']], fx['gen_len'], temperature = 0.).cpu()
    ref, margins = fx['generated'], fx['margins']
    assert gen_.shape == ref.shape
    for b in range(gen_.shape[0]):
        neq = (gen_[b] != ref[b]).nonzero()
        if neq.numel():
            k = int(neq[0])
            assert margins[b, k].item() < MARGIN_BOUND, f'row {b}: token {k} differs although the reference margin is {margins[b, k].item():.4f}'


def test_sample_many_matches_reference():
    fx = load_golden('sampling_dh128')
    model = build(fx['ctor'], fx['seed'])
    out = model.sample_many(copy.deepcopy(fx['prompts']), init_modality_noise = fx['noise'], **fx['kw'])
    rep = compare_sampling(model, out, fx, bound = MARGIN_BOUND, lat_tol = LATENT_TOL)
    assert len(rep) == len(fx['samples']) and all(len(r['latent_err']) >= 1 for r in rep)


def ctor_small(**tr):
    return dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0., transformer = dict(dim = 256, depth = 4, **tr))


@pytest.mark.parametrize('tr', [dict(heads = 2, dim_head = 128), dict(heads = 3, dim_head = 128), dict(heads = 1, dim_head = 128, qk_rmsnorm = False)],
                         ids = ['h2', 'h3_odd', 'h1_noqknorm'])
def test_training_step_matches_checker(tr):
    batch, times, noise = small_inputs()
    out = {}
    for dev in ('cuda', 'cpu'):
        model = build(ctor_small(**tr), 3, dev)
        loss, bd = model(batch, times = times, noise = noise, return_breakdown = True)
        loss.backward()
        grads = {n: p.grad.detach().float().cpu().clone() for n, p in model.named_parameters() if p.grad is not None}
        out[dev] = (loss.item(), bd.text.item(), grads)
    (lc, tc, gc), (lo, to_, go) = out['cuda'], out['cpu']
    assert abs(lc - lo) / abs(lo) < LOSS_REL and abs(tc - to_) / abs(to_) < LOSS_REL, (lc, lo, tc, to_)
    assert set(gc) == set(go)
    for n in gc:
        if any(s in n for s in ('to_qk', 'to_v', 'to_out', 'to_gates', 'q_norm', 'k_norm', 'net.0.weight', 'text_embed')):
            assert (gc[n] - go[n]).norm() / go[n].norm().clamp(min = 1e-12) < GRAD_REL, n


def test_greedy_text_matches_checker():
    ctor = dict(num_text_tokens = 64, transformer = dict(dim = 256, depth = 2, heads = 2, dim_head = 128))
    prompt = torch.randint(0, 64, (3, 6), generator = torch.Generator().manual_seed(3))
    toks = {}
    for dev in ('cuda', 'cpu'):
        model = build(ctor, 5, dev)
        toks[dev] = model.generate_text_only(prompt.to(dev), 20, temperature = 0.).cpu()
    assert toks['cuda'].shape == toks['cpu'].shape
    assert (toks['cuda'] == toks['cpu']).float().mean().item() >= 0.9


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


def test_launch_lists():
    batch, times, noise = small_inputs()
    d128 = _launches(build(ctor_small(heads = 2, dim_head = 128), 1).train(), batch, times, noise)
    d64 = _launches(build(ctor_small(heads = 4), 1).train(), batch, times, noise)
    assert not {'attn_fast_params', 'attn_fwd_tc', 'attn_bwd_tc', 'attn_fwd', 'attn_bwd', 'gemm_qkvg', 'qk_bwd_pack', 'attn_bwd_prep'} & set(d128)
    assert d128.count('attn_fwd_d128') == 4 and d128.count('attn_bwd_d128') == 4 and d128.count('gemm_qkvg_d128') == 4
    assert d64.count('attn_fwd_tc') == 4 and not [n for n in d64 if n.endswith('_d128')]
    assert d128 == [n + '_d128' if n in ('gemm_qkvg', 'attn_fwd', 'attn_bwd', 'attn_bwd_prep', 'qk_bwd_pack') else n
                    for n in d64 if n not in ('attn_fast_params', 'attn_fwd_tc', 'attn_bwd_tc')]


def test_graph_replay_follows_eager_trajectory():
    from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
    batch, times, noise = small_inputs(4, seed = 3)
    rows = noise[0].shape[0]
    results = []
    for use_graph in (False, True):
        model = build(ctor_small(heads = 3, dim_head = 128, attn_laser = True, use_value_residual = True), 7).train()
        tr = DataParallelTrainer(model, lr = 1e-3, cuda_graph = use_graph)
        losses = []
        for step in range(6):
            nz = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(500 + step))]
            losses.append(tr.step(batch, times = times, noise = nz).item())
        results.append((losses, model.engine.flat.clone()))
        if use_graph:
            assert any(g.graph is not None for g in tr._graphs.values()), 'the step was never captured'
    (l0, p0), (l1, p1) = results
    assert all(abs(a - b) / abs(a) < 2e-3 for a, b in zip(l0, l1)), (l0, l1)
    assert (p1 - p0).abs().max().item() < 2e-3 * p0.abs().max().item() + 2e-4
