"""GPU (H100): FFN dropout - the GEGLU GEMM epilogue and the GEGLU backward with the counter-based mask of csrc/dropout.cuh, read back
bit for bit against the restatement (oracle/dropout_mask.py); the training step against the reference fixture (tests/golden/small_dropout.pt)
and the CPU checker; inactive dropout launching exactly the kernels of a model without dropout; CUDA-graph replays; mask statistics."""
import numpy as np
import pytest
import torch

from helpers import load_golden, grad_fingerprint, unpack_rows
from transfusion_pytorch_b200 import Transfusion, _lib, synth
from oracle.dropout_mask import DropoutOracleEngine, keep_mask, scale, SITE_FFN

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
LOSS_REL, HID_REL, GRAD_REL = 1e-3, 2e-2, 6e-2          # tests/test_parity_gpu.py


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


def dev_key(k0, k1):
    return torch.from_numpy(np.array([k0, k1], dtype = np.uint32).view(np.int32)).cuda()


def ffn_keep(key, p, layer, M, cols):
    return torch.from_numpy(keep_mask(key, p, SITE_FFN, layer, 0, np.arange(M), np.arange(cols))).cuda()


def geglu_inputs(M, D = 512, inner = 1365, seed = 13):
    """packed W1 / bias as the engine lays them out (tile t = [64 value | 64 gate] columns), as in tests/test_block_epilogues_gpu.py"""
    g = torch.Generator(device = 'cuda').manual_seed(seed)
    Ip = (inner + 63) // 64 * 64
    W1 = torch.randn(2 * inner, D, device = 'cuda', generator = g) / D ** 0.5
    b1 = torch.randn(2 * inner, device = 'cuda', generator = g) * 0.3
    u = torch.randn(M, D, device = 'cuda', generator = g).to(BF16)
    Wp = torch.zeros(2 * Ip, D, device = 'cuda'); bp = torch.zeros(2 * Ip, device = 'cuda')
    col = torch.arange(Ip, device = 'cuda')
    valid = col < inner
    tile, j = col // 64, col % 64
    Wp[(tile * 128 + j)[valid]] = W1[col[valid]]; Wp[(tile * 128 + 64 + j)[valid]] = W1[inner + col[valid]]
    bp[(tile * 128 + j)[valid]] = b1[col[valid]]; bp[(tile * 128 + 64 + j)[valid]] = b1[inner + col[valid]]
    return u, Wp.to(BF16), bp, W1, b1, Ip


def test_geglu_epilogue_dropout(ops):
    """every CTA takes several ping-pong work items (40 x 22 tiles); p = 0.5 scales by exactly 2, so h is bit-identical to the undropped h
    times 2 x mask; other p against float64 GEGLU x mask; vg is never dropped"""
    M, D, inner = 5000, 512, 1365
    u, Wp, bp, W1, b1, Ip = geglu_inputs(M, D, inner)
    vg0 = torch.zeros(M, 2 * Ip, device = 'cuda', dtype = BF16); h0 = torch.zeros(M, Ip, device = 'cuda', dtype = BF16)
    ops.gemm_geglu(u, D, Wp, D, bp, M, 2 * Ip, D, vg0, h0)
    pre = u.double() @ W1.to(BF16).double().t() + b1.double()
    ref = torch.nn.functional.gelu(pre[:, inner:]) * pre[:, :inner]
    key = (0x9E3779B9, 0x00C0FFEE)
    for p, layer in ((0.5, 3), (0.1, 0), (0.2, 7), (1.0, 1)):
        vg = torch.full_like(vg0, 7.); h = torch.full_like(h0, 7.)
        ops.gemm_geglu_drop(u, D, Wp, D, bp, M, 2 * Ip, D, vg, h, dev_key(*key), p, layer)
        keep = ffn_keep(key, p, layer, M, Ip)
        torch.cuda.synchronize()
        assert torch.equal(vg, vg0), p
        assert torch.equal(h == 0, (~keep) | (h0 == 0)), p                   # dropped exactly where the restated mask drops
        if p == 0.5:
            assert torch.equal(h, torch.where(keep, h0 * 2, torch.zeros_like(h0)))
        want = ref * keep[:, :inner].double() * scale(p)
        assert torch.allclose(h[:, :inner].double(), want, atol = 6e-2 * max(scale(p), 1.), rtol = 3e-2), p
        assert (h[:, inner:] == 0).all()
        if p < 1.:                                                           # the mask is not trivially all-kept / all-dropped
            frac = keep[:, :inner].float().mean().item()
            assert abs(frac - (1 - p)) < 5 * (p * (1 - p) / (M * inner)) ** 0.5, (p, frac)


def test_geglu_bwd_dropout(ops):
    """geglu_bwd_drop(dh) = geglu_bwd(dh x mask / (1 - p)): bit for bit at p = 0.5 (scale 2 is exact in bf16), against float64 autograd otherwise;
    bias-gradient partials included"""
    M, inner = 3001, 1365
    Ip = (inner + 63) // 64 * 64
    g = torch.Generator(device = 'cuda').manual_seed(5)
    vg = (torch.randn(M, 2 * Ip, device = 'cuda', generator = g) * 1.5).to(BF16)
    dh = torch.randn(M, Ip, device = 'cuda', generator = g).to(BF16)
    rpb = ops.lib.tfx_geglu_bwd_rows_per_block()
    nblk = (M + rpb - 1) // rpb
    key = (0x01234567, 0x89ABCDEF)
    v = vg.double().reshape(M, Ip // 64, 2, 64)[:, :, 0].reshape(M, Ip)
    gt = vg.double().reshape(M, Ip // 64, 2, 64)[:, :, 1].reshape(M, Ip)
    for p, layer in ((0.5, 2), (0.1, 0), (1.0, 5)):
        keep = ffn_keep(key, p, layer, M, Ip)
        dvg, part = torch.zeros_like(vg), torch.zeros(nblk, 2 * Ip, device = 'cuda')
        ops.geglu_bwd_drop(dh, vg, dvg, M, Ip, None, None, part, dev_key(*key), p, layer)
        if p == 0.5:
            dvg0, part0 = torch.zeros_like(vg), torch.zeros_like(part)
            ops.geglu_bwd(torch.where(keep, dh * 2, torch.zeros_like(dh)), vg, dvg0, M, Ip, None, None, part0)
            torch.cuda.synchronize()
            assert torch.equal(dvg, dvg0) and torch.equal(part, part0)
        vv, gg = v.clone().requires_grad_(), gt.clone().requires_grad_()
        (torch.nn.functional.gelu(gg) * vv * keep.double() * scale(p) * dh.double()).sum().backward()
        got = dvg.double().reshape(M, Ip // 64, 2, 64)
        tol = lambda ref: 1e-2 * ref.abs().max().item() + 1e-6
        assert (got[:, :, 0].reshape(M, Ip) - vv.grad).abs().max().item() <= tol(vv.grad), p
        assert (got[:, :, 1].reshape(M, Ip) - gg.grad).abs().max().item() <= tol(gg.grad), p
        assert torch.equal(got[:, :, 0].reshape(M, Ip) == 0, (vv.grad == 0) | (got[:, :, 0].reshape(M, Ip) == 0)), p
        if p == 1.0:
            assert (dvg == 0).all() and (part == 0).all()


def _model(ctor, seed):
    torch.manual_seed(0)
    model = Transfusion(**ctor).cuda()
    synth.fill_parameters_(model, seed = seed)
    return model


def test_train_step_with_dropout_matches_reference():
    """the reference with nn.Dropout replaced by the restated mask for the fixture's key (oracle/make_golden_dropout.py)"""
    fx = load_golden('small_dropout')
    model = _model(fx['ctor'], fx['seed']).train()
    batch = synth.dropout_batch()
    noise = [torch.randn(rows, dl, generator = torch.Generator().manual_seed(9000 + k + 17 * fx['seed'])) for k, (rows, dl) in enumerate(fx['noise_shapes'])]
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = noise, prob_uncond = 0., dropout_key = fx['dropout_key'])
    rb = model._last_batch
    assert rb.modality_positions == fx['modality_positions']
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < LOSS_REL
    assert abs(bd.text.item() - fx['text_loss'].item()) / fx['text_loss'].item() < LOSS_REL
    for a, b in zip(bd.flow, fx['flow_losses']):
        assert abs(a.item() - b.item()) / b.item() < LOSS_REL
    for l, h in enumerate(fx['hiddens']):
        ours = unpack_rows(model.engine.state['hid'][l], rb).float().cpu()
        for b in range(rb.B):
            n = int(rb.seq_lens[b])
            assert ((ours[b, :n] - h[b, :n]).abs().max() / h[b, :n].abs().max()).item() < HID_REL, f'hidden {l} sample {b}'
    loss.backward()
    fp = grad_fingerprint((n, p.grad) for n, p in model.named_parameters() if p.grad is not None)
    for k, v in fx['grads'].items():
        ref_n = max(v['stats'][3].item(), 1e-12)
        assert abs(fp[k]['stats'][2].item() - v['stats'][2].item()) / ref_n < GRAD_REL, k
        assert abs(fp[k]['stats'][3].item() - v['stats'][3].item()) / ref_n < GRAD_REL, k


def test_config2_train_step_with_dropout_matches_the_checker():
    ctor = dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), prob_uncond = 0.,
                transformer = dict(dim = 512, depth = 8, ff_kwargs = dict(dropout = 0.1)))
    batch, times = synth.config2_batch(2, seed = 4), synth.config2_times(2, seed = 4)
    noise = [torch.randn(1024, 384, generator = torch.Generator().manual_seed(3))]
    key = (0xDEADBEEF, 12345)
    model = _model(ctor, 4).train()
    got = model(batch, times = times, noise = noise, dropout_key = key).item()
    torch.manual_seed(0)
    ref = Transfusion(**ctor)
    synth.fill_parameters_(ref, seed = 4)
    ref.train()
    ref._engine = DropoutOracleEngine(ref)
    with torch.no_grad():
        want = ref(batch, times = times, noise = noise, dropout_key = key).item()
    assert abs(got - want) / abs(want) < LOSS_REL, (got, want)


def _launches(model, batch, times, noise, **kw):
    """entry points in launch order and their non-pointer arguments (tensors by shape / dtype) of one train step"""
    eng = model.engine
    eng.ensure_attached()
    eng.ops.timing, eng.ops.order = {}, []
    loss = model(batch, times = times, noise = noise, **kw)
    loss.backward()
    torch.cuda.synchronize()
    order, timing = eng.ops.order, eng.ops.timing
    eng.ops.timing = eng.ops.order = None
    def norm(a):
        if torch.is_tensor(a):
            return ('tensor', tuple(a.shape), a.dtype)
        return a if isinstance(a, (int, float, str, type(None))) else type(a).__name__
    return order, {n: [tuple(norm(a) for a in args) for (_, _, args) in calls] for n, calls in timing.items()}


def test_inactive_dropout_launches_the_kernels_of_a_model_without_dropout():
    base = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0.)
    tr = lambda **kw: dict(dim = 128, depth = 2, heads = 2, **kw)
    batch = synth.dropout_batch()
    times = torch.rand(3, 2, generator = torch.Generator().manual_seed(5))
    noise = [torch.randn(52, 32, generator = torch.Generator().manual_seed(1))]
    want = _launches(_model(dict(base, transformer = tr()), 1).train(), batch, times, noise)
    cases = [('eval', _model(dict(base, transformer = tr(ff_kwargs = dict(dropout = 0.1))), 1).eval()),
             ('p = 0', _model(dict(base, transformer = tr(ff_kwargs = dict(dropout = 0.))), 1).train()),
             ('flex', _model(dict(base, transformer = tr(dropout = 0.1, use_flex_attn = True)), 1).train())]
    for name, model in cases:
        assert _launches(model, batch, times, noise) == want, name
    order, _ = _launches(_model(dict(base, transformer = tr(ff_kwargs = dict(dropout = 0.1))), 1).train(), batch, times, noise, dropout_key = (1, 2))
    assert order.count('gemm_geglu_drop') == 2 and order.count('geglu_bwd_drop') == 2 and 'gemm_geglu' not in order
    assert [n.replace('_drop', '') for n in order] == want[0]


def test_graph_replay_with_dropout_follows_eager_and_draws_a_key_per_replay():
    from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
    from transfusion_pytorch_b200.modality_processing import pack_batch
    ctor = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0.,
                transformer = dict(dim = 128, depth = 2, heads = 2, ff_kwargs = dict(dropout = 0.3)))
    batch = synth.dropout_batch()
    times = torch.rand(3, 2, generator = torch.Generator().manual_seed(5))
    results = []
    for use_graph in (False, True):
        model = _model(ctor, 7).train()
        trn = DataParallelTrainer(model, lr = 1e-3, cuda_graph = use_graph)
        eng = model.engine
        eng.ensure_attached()
        samples = [[torch.tensor([model.sos_id]), *s, torch.tensor([model.eos_id])] for s in batch]
        rb = pack_batch(samples, times, model, return_loss = True, return_embed = False)
        lat = model._latents_to_device(rb)
        eng.upload(rb)
        losses = []
        for step in range(6):
            noise = [torch.randn(52, 32, generator = torch.Generator().manual_seed(500 + step)).cuda()]
            losses.append(trn.step_packed(rb, lat, noise = noise, dropout_key = (1000 + step, 77)).item())
        results.append((losses, eng.flat.clone()))
        if use_graph:
            graphs = [g for g in trn._graphs.values() if g.graph is not None]
            assert len(graphs) == 1, 'the step was never captured'
            assert graphs[0].drop_key.cpu().numpy().view(np.uint32).tolist() == [1005, 77]
            keys = []
            for _ in range(2):                                   # no fixed key: one drawn per replay
                trn.step_packed(rb, lat, noise = noise)
                keys.append(graphs[0].drop_key.cpu().tolist())
            assert keys[0] != keys[1]
    (l0, p0), (l1, p1) = results
    assert all(abs(a - b) / abs(a) < 2e-3 for a, b in zip(l0, l1)), (l0, l1)
    assert (p1 - p0).abs().max().item() < 2e-3 * p0.abs().max().item() + 2e-4


def test_mask_statistics_and_seeding(ops):
    """config-2 FFN at b = 128 (131,072 rows x 1,365 columns): per layer the kept fraction is within 5 sigma of 1 - p; masks of different layers
    and of consecutive forwards' keys are uncorrelated (|corr| within 5 sigma of 0); torch.manual_seed reproduces the drawn key"""
    model = _model(dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), transformer = dict(dim = 512, depth = 2,
                                                                                                                         ff_kwargs = dict(dropout = 0.1))), 4)
    eng = model.engine
    eng.ensure_attached()
    torch.manual_seed(123); k1 = eng.dropout_key().clone()
    k2 = eng.dropout_key().clone()
    torch.manual_seed(123); k1b = eng.dropout_key().clone()
    assert torch.equal(k1, k1b) and not torch.equal(k1, k2)
    M, D, inner, p = 131072, 512, 1365, 0.1
    Ip = (inner + 63) // 64 * 64
    # u = 0, bias only: value 1, gate 3 on every column, so h = gelu(3) != 0 wherever it is kept
    u = torch.zeros(M, D, device = 'cuda', dtype = BF16)
    W = torch.zeros(2 * Ip, D, device = 'cuda', dtype = BF16)
    b = torch.tensor([1.] * 64 + [3.] * 64, device = 'cuda').repeat(Ip // 64)
    vg = torch.empty(M, 2 * Ip, device = 'cuda', dtype = BF16); h = torch.empty(M, Ip, device = 'cuda', dtype = BF16)
    masks = {}
    for name, key, layer in (('k1 l0', k1, 0), ('k1 l1', k1, 1), ('k2 l0', k2, 0)):
        ops.gemm_geglu_drop(u, D, W, D, b, M, 2 * Ip, D, vg, h, key, p, layer)
        masks[name] = (h[:, :inner] != 0).float().reshape(-1)
    n = M * inner
    for name, m in masks.items():
        assert abs(m.mean().item() - (1 - p)) < 5 * (p * (1 - p) / n) ** 0.5, name
    names = list(masks)
    for i in range(len(names)):
        for j in range(i + 1, len(names)):
            a, c = masks[names[i]], masks[names[j]]
            corr = (((a - a.mean()) * (c - c.mean())).mean() / (a.std() * c.std())).item()
            assert abs(corr) < 5 / n ** 0.5, (names[i], names[j], corr)
    # neighbouring rows and columns of one mask are uncorrelated too (Philox counters differ in one word)
    m = masks['k1 l0'].reshape(M, inner)
    for a, c in ((m[:-1], m[1:]), (m[:, :-1], m[:, 1:])):
        a, c = a.reshape(-1), c.reshape(-1)
        corr = (((a - a.mean()) * (c - c.mean())).mean() / (a.std() * c.std())).item()
        assert abs(corr) < 5 / a.numel() ** 0.5, corr
