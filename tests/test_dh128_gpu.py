"""GPU: `Transformer(dim_head = 128)` end to end - the engine's routing (general running-maximum attention only, no bounded-logit launch; a
64-wide model keeps its launch list), parity of whole training steps and greedy decoding with the reference's own outputs and the fp32
checker (oracle/dh128_reference.py), and graph replay against eager.  Every dim_head = 128 kernel is tested against float64 in
tests/test_dh128_kernels_gpu.py."""
import pytest
import torch

import copy

from helpers import compare_sampling, golden_noise, grad_fingerprint, load_golden, unpack_rows
from transfusion_pytorch_b200 import Transfusion, synth
from oracle.dh128_reference import HeadDimOracleEngine

pytestmark = pytest.mark.gpu
LOSS_REL, HID_REL, GRAD_REL = 1e-3, 2e-2, 6e-2
MARGIN_BOUND, LATENT_TOL = 0.1, 5e-2


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
