"""CPU: `Transformer(dim_head = 128)`.  The constructor accepts 64 and 128 (with any head count in [1, 16] at 128) and keeps the reference's
state-dict layout (tests/golden/state_dict_keys_dh128.json, listed from the reference's own state_dicts); the fp32 checker at any head dim
(oracle/dh128_reference.py) reproduces the reference's own outputs (tests/golden/*dh128*.pt, oracle/make_golden_dh128.py) and equals the
existing checker at 64.  The LASER / value-residual fixture is checked on the GPU only (the checker does not restate those variants)."""
import copy
import json
import os

import pytest
import torch

from helpers import load_golden, golden_noise, grad_fingerprint
from transfusion_pytorch_b200 import Transfusion, synth
from oracle.torch_reference import OracleEngine
from oracle.dh128_reference import HeadDimOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 2e-5          # fp32 restatement vs fp32 reference


def two_type_batch():
    return synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)


def build(fx, engine = HeadDimOracleEngine):
    torch.manual_seed(0)
    model = Transfusion(**fx['ctor'])
    synth.fill_parameters_(model, seed = fx['seed'])
    model.eval()
    model._engine = engine(model)
    return model


def tr(**kw):
    return Transfusion(num_text_tokens = 8, transformer = dict(dim = 256, depth = 1, **kw)).transformer


def test_constructor_head_dim_rules():
    for h in range(1, 17):
        t = tr(dim_head = 128, heads = h)
        assert (t.dim_head, t.heads) == (128, h)
    assert tr(dim_head = 128, heads = 16, use_value_residual = True).use_value_residual
    for kw in (dict(dim_head = 128, heads = 17), dict(dim_head = 128, heads = 0), dict(dim_head = 32), dict(dim_head = 96), dict(dim_head = 256)):
        with pytest.raises(NotImplementedError):
            tr(**kw)
    with pytest.raises(NotImplementedError, match = r'dim_head 32 \(the attention kernels take 64 or 128\)'):
        tr(dim_head = 32)
    with pytest.raises(NotImplementedError, match = r'heads 3 \(must be even and in \[2, 32\]\)'):      # the 64-wide rule is unchanged
        tr(heads = 3)
    with pytest.raises(NotImplementedError, match = r'heads 17 at dim_head 128 \(must be in \[1, 16\]\)'):
        tr(dim_head = 128, heads = 17)


def test_state_dict_layout_matches_the_reference():
    listing = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'state_dict_keys_dh128.json')))
    names = ('small_dh128', 'small_dh128_laser_vres', 'small_dh128_noqknorm', 'sampling_dh128', 'text_dh128')
    assert set(listing) == set(names)
    for name in names:
        model = Transfusion(**load_golden(name)['ctor'])
        sd = model.state_dict()
        assert {k: [list(v.shape), str(v.dtype)] for k, v in sd.items()} == listing[name], name
        H = model.transformer.heads
        assert list(sd['transformer.layers.0.1.fn.q_norm.gamma'].shape) == [128] and list(sd['rotary_emb.freqs'].shape) == [64]
        assert list(sd['transformer.layers.0.1.fn.to_qk.0.weight'].shape) == [2 * H * 128, model.transformer.dim]


def test_generic_checker_equals_the_existing_one_at_64():
    fx = load_golden('small_dh128')
    ctor = copy.deepcopy(fx['ctor'])
    ctor['transformer'].update(heads = 4, dim_head = 64)
    batch = two_type_batch()
    losses = []
    for engine in (OracleEngine, HeadDimOracleEngine):
        model = build(dict(fx, ctor = ctor), engine)
        losses.append(model(batch, times = fx['times'], noise = golden_noise(fx, batch, model.dim_latents)).item())
    assert losses[0] == losses[1]


def test_gammas_in_the_fixtures_are_non_zero():
    """a q / k norm over two 64-wide halves would not reproduce the fixtures"""
    for name in ('small_dh128', 'small_dh128_laser_vres', 'small_dh128_noqknorm'):
        model = build(load_golden(name))
        gam = [p for n, p in model.named_parameters() if n.endswith(('q_norm.gamma', 'k_norm.gamma'))]
        assert gam and all(g.abs().min() > 0 for g in gam)


@pytest.mark.parametrize('name', ['small_dh128', 'small_dh128_noqknorm'])
def test_checker_matches_reference_training_step(name):
    fx = load_golden(name)
    model = build(fx)
    batch = two_type_batch()
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = golden_noise(fx, batch, model.dim_latents))
    rb = model._last_batch
    assert rb.modality_positions == fx['modality_positions'] and rb.total_tokens == fx['total_tokens']
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < REL
    assert abs(bd.text.item() - fx['text_loss'].item()) / fx['text_loss'].item() < REL
    assert len(bd.flow) == 2 and all(abs(a.item() - b.item()) / b.item() < REL for a, b in zip(bd.flow, fx['flow_losses']))
    st = model._engine.state
    rows = fx['hidden_rows']
    for l, h in enumerate(fx['hiddens'] + [fx['embed']]):
        ours = st['hiddens'][l] if l < len(fx['hiddens']) else st['embed']
        for b in range(rb.B):
            k = rows < int(rb.seq_lens[b])
            assert torch.allclose(ours[b, rows[k]], h[b, k], atol = 2e-4, rtol = 1e-4), f'hidden {l} sample {b}'
    loss.backward()
    assert sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None) == fx['no_grad']
    fp = grad_fingerprint((n, p.grad) for n, p in model.named_parameters() if p.grad is not None)
    assert set(fp) == set(fx['grads'])
    for k, v in fx['grads'].items():
        ref_n = max(v['stats'][3].item(), 1e-12)
        assert abs(fp[k]['stats'][2].item() - v['stats'][2].item()) / ref_n < 1e-3, k
        assert abs(fp[k]['stats'][3].item() - v['stats'][3].item()) / ref_n < 1e-3, k


def test_checker_generate_text_only():
    fx = load_golden('text_dh128')
    model = build(fx)
    text = synth.text_batch(4, 257, seed = 3)
    loss = model(text)
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < REL
    gen = model.generate_text_only(text[:, :fx['prompt_len']], fx['gen_len'], temperature = 0.)
    assert torch.equal(gen, fx['generated'])


def test_checker_sample_many():
    fx = load_golden('sampling_dh128')
    model = build(fx)
    out = model.sample_many(copy.deepcopy(fx['prompts']), init_modality_noise = fx['noise'], **fx['kw'])
    assert len(out) == len(fx['samples'])
    for s, r in zip(out, fx['samples']):
        assert len(s) == len(r)
        for a, b in zip(s, r):
            if torch.is_tensor(b):
                assert torch.equal(a.cpu(), b)
            else:
                assert a[0] == b[0] and a[1].shape == b[1].shape
                assert torch.allclose(a[1].float().cpu(), b[1], atol = 1e-4, rtol = 1e-3)
