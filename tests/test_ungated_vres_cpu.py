"""CPU: ungated attention (`attn_kwargs = dict(gate_values = False)`, T.py:901-904, 1026-1027) and the learned value residual at every accepted head
count.  The constructor accepts both and keeps the reference's state-dict layout (tests/golden/state_dict_keys_ungated.json, written by
oracle/make_golden_ungated.py from the reference itself); the engine's packed QKVG layout has a gate tile iff the model is gated or has the
value residual; the fp32 checker of oracle/ungated_reference.py reproduces the reference's own outputs for ungated models (tests/golden/*ungated*.pt).  The LASER / value-residual
fixtures (small_ungated_laser_vres, small_vres_h32, small_wide1536_vres) are checked on the GPU only: the checkers do not restate those variants."""
import copy
import json
import os

import numpy as np
import pytest
import torch

from helpers import load_golden, golden_noise, grad_fingerprint
from transfusion_pytorch_b200 import Transfusion, synth
from transfusion_pytorch_b200.engine import Engine, _round_up
from transfusion_pytorch_b200.transfusion import Transformer
from oracle.ungated_reference import UngatedOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 2e-5          # fp32 restatement vs fp32 reference
LISTING = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'state_dict_keys_ungated.json')))


def two_type_batch():
    return synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)


def listed_ctor(name):
    from oracle.make_golden_ungated import TRAINING, SAMPLING, LISTED
    return dict(TRAINING, sampling_ungated = SAMPLING, **LISTED)[name]


def test_constructor_accepts_both_options_and_rejects_other_attn_kwargs():
    tr = Transformer(128, depth = 2, heads = 4, attn_kwargs = dict(gate_values = False))
    assert tr.gate_values is False and not any('to_gates' in n for n, _ in tr.named_parameters())
    tr = Transformer(128, depth = 2, heads = 4, attn_kwargs = dict(gate_values = True, softcap_value = 30.))
    assert tr.gate_values is True and tr.softcap_value == 30. and all(hasattr(l[1].fn, 'to_gates') for l in tr.layers)
    assert Transformer(128, depth = 1, heads = 2).gate_values is True
    for H in (18, 20, 24, 30, 32):
        tr = Transformer(128, depth = 2, heads = H, use_value_residual = True)
        assert tr.layers[1][1].fn.to_learned_value_residual[0].weight.shape == (H, 128)
    assert Transformer(2048, depth = 2, heads = 16, dim_head = 128, use_value_residual = True, attn_kwargs = dict(gate_values = False)).use_value_residual
    with pytest.raises(NotImplementedError, match = r"attn_kwargs \['dim_head_scale'\]"):
        Transformer(128, depth = 1, heads = 2, attn_kwargs = dict(gate_values = False, dim_head_scale = 2.))
    with pytest.raises(NotImplementedError, match = 'heads 34'):        # the head-count limits themselves are unchanged
        Transformer(128, depth = 1, heads = 34, use_value_residual = True)


@pytest.mark.parametrize('name', sorted(LISTING))
def test_state_dict_matches_the_reference(name):
    torch.manual_seed(0)
    sd = Transfusion(**listed_ctor(name)).state_dict()
    assert {k: [list(v.shape), str(v.dtype)] for k, v in sd.items()} == LISTING[name]


def test_listing_covers_ungated_models_and_the_wide_head_counts():
    heads = {}
    for name in LISTING:
        tr = listed_ctor(name)['transformer']
        heads.setdefault(tr['heads'], set()).add((tr.get('attn_kwargs', {}).get('gate_values', True), tr.get('use_value_residual', False)))
        gated = any('to_gates' in k for k in LISTING[name])
        assert gated == tr.get('attn_kwargs', {}).get('gate_values', True), name
    assert {18, 24, 32} <= set(heads) and all(any(v for _, v in heads[h]) for h in (18, 24, 32))
    assert any(not g for s in heads.values() for g, _ in s)


def layout(ctor):
    """the engine's QKVG layout of a model: NQ, MIX and the wgrad row map, with the parameters laid out as `Engine.attach` does"""
    torch.manual_seed(0)
    eng = Engine(Transfusion(**ctor))
    named = eng._trainable()
    offs, total = {}, 0
    for n, p in named:
        offs[n] = total
        total += _round_up(p.numel(), 4)
    eng.offs, eng.named, eng.device = offs, dict(named), torch.device('cpu')
    eng._build_maps()
    return eng, offs


@pytest.mark.parametrize('gated', [True, False])
@pytest.mark.parametrize('vres', [True, False])
@pytest.mark.parametrize('H,dh', [(4, 64), (18, 64), (24, 64), (32, 64), (3, 128)])
def test_engine_layout_follows_the_gate_tile_rule(gated, vres, H, dh):
    ctor = dict(num_text_tokens = 64, dim_latent = 32, transformer = dict(dim = 256, depth = 2, heads = H, dim_head = dh, use_value_residual = vres,
                                                                         attn_kwargs = dict(gate_values = gated)))
    eng, offs = layout(ctor)
    HI, D = H * dh, 256
    assert eng.gated == gated and eng.gate_tile == (gated or vres)
    assert eng.NQ == 3 * HI + (128 if gated or vres else 0)
    assert eng.MIX == 3 * HI + H + (H % 2)             # gates stay at [0, H) of the tile, the mix at [round_even(H), + H)
    for i, lm in enumerate(eng.layer_maps):
        pre = f'transformer.layers.{i}.1.fn'
        r = lm['qkvg_rows'].numpy()
        want = np.full(eng.NQ, -1, dtype = np.int64)
        want[:2 * HI] = offs[f'{pre}.to_qk.0.weight'] + np.arange(2 * HI) * D
        want[2 * HI:3 * HI] = offs[f'{pre}.to_v.0.weight'] + np.arange(HI) * D
        if gated:
            want[3 * HI:3 * HI + H] = offs[f'{pre}.to_gates.0.weight'] + np.arange(H) * D
        if vres and i > 0:
            want[eng.MIX:eng.MIX + H] = offs[f'{pre}.to_learned_value_residual.0.weight'] + np.arange(H) * D
        assert np.array_equal(r, want), i
        # every parameter row of the attention's Linears is reached exactly once; nothing else is
        assert len(set(r[r >= 0].tolist())) == int((r >= 0).sum())


def build(fx, engine):
    torch.manual_seed(0)
    model = Transfusion(**fx['ctor'])
    synth.fill_parameters_(model, seed = fx['seed'])
    model.eval()
    model._engine = engine(model)
    return model


def check_training_fixture(name, engine):
    fx = load_golden(name)
    model = build(fx, engine)
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
    return fx, loss.item()


@pytest.mark.parametrize('name', ['small_ungated', 'small_ungated_noqknorm'])
def test_checker_matches_reference_without_gates(name):
    fx, loss = check_training_fixture(name, UngatedOracleEngine)
    assert not any('to_gates' in k for k in fx['grads'])
    # the same model with gates (their weights drawn as fill_parameters_ draws every weight) is far off: the fixture tells the two apart
    ctor = copy.deepcopy(fx['ctor'])
    ctor['transformer']['attn_kwargs'] = dict(gate_values = True)
    model = build(dict(fx, ctor = ctor), UngatedOracleEngine)
    batch = two_type_batch()
    gated = model(batch, times = fx['times'], noise = golden_noise(fx, batch, model.dim_latents)).item()
    assert abs(gated - loss) / loss > 5 * REL


def test_checker_sample_many_without_gates():
    fx = load_golden('sampling_ungated')
    model = build(fx, UngatedOracleEngine)
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


@pytest.mark.parametrize('name', ['small_ungated_laser_vres', 'small_vres_h32', 'small_wide1536_vres'])
def test_value_residual_fixtures_hold_the_mix_of_every_later_layer(name):
    """the GPU-checked fixtures carry gradients for every later layer's mix Linear (and none for a gate an ungated model lacks)"""
    fx = load_golden(name)
    tr = fx['ctor']['transformer']
    mix = sorted(k for k in fx['grads'] if 'to_learned_value_residual' in k)
    assert mix == sorted(f'transformer.layers.{i}.1.fn.to_learned_value_residual.0.{w}' for i in range(1, tr['depth']) for w in ('weight', 'bias'))
    assert any('to_gates' in k for k in fx['grads']) == tr.get('attn_kwargs', {}).get('gate_values', True)


def test_bench_step_takes_the_gate_and_value_residual_keys():
    import sys
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    from bench_step import parse_arm
    ctor, _, _ = parse_arm('512x8x128:gated=0')
    assert ctor['transformer']['attn_kwargs'] == dict(gate_values = False) and 'use_value_residual' not in ctor['transformer']
    ctor, _, B = parse_arm('2048x8x16:heads=32,vres=1,gated=1')
    assert ctor['transformer'] == dict(dim = 2048, depth = 8, dim_head = 64, heads = 32, attn_kwargs = dict(gate_values = True), use_value_residual = True) and B == 16
    Transfusion(**parse_arm('2048x1x1:heads=32,vres=1,gated=0')[0])
    for bad in ('512x8x1:gated=2', '512x8x1:vres=yes'):
        with pytest.raises(ValueError, match = 'is 0 or 1'):
            parse_arm(bad)
