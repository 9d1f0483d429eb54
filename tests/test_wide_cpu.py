"""CPU: model widths 1536 and 2048.  The constructor accepts both, the state-dict layout is the reference's (tests/golden/state_dict_keys_wide.json,
listed from the reference's own state_dicts), and the fp32 checker (oracle/dh128_reference.py over oracle/torch_reference.py) reproduces the
reference's own outputs at those widths (tests/golden/*wide*.pt, oracle/make_golden_wide.py).  The LASER / value-residual fixture is checked on
the GPU only (the checker does not restate those variants)."""
import copy
import json
import os

import pytest
import torch

from helpers import load_golden, golden_noise, grad_fingerprint
from transfusion_pytorch_b200 import Transfusion, synth
from transfusion_pytorch_b200.transfusion import MODEL_DIMS, Transformer
from oracle.dh128_reference import HeadDimOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 2e-5          # fp32 restatement vs fp32 reference
NAMES = ('small_wide1536', 'small_wide2048', 'small_wide2048_laser_vres', 'sampling_wide2048')


def build(fx):
    torch.manual_seed(0)
    model = Transfusion(**fx['ctor'])
    synth.fill_parameters_(model, seed = fx['seed'])
    model.eval()
    model._engine = HeadDimOracleEngine(model)
    return model


def test_constructor_accepts_the_wide_widths():
    assert MODEL_DIMS[-2:] == (1536, 2048)
    for dim, kw in ((1536, dict(heads = 24)), (1536, dict(heads = 12, dim_head = 128)), (2048, dict(heads = 32)), (2048, dict(heads = 16, dim_head = 128))):
        t = Transformer(dim, depth = 1, **kw)
        assert t.dim == dim and t.heads == kw['heads']
    for dim in (2176, 2560, 4096):
        with pytest.raises(NotImplementedError, match = f'dim {dim}'):
            Transformer(dim, depth = 1, heads = 2)


def test_state_dict_layout_matches_the_reference():
    listing = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'state_dict_keys_wide.json')))
    assert set(listing) == set(NAMES)
    for name in NAMES:
        model = Transfusion(**load_golden(name)['ctor'])
        sd = model.state_dict()
        assert {k: [list(v.shape), str(v.dtype)] for k, v in sd.items()} == listing[name], name
        D = model.transformer.dim
        assert list(sd['transformer.layers.0.1.fn.to_qk.0.weight'].shape) == [2 * model.transformer.heads * model.transformer.dim_head, D]


@pytest.mark.parametrize('name', ['small_wide1536', 'small_wide2048'])
def test_checker_matches_reference_training_step(name):
    fx = load_golden(name)
    model = build(fx)
    batch = synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = golden_noise(fx, batch, model.dim_latents))
    rb = model._last_batch
    assert rb.modality_positions == fx['modality_positions'] and rb.total_tokens == fx['total_tokens']
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < REL
    assert abs(bd.text.item() - fx['text_loss'].item()) / fx['text_loss'].item() < REL
    assert len(bd.flow) == 2 and all(abs(a.item() - b.item()) / b.item() < REL for a, b in zip(bd.flow, fx['flow_losses']))
    st = model._engine.state
    rows = fx['hidden_rows']
    cols = fx['hidden_cols']
    for l, h in enumerate(fx['hiddens'] + [fx['embed']]):
        ours = st['hiddens'][l] if l < len(fx['hiddens']) else st['embed']
        for b in range(rb.B):
            k = rows < int(rb.seq_lens[b])
            assert torch.allclose(ours[b, rows[k]][:, cols], h[b, k], atol = 2e-4, rtol = 1e-4), f'hidden {l} sample {b}'
    loss.backward()
    assert sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None) == fx['no_grad']
    fp = grad_fingerprint((n, p.grad) for n, p in model.named_parameters() if p.grad is not None)
    assert set(fp) == set(fx['grads'])
    for k, v in fx['grads'].items():
        ref_n = max(v['stats'][3].item(), 1e-12)
        assert abs(fp[k]['stats'][2].item() - v['stats'][2].item()) / ref_n < 1e-3, k
        assert abs(fp[k]['stats'][3].item() - v['stats'][3].item()) / ref_n < 1e-3, k


def test_checker_sample_many():
    fx = load_golden('sampling_wide2048')
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
