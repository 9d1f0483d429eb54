"""CPU: FFN dropout (`ff_kwargs = dict(dropout = p)`) - the Philox restatement of csrc/dropout.cuh, the dropout checker against a fixture
from the reference itself (tests/golden/small_dropout.pt), constructor validation and when a forward drops."""
import numpy as np
import pytest
import torch

from helpers import load_golden
from test_oracle_cpu import REL, check_grads
from transfusion_pytorch_b200 import Transfusion, synth
from transfusion_pytorch_b200.transfusion import Transformer
from oracle.dropout_mask import DropoutOracleEngine, keep_mask, philox4x32_10, scale, threshold, SITE_FFN


def test_philox_known_answers():
    """Random123's known-answer vectors for Philox4x32-10"""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    ctr = np.array([c for c, _, _ in cases], dtype = np.uint32)
    key = np.array([k for _, k, _ in cases], dtype = np.uint32)
    assert philox4x32_10(ctr, key).tolist() == [list(o) for _, _, o in cases]


def test_mask_layout_and_limits():
    key = (0x12345678, 0x9abcdef0)
    # element j of a group takes half-word j & 7 of the call with counter (j >> 3, i, head, 2 layer + site), low half first
    w = philox4x32_10(np.array([5, 77, 0, 2 * 3 + SITE_FFN], dtype = np.uint32), np.array(key, dtype = np.uint32))
    u16 = [(int(w[e >> 1]) >> (16 * (e & 1))) & 0xFFFF for e in range(8)]
    thr = threshold(0.5)
    assert thr == 32768
    assert keep_mask(key, 0.5, SITE_FFN, 3, 0, [77], range(40, 48))[0].tolist() == [u >= thr for u in u16]
    # a column subset gives the same bits as the full row
    full = keep_mask(key, 0.3, SITE_FFN, 1, 0, [0, 1, 999], np.arange(341))
    assert np.array_equal(keep_mask(key, 0.3, SITE_FFN, 1, 0, [999], [3, 17, 340])[0], full[2, [3, 17, 340]])
    assert full.all() == False and keep_mask(key, 0., SITE_FFN, 1, 0, [0, 1], np.arange(341)).all()
    assert not keep_mask(key, 1., SITE_FFN, 1, 0, [0, 1], np.arange(341)).any() and scale(1.) == 0.
    assert scale(0.2) == np.float32(1.25)
    # rows, layers, sites and keys give different masks
    base = keep_mask(key, 0.5, SITE_FFN, 0, 0, [10], np.arange(256))
    for other in (keep_mask(key, 0.5, SITE_FFN, 0, 0, [11], np.arange(256)), keep_mask(key, 0.5, SITE_FFN, 1, 0, [10], np.arange(256)),
                  keep_mask(key, 0.5, 0, 0, 0, [10], np.arange(256)), keep_mask((1, 2), 0.5, SITE_FFN, 0, 0, [10], np.arange(256))):
        assert 0.3 < (base != other).mean() < 0.7


def test_dropout_oracle_matches_reference():
    """the checker, with the fixture's key, against the reference whose nn.Dropout applied the same restated mask"""
    fx = load_golden('small_dropout')
    torch.manual_seed(0)
    model = Transfusion(**fx['ctor'])
    synth.fill_parameters_(model, seed = fx['seed'])
    model.train()
    model._engine = DropoutOracleEngine(model)
    batch = synth.dropout_batch()
    noise = [torch.randn(rows, dl, generator = torch.Generator().manual_seed(9000 + k + 17 * fx['seed'])) for k, (rows, dl) in enumerate(fx['noise_shapes'])]
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = noise, prob_uncond = 0., dropout_key = fx['dropout_key'])
    rb = model._last_batch
    assert rb.modality_positions == fx['modality_positions'] and rb.total_tokens == fx['total_tokens']
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < REL
    assert abs(bd.text.item() - fx['text_loss'].item()) / fx['text_loss'].item() < REL
    for a, b in zip(bd.flow, fx['flow_losses']):
        assert abs(a.item() - b.item()) / b.item() < REL
    st = model._engine.state
    for l, h in enumerate(fx['hiddens']):
        for b in range(rb.B):
            n = int(rb.seq_lens[b])
            assert torch.allclose(st['hiddens'][l][b, :n], h[b, :n], atol = 2e-4, rtol = 1e-4), f'hidden {l} sample {b}'
    loss.backward()
    check_grads(model, fx, 1e-3)
    # the masks matter: the same forward without dropout is a different loss
    model.eval()
    loss0 = model(batch, times = fx['times'], noise = noise, prob_uncond = 0.)
    assert abs(loss0.item() - fx['loss'].item()) / fx['loss'].item() > 1e-3


def test_ctor_accepts_ffn_dropout_and_rejects_the_rest():
    kw = dict(dim = 128, depth = 2, heads = 2)
    assert Transformer(**kw, ff_kwargs = dict(dropout = 0.1)).ff_dropout == 0.1
    assert Transformer(**kw).ff_dropout == 0.
    assert Transformer(**kw, ff_kwargs = dict(dropout = 1.)).ff_dropout == 1.
    # the reference's flex_attention branch applies no attention dropout: accepted, no effect
    Transformer(**kw, dropout = 0.1, use_flex_attn = True, ff_kwargs = dict(dropout = 0.1))
    with pytest.raises(NotImplementedError, match = 'attention dropout'):
        Transformer(**kw, dropout = 0.1)
    with pytest.raises(NotImplementedError, match = 'ff_kwargs'):
        Transformer(**kw, ff_kwargs = dict(dropout = 0.1, glu_mult_bias = True))
    for bad in (-0.1, 1.5):
        with pytest.raises(ValueError):
            Transformer(**kw, ff_kwargs = dict(dropout = bad))
        with pytest.raises(ValueError):
            Transformer(**kw, dropout = bad, use_flex_attn = True)
    # parameters (state-dict keys) do not depend on dropout
    assert Transformer(**kw, ff_kwargs = dict(dropout = 0.3)).state_dict().keys() == Transformer(**kw).state_dict().keys()


def test_dropout_active_only_in_training_forwards():
    tr = Transformer(dim = 128, depth = 2, heads = 2, ff_kwargs = dict(dropout = 0.25))
    assert tr.ff_dropout_p(True, True) == 0.25
    assert tr.ff_dropout_p(True, False) == 0.           # eval()
    assert tr.ff_dropout_p(False, True) == 0.           # inference forward of a module in training mode (sampling, EMA teacher)
    assert Transformer(dim = 128, depth = 2, heads = 2).ff_dropout_p(True, True) == 0.
    # attention dropout under use_flex_attn never reaches the kernels; FFN dropout still applies
    assert Transformer(dim = 128, depth = 2, heads = 2, dropout = 0.3, use_flex_attn = True).ff_dropout_p(True, True) == 0.
    assert Transformer(dim = 128, depth = 2, heads = 2, dropout = 0.3, use_flex_attn = True, ff_kwargs = dict(dropout = 0.1)).ff_dropout_p(True, True) == 0.1


class _Recorder:
    """engine double: records the keyword arguments of every forward"""

    def __init__(self, model):
        self.inner = DropoutOracleEngine(model)
        self.calls = []

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def forward(self, *a, **kw):
        self.calls.append(kw)
        return self.inner.forward(*a, **kw)


@pytest.mark.parametrize('p, training, expect', [(0.2, True, True), (0.2, False, False), (0., True, False)])
def test_transfusion_passes_the_dropout_arguments_only_when_active(p, training, expect):
    ctor = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), transformer = dict(dim = 128, depth = 2, heads = 2, ff_kwargs = dict(dropout = p)))
    torch.manual_seed(0)
    model = Transfusion(**ctor)
    synth.fill_parameters_(model, seed = 1)
    model.train(training)
    model._engine = rec = _Recorder(model)
    model(synth.dropout_batch(), prob_uncond = 0., dropout_key = (1, 2))
    model.forward_text(synth.text_batch(2, 17, vocab = 64, seed = 1), dropout_key = (3, 4))
    for kw, key in zip(rec.calls, [(1, 2), (3, 4)]):
        assert ('dropout' in kw) == expect
        if expect:
            assert kw['dropout'] is True and kw['dropout_key'] == key
