"""CPU: `SelfMaskedRepTraining` - the constructor's rules, state-dict keys against the reference wrapper's, the pad rows of `pack(pad_rows = True)`,
and the fp32 restatement of the wrapper's loss (oracle/selfflow_reference.py) against the reference fixtures (tests/golden/small_selfflow*.pt)."""
import numpy as np
import pytest
import torch

from helpers import load_golden
from transfusion_pytorch_b200 import Transfusion, SelfMaskedRepTraining, synth
from oracle.selfflow_reference import selfflow_loss

FIXTURES = ('small_selfflow', 'small_selfflow_last', 'small_selfflow_tokens', 'small_selfflow_drop')
SMALL = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0.)


def selfflow_noise(fx, side):
    """the fixture's injected flow noise of the student (side 0) or the teacher (side 1), per modality type (oracle/make_golden_selfflow.py)"""
    return [torch.randn(rows, dl, generator = torch.Generator().manual_seed(9000 + 500 * side + k + 17 * fx['seed'])) for k, (rows, dl) in enumerate(fx['noise_shapes'])]


def selfflow_wrapper(fx, device = 'cpu'):
    torch.manual_seed(0)
    model = Transfusion(**fx['ctor'])
    synth.fill_parameters_(model, seed = fx['seed'])
    model = model.to(device)
    wrapper = SelfMaskedRepTraining(model, **fx['wrapper_kwargs'])
    synth.fill_parameters_(wrapper.student_predict_head, seed = fx['head_seed'])
    return wrapper.to(device).train()


def grads_close(fp, ref, rel):
    for k, v in ref.items():
        ref_n = max(v['stats'][3].item(), 1e-12)
        assert abs(fp[k]['stats'][2].item() - v['stats'][2].item()) / ref_n < rel, k
        assert abs(fp[k]['stats'][3].item() - v['stats'][3].item()) / ref_n < rel, k


@pytest.mark.parametrize('name', [n for n in FIXTURES if n != 'small_selfflow_drop'])
def test_checker_matches_reference(name):
    from helpers import grad_fingerprint
    fx = load_golden(name)
    wrapper = selfflow_wrapper(fx)
    total, student, ssl = selfflow_loss(wrapper, synth.dropout_batch(), fx['times'], selfflow_noise(fx, 0), selfflow_noise(fx, 1))
    for got, want in ((total, fx['loss']), (student, fx['student_loss']), (ssl, fx['ssl_loss'])):
        assert abs(got.item() - want.item()) / abs(want.item()) < 2e-5, (got.item(), want.item())
    total.backward()
    named = [(n, p.grad) for n, p in wrapper.student.named_parameters() if p.grad is not None]
    named += [(f'student_predict_head.{n}', p.grad) for n, p in wrapper.student_predict_head.named_parameters()]
    grads_close(grad_fingerprint(named), fx['grads'], 1e-4)


def test_state_dict_keys_match_the_reference_wrapper():
    fx = load_golden('small_selfflow')
    wrapper = selfflow_wrapper(fx)
    ours = list(wrapper.state_dict().keys())
    ref_keys = fx['state_dict_keys']
    for prefix in ('student.', 'student_predict_head.'):
        assert [k for k in ours if k.startswith(prefix)] == [k for k in ref_keys if k.startswith(prefix)], prefix
    assert 'zero' in ours and 'zero' in ref_keys
    ema = wrapper.student.create_ema()
    assert [k for k in ours if k.startswith('teacher.')] == ['teacher.' + k for k in ema.state_dict().keys()]
    params = set(map(id, wrapper.parameters()))
    assert params == set(map(id, [*wrapper.student.parameters(), *wrapper.student_predict_head.parameters()]))
    assert not params & set(map(id, wrapper.teacher.parameters()))


def test_constructor_rules():
    model = lambda **tr: Transfusion(**SMALL, transformer = dict(dim = 128, depth = 2, heads = 2, **tr))
    with pytest.raises(NotImplementedError, match = 'loss_fn'):
        SelfMaskedRepTraining(model(), use_asymmetric_dropout = False, loss_fn = lambda a, b: (a - b).pow(2).mean())
    with pytest.raises(NotImplementedError, match = 'attention dropout'):
        SelfMaskedRepTraining(model())                                         # the defaults: asymmetric dropout 0.1 / 0
    with pytest.raises(AssertionError, match = 'greater dropout'):
        SelfMaskedRepTraining(model(use_flex_attn = True), student_dropout_rate = 0.1, teacher_dropout_rate = 0.1)
    for layer in (-5, 4):
        with pytest.raises(IndexError, match = 'student_layer'):
            SelfMaskedRepTraining(model(), use_asymmetric_dropout = False, student_layer = layer)
    w = SelfMaskedRepTraining(model(use_flex_attn = True))
    assert w.teacher.ema_model.training and w.student.transformer.ff_dropout == 0.       # the rate is set by forward (set_dropout_)
    w.eval()
    assert not w.teacher.ema_model.training
    w = SelfMaskedRepTraining(model(), use_asymmetric_dropout = False, rep_loss_weight = 0.)
    assert not w.has_ssl_loss and w.student_predict_head[1].net[0].weight.shape == (2 * int(128 * 8 / 3), 128)
    with pytest.raises(TypeError):
        w(torch.randint(0, 64, (2, 9)))


def _pack(model, batch, times, pad_rows):
    return model.pack(batch, times = times, prob_uncond = 0., return_loss = True, pad_rows = pad_rows)[0]


def test_pad_rows_metadata():
    """each shorter sample is fed at the longest length: its last token (no longer cut by the shift) then token 0, as text rows with label -1,
    causal, continuing rotary positions; the real rows keep their metadata relative to their sample and the loss counts are unchanged"""
    model = Transfusion(**SMALL, transformer = dict(dim = 128, depth = 2, heads = 2))
    batch = synth.dropout_batch()
    times = torch.rand(3, 2, generator = torch.Generator().manual_seed(5))
    a, b = _pack(model, batch, times, False), _pack(model, batch, times, True)
    n = int(a.seq_lens.max())
    assert a.seq_lens.tolist() == [37, 43, 45] and b.seq_lens.tolist() == [n] * 3 and b.M == 3 * n
    assert (b.total_tokens, b.n_valid, b.n_type_tokens, b.S) == (a.total_tokens, a.n_valid, a.n_type_tokens, a.S)
    for s in range(3):
        ra, rb_ = np.arange(a.cu[s], a.cu[s + 1]), np.arange(b.cu[s], b.cu[s + 1])
        k = len(ra)
        for f in ('text_id', 'label', 'rope_pos', 'cond_row'):
            assert np.array_equal(getattr(a, f)[ra], getattr(b, f)[rb_[:k]]), (f, s)
        assert np.array_equal(a.kv_limit[ra] - a.cu[s], b.kv_limit[rb_[:k]] - b.cu[s])
        assert np.array_equal(a.slot[ra] >= 0, b.slot[rb_[:k]] >= 0)
        pad = rb_[k:]
        if len(pad):
            assert b.text_id[pad[0]] == model.eos_id and (b.text_id[pad[1:]] == 0).all()
            assert (b.label[pad] == -1).all() and (b.slot[pad] == -1).all() and (b.cond_row[pad] == -1).all()
            assert np.array_equal(b.kv_limit[pad], pad)
            assert np.array_equal(b.rope_pos[pad], a.rope_pos[ra[-1]] + 1 + np.arange(len(pad)))
    # compact rows point at the same tokens, shifted by the pad rows of the samples before them
    shift = np.repeat(b.cu[:-1] - a.cu[:-1], a.seq_lens)
    assert np.array_equal(b.row_token, a.row_token + shift[a.row_token])
    # equal lengths: no pad rows
    same = [batch[0], batch[0]]
    assert np.array_equal(_pack(model, same, times[:2], True).text_id, _pack(model, same, times[:2], False).text_id)
