"""CPU: `Transformer(qk_rmsnorm = False)` (T.py:949-951: q and k go to RoPE without their RMSNorms).  The constructor accepts the flag and
keeps the reference's state-dict layout (the norms are built unconditionally, T.py:886-888); the fp32 checker (oracle/noqknorm_reference.py)
reproduces the reference's own outputs for it (tests/golden/*noqknorm*.pt, oracle/make_golden_noqknorm.py), gradients that stay None included.
The LASER / value-residual fixture is checked on the GPU only (the checker does not restate those variants, as for small_laser_vres)."""
import copy
import json
import os

import torch

from helpers import load_golden, golden_noise, grad_fingerprint
from transfusion_pytorch_b200 import Transfusion, synth
from oracle.torch_reference import OracleEngine
from oracle.noqknorm_reference import NoQkNormOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 2e-5          # fp32 restatement vs fp32 reference


def two_type_batch():
    return synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)


def build(fx, engine = NoQkNormOracleEngine):
    torch.manual_seed(0)
    model = Transfusion(**fx['ctor'])
    synth.fill_parameters_(model, seed = fx['seed'])
    model.eval()
    model._engine = engine(model)
    return model


def test_constructor_accepts_qk_rmsnorm_false_and_keeps_the_reference_layout():
    listing = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'state_dict_keys.json')))
    ctors = dict(
        config1 = dict(num_text_tokens = 256, transformer = dict(dim = 128, depth = 2, qk_rmsnorm = False)),
        config2 = dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), transformer = dict(dim = 512, depth = 8, qk_rmsnorm = False)))
    for name, ctor in ctors.items():
        model = Transfusion(**ctor)
        assert model.transformer.qk_rmsnorm is False
        sd = model.state_dict()
        assert {k: [list(v.shape), str(v.dtype)] for k, v in sd.items()} == listing[name], name
    assert Transfusion(num_text_tokens = 8, transformer = dict(dim = 128, depth = 1)).transformer.qk_rmsnorm is True


def test_gammas_stay_in_the_fixture_and_are_non_zero():
    """the fixtures were made with non-zero q / k norm gammas: a model that applied the norm anyway would not reproduce them"""
    for name in ('small_noqknorm', 'small_noqknorm_laser_vres'):
        fx = load_golden(name)
        model = build(fx)
        gam = [p for n, p in model.named_parameters() if n.endswith(('q_norm.gamma', 'k_norm.gamma'))]
        assert len(gam) == 2 * fx['ctor']['transformer']['depth'] and all(g.abs().min() > 0 for g in gam)
        assert fx['no_grad'] == sorted(n for n, p in model.named_parameters() if n.endswith(('q_norm.gamma', 'k_norm.gamma')))


def check_training_fixture(name):
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
    rows = fx['hidden_rows']                            # the positions the fixture keeps
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


def test_checker_matches_reference_without_qk_norm():
    fx, loss = check_training_fixture('small_noqknorm')
    # the normed checker on the same model is far off: the fixture tells the two paths apart
    model = build(fx, OracleEngine)
    batch = two_type_batch()
    normed = model(batch, times = fx['times'], noise = golden_noise(fx, batch, model.dim_latents)).item()
    assert abs(normed - loss) / loss > 5 * REL
    h = model._engine.state['hiddens'][1][:, fx['hidden_rows']]
    assert (h - fx['hiddens'][1]).abs().max() > 0.05 * fx['hiddens'][1].abs().max()


def test_checker_generate_text_only_without_qk_norm():
    fx = load_golden('text_noqknorm')
    model = build(fx)
    text = synth.text_batch(4, 257, seed = 3)
    loss = model(text)
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < REL
    gen = model.generate_text_only(text[:, :fx['prompt_len']], fx['gen_len'], temperature = 0.)
    assert torch.equal(gen, fx['generated'])


def test_checker_sample_many_without_qk_norm():
    fx = load_golden('sampling_noqknorm')
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
