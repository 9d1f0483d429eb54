"""CPU: the reconstruction loss (MP.py:177-194, T.py:3420-3431, 2836-2856) - the host-side restatement (oracle/recon_reference.py) against the
reference's own fixtures (tests/golden/small_recon*.pt), constructor validation, and the per-row / per-instance metadata of ragged batches."""
import numpy as np
import pytest
import torch

from helpers import load_golden, golden_noise
from transfusion_pytorch_b200 import Transfusion, synth
from transfusion_pytorch_b200.modality_processing import pack_batch
from oracle.recon_reference import ReconOracleEngine

TOL = 2e-5


def _model(ctor, seed, **extra):
    torch.manual_seed(0)
    model = Transfusion(**ctor, **extra)
    synth.fill_parameters_(model, seed = seed)
    model.eval()
    model._engine = ReconOracleEngine(model)
    return model


def _rel(a, b):
    a, b = float(torch.as_tensor(a).detach()), float(torch.as_tensor(b).detach())
    return abs(a - b) / max(abs(b), 1e-12)


@pytest.mark.parametrize('name', ['small_recon', 'small_recon_only'])
def test_checker_matches_reference_interleaved(name):
    fx = load_golden(name)
    model = _model(fx['ctor'], fx['seed'])
    batch = synth.recon_batch()
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = golden_noise(fx, batch, model.dim_latents))
    assert _rel(loss, fx['loss']) < TOL
    assert [len(r) for r in bd.recon] == [len(r) for r in fx['recon_losses']] == [3, 3]
    for ours, ref in zip(bd.recon, fx['recon_losses']):
        for a, b in zip(ours, ref):
            assert _rel(a, b) < TOL


@pytest.mark.parametrize('name', ['small_recon_mod', 'small_recon_mod_encdec', 'small_recon_mod_vel'])
def test_checker_matches_reference_forward_modality(name):
    fx = load_golden(name)
    extra = dict(modality_encoder = synth.StandInEncoder(24, 32), modality_decoder = synth.StandInDecoder(32, 24)) if fx['encdec'] else {}
    model = _model(fx['ctor'], fx['seed'], **extra)
    kw = {}
    if fx['ema_seed'] is not None:
        kw = dict(velocity_consistency_ema_model = _model(fx['ctor'], fx['ema_seed'], **extra), velocity_consistency_delta_time = fx['delta'])
    x = synth.modality_batch(dim = 24 if fx['encdec'] else 32)
    (shape,) = fx['noise_shapes']
    noise = torch.randn(int(np.prod(shape[:-1])), shape[-1], generator = torch.Generator().manual_seed(9000 + 17 * fx['seed']))
    loss, (flow, vel, recon) = model.forward_modality(x, times = fx['times'], return_loss_breakdown = True, noise = noise, **kw)
    assert _rel(loss, fx['loss']) < TOL and _rel(flow, fx['flow_loss']) < TOL and _rel(recon, fx['recon_loss']) < TOL
    assert abs(float(vel) - float(fx['velocity_loss'])) <= TOL * max(float(fx['velocity_loss']), 1.)


def test_residual_identity_in_float64():
    """noised - noise = t flow, so the reference's residual noised - (noise + p (1 - t)) is t flow - (1 - t) p: what the kernel computes"""
    g = torch.Generator().manual_seed(0)
    x, e, p = (torch.randn(257, 48, generator = g, dtype = torch.float64) for _ in range(3))
    for t in (0., 1e-4, 0.3, 0.9999, 1.):
        noised = x * t + e * (1. - t)
        assert torch.allclose(noised - (e + p * (1. - t)), t * (x - e) - (1. - t) * p, atol = 1e-13, rtol = 0)


def test_ctor_accepts_the_reconstruction_loss_and_still_rejects_the_unet():
    ctor = dict(num_text_tokens = 64, dim_latent = 32, transformer = dict(dim = 128, depth = 2, heads = 2))
    m = Transfusion(**ctor, reconstruction_loss_weight = 0.1)
    assert m.has_recon_loss and m.reconstruction_loss_weight == 0.1
    assert not Transfusion(**ctor).has_recon_loss
    with pytest.raises(NotImplementedError):
        Transfusion(**ctor, reconstruction_loss_weight = 0.1, pre_post_transformer_enc_dec = (torch.nn.Identity(), torch.nn.Identity()))


def _pack(model, batch, times):
    samples = [[torch.tensor([model.sos_id]), *s, torch.tensor([model.eos_id])] for s in batch]
    return pack_batch(samples, times, model, return_loss = True, return_embed = False)


def test_metadata_of_ragged_batches_with_an_absent_type():
    ctor = dict(num_text_tokens = 64, dim_latent = (32, 16, 24), modality_default_shape = ((4,), (2,), (3,)), transformer = dict(dim = 128, depth = 2, heads = 2))
    model = Transfusion(**ctor, reconstruction_loss_weight = 0.1)
    batch = synth.recon_batch()
    rb = _pack(model, batch, synth.recon_times())
    assert rb.type_rows[2][0] == rb.type_rows[2][1]                  # type 2 never occurs
    S = rb.S
    assert rb.row_inst.shape == (S,) and rb.inst_w.shape == (S,) and rb.row_inst.dtype == np.int32 and rb.inst_w.dtype == np.float32
    # brute force: walk the instances in scan order
    want_inst = np.full(S, -1)
    want_w = np.zeros(S)
    counts = {t: sum(1 for i in rb.instances if i.modality_type == t) for t in range(3)}
    assert counts == {0: 3, 1: 3, 2: 0}
    for k, inst in enumerate(rb.instances):
        r0 = rb.type_rows[inst.modality_type][0] + inst.row0
        want_inst[r0:r0 + inst.length] = k
        want_w[k] = 1. / (counts[inst.modality_type] * inst.length)
    assert (rb.row_inst == want_inst).all()
    assert np.allclose(rb.inst_w, want_w, rtol = 1e-7, atol = 0)
    assert [i.length for i in rb.instances] == [5, 31, 33, 1, 12, 7]
    # the per-type sums of the weights over the rows are 1 (each type's mean of per-instance means)
    for t in (0, 1):
        s0, s1 = rb.type_rows[t]
        assert abs(rb.inst_w[rb.row_inst[s0:s1]].sum() - 1.) < 1e-5
    # no reconstruction loss: no metadata (nothing extra is uploaded)
    rb0 = _pack(Transfusion(**ctor), batch, synth.recon_times())
    assert rb0.row_inst is None and rb0.inst_w is None


def test_metadata_shapes_depend_only_on_the_signature():
    """two batches with the same rows per type but another instance split: same shapes, other values (what a replayed CUDA graph sees)"""
    ctor = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), transformer = dict(dim = 128, depth = 2, heads = 2))
    model = Transfusion(**ctor, reconstruction_loss_weight = 0.1)
    g = torch.Generator().manual_seed(0)
    txt = lambda n: torch.randint(0, 64, (n,), generator = g)
    lat = lambda n: torch.randn(n, 32, generator = g)
    a = _pack(model, [[txt(4), lat(12), txt(4), lat(12), txt(4)]], torch.rand(1, 2, generator = g))
    b = _pack(model, [[txt(4), lat(14), txt(4), lat(10), txt(4)]], torch.rand(1, 2, generator = g))
    assert a.S == b.S and a.M == b.M and a.row_inst.shape == b.row_inst.shape and a.inst_w.shape == b.inst_w.shape
    assert not np.array_equal(a.row_inst, b.row_inst)
    assert np.allclose(b.inst_w[:2], [1 / 28, 1 / 20]) and (b.inst_w[2:] == 0).all()
