"""TEST INFRASTRUCTURE ONLY - generates the reconstruction-loss fixtures tests/golden/small_recon*.pt from the UNMODIFIED reference (imported as
oracle/make_golden.py does; `TFX_REFERENCE_ROOT=... python -m oracle.make_golden_recon`).  Noise is injected through `torch.randn_like`
(one seeded draw per call, in call order) and times are passed explicitly.  Writes these fixtures only:

  small_recon            interleaved, two modality types with 3 / 0 / 1 / 2 instances per sample (MP.py:177-194, T.py:3420-3431).  A type absent
                         from the batch cannot be pinned here: the reference's flow-loss weighting (T.py:3371) fails on such a batch
  small_recon_only       the same with text_loss_weight = flow_loss_weight = 0: the reconstruction term alone drives the flow head
  small_recon_clean_vel  model_output_clean + velocity consistency (EMA teacher) + reconstruction
  small_recon_mod        forward_modality, no encoder / decoder (T.py:2836-2856)
  small_recon_mod_encdec forward_modality through a deterministic encoder / decoder pair (synth.StandInEncoder / StandInDecoder)
  small_recon_mod_vel    forward_modality with velocity consistency (T.py:2823-2834) and reconstruction
"""
from __future__ import annotations

import os
import sys
from unittest import mock

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.reference_loader import load_reference          # noqa: E402
from oracle.make_golden import GOLDEN, compact, grad_fingerprint, noise_for        # noqa: E402
from transfusion_pytorch_b200 import synth                   # noqa: E402

W_R = 0.1
INTERLEAVED = dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)), reconstruction_loss_weight = W_R,
                   transformer = dict(dim = 128, depth = 2, heads = 2))
CLEAN_VEL = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), model_output_clean = True, reconstruction_loss_weight = W_R,
                 transformer = dict(dim = 128, depth = 2, heads = 2))
MODALITY = dict(num_text_tokens = 64, dim_latent = 32, reconstruction_loss_weight = W_R, transformer = dict(dim = 128, depth = 2, heads = 2))
ENC_IN = 24


class Draws:
    """stands in for torch.randn_like: call k returns the seeded draw noise_for(rows, dl, 9000 + k + 17 seed) in the tensor's shape"""

    def __init__(self, seed):
        self.seed, self.shapes = seed, []

    def __call__(self, t):
        shape = tuple(t.shape)
        e = noise_for(t.numel() // shape[-1], shape[-1], 9000 + len(self.shapes) + 17 * self.seed).reshape(shape)
        self.shapes.append(shape)
        return e.to(t)


def interleaved(ref, name, ctor, batch, times, seed, ema_seed = None, delta = 1e-3, keep_hiddens = True):
    torch.manual_seed(0)
    model = ref.Transfusion(**ctor, modality_processing = 'flat')
    synth.fill_parameters_(model, seed = seed)
    model.eval()
    kw = {}
    if ema_seed is not None:
        ema = model.create_ema(0.99)
        synth.fill_parameters_(ema.ema_model, seed = ema_seed)
        kw = dict(velocity_consistency_ema_model = ema, velocity_consistency_delta_time = delta)
    draws = Draws(seed)
    with mock.patch('torch.randn_like', side_effect = draws):
        loss, bd, hiddens = model(batch, times = times, return_breakdown = True, return_hiddens = True, **kw)
    loss.backward()
    fx = dict(name = name, ctor = ctor, seed = seed, ema_seed = ema_seed, delta = delta, times = times, noise_shapes = draws.shapes,
              loss = loss.detach().double(), text_loss = bd.text.detach().double(), flow_losses = [f.detach().double() for f in bd.flow],
              velocity_losses = [v.detach().double() for v in bd.velocity] if bd.velocity is not None else None,
              recon_losses = [[r.detach().double() for r in rs] for rs in bd.recon], grads = grad_fingerprint(model),
              embed = hiddens[-1].detach().clone())
    if keep_hiddens:
        fx['hiddens'] = [h.detach().clone() for h in hiddens[:-1]]
    torch.save(compact(fx), os.path.join(GOLDEN, f'{name}.pt'))
    print(f'{name}: loss {loss.item():.6f} flow {[round(f.item(), 6) for f in bd.flow]} recon {[[round(r.item(), 6) for r in rs] for rs in bd.recon]} draws {draws.shapes}')


def modality(ref, name, ctor, seed, encdec = False, ema_seed = None, delta = 1e-2):
    torch.manual_seed(0)
    extra = dict(modality_encoder = synth.StandInEncoder(ENC_IN, 32), modality_decoder = synth.StandInDecoder(32, ENC_IN)) if encdec else {}
    model = ref.Transfusion(**ctor, **extra)
    synth.fill_parameters_(model, seed = seed)
    model.eval()
    kw = {}
    if ema_seed is not None:
        teacher = ref.Transfusion(**ctor, **extra)
        synth.fill_parameters_(teacher, seed = ema_seed)
        kw = dict(velocity_consistency_ema_model = teacher, velocity_consistency_delta_time = delta)
    x = synth.modality_batch(dim = ENC_IN if encdec else 32)
    times = torch.rand(x.shape[0], generator = torch.Generator().manual_seed(43))
    draws = Draws(seed)
    with mock.patch('torch.randn_like', side_effect = draws):
        loss, (flow, vel, recon) = model.forward_modality(x, times = times, return_loss_breakdown = True, **kw)
    loss.backward()
    fx = dict(name = name, ctor = ctor, seed = seed, encdec = encdec, ema_seed = ema_seed, delta = delta, times = times, noise_shapes = draws.shapes,
              loss = loss.detach().double(), flow_loss = flow.detach().double(), velocity_loss = vel.detach().double(), recon_loss = recon.detach().double(),
              grads = grad_fingerprint(model))
    torch.save(compact(fx), os.path.join(GOLDEN, f'{name}.pt'))
    print(f'{name}: loss {loss.item():.6f} flow {flow.item():.6f} velocity {vel.item():.6f} recon {recon.item():.6f} draws {draws.shapes}')


def main():
    ref = load_reference()
    interleaved(ref, 'small_recon', INTERLEAVED, synth.recon_batch(), synth.recon_times(), seed = 3)
    interleaved(ref, 'small_recon_only', dict(INTERLEAVED, text_loss_weight = 0., flow_loss_weight = 0.), synth.recon_batch(), synth.recon_times(), seed = 3,
                keep_hiddens = False)      # the forward of small_recon: only the losses and gradients differ
    batch = synth.small_batch(3, seed = 1, dim_latent = 32, text_vocab = 64)
    times = (torch.rand(3, 3, generator = torch.Generator().manual_seed(7)) * 1.2).clamp(max = 0.999)
    interleaved(ref, 'small_recon_clean_vel', CLEAN_VEL, batch, times, seed = 1, ema_seed = 6, keep_hiddens = False)
    modality(ref, 'small_recon_mod', MODALITY, seed = 4)
    modality(ref, 'small_recon_mod_encdec', MODALITY, seed = 4, encdec = True)
    modality(ref, 'small_recon_mod_vel', MODALITY, seed = 4, ema_seed = 9)


if __name__ == '__main__':
    main()
