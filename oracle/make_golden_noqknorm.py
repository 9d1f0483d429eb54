"""TEST INFRASTRUCTURE ONLY - generates the `qk_rmsnorm = False` fixtures from the UNMODIFIED reference (imported as oracle/make_golden.py
does; `TFX_REFERENCE_ROOT=... python -m oracle.make_golden_noqknorm`).  Writes these fixtures only:

  small_noqknorm            training step on an interleaved two-type batch (depth 4: two U-Net skips): loss, breakdown, hiddens and final
                            embedding at every HIDDEN_STRIDE-th position (`hidden_rows`), gradient fingerprints and the names of the parameters
                            left without a gradient (the q / k norm gammas, T.py:886-888, 949-951)
  small_noqknorm_laser_vres the same model with `attn_laser = True` and `use_value_residual = True`
  sampling_noqknorm         `sample_many`: greedy text with the reference's top-2 margin at every sampled token, decoded latents
  text_noqknorm             `generate_text_only` (greedy, with margins) plus a text-only training step

Every model gets the non-zero gammas of synth.fill_parameters_, so a kernel that applied the norm anyway would not match.
"""
from __future__ import annotations

import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.reference_loader import load_reference          # noqa: E402
from oracle.make_golden import GOLDEN, compact, count_modalities, run_interleaved, run_sampling_sized, run_text_only     # noqa: E402
from transfusion_pytorch_b200 import synth                   # noqa: E402

TWO_TYPES = dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)),
                 transformer = dict(dim = 128, depth = 4, heads = 4, qk_rmsnorm = False))
LASER_VRES = dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)),
                  transformer = dict(dim = 128, depth = 4, heads = 4, qk_rmsnorm = False, attn_laser = True, use_value_residual = True))
SAMPLING = dict(num_text_tokens = 16, dim_latent = 32, modality_default_shape = (6,), transformer = dict(dim = 128, depth = 2, heads = 2, qk_rmsnorm = False))
HIDDEN_STRIDE = 4                 # positions kept of the [B, n, D] hidden states: keeps a fixture of a depth-4 model small

TEXT = dict(num_text_tokens = 256, transformer = dict(dim = 128, depth = 2, qk_rmsnorm = False))


def two_type_batch():
    return synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)


def main():
    ref = load_reference()
    built = {}

    def recording(name):                              # the reference's Transfusion, keeping the instance to list its parameters without a gradient
        def build(**kw):
            built[name] = ref.Transfusion(**kw)
            return built[name]
        return types.SimpleNamespace(Transfusion = build)

    for name, ctor in (('small_noqknorm', TWO_TYPES), ('small_noqknorm_laser_vres', LASER_VRES)):
        batch = two_type_batch()
        times = torch.rand(2, count_modalities(batch), generator = torch.Generator().manual_seed(6))
        run_interleaved(recording(name), name, ctor, batch, times, seed = 2)
        model = built[name]
        path = os.path.join(GOLDEN, f'{name}.pt')
        fx = torch.load(path, weights_only = False)
        rows = torch.arange(0, fx['embed'].shape[1], HIDDEN_STRIDE)
        fx.update(hidden_rows = rows, hiddens = [h[:, rows] for h in fx['hiddens']], embed = fx['embed'][:, rows])
        fx['no_grad'] = sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None)
        assert fx['no_grad'] and all(n.endswith(('q_norm.gamma', 'k_norm.gamma')) for n in fx['no_grad']), fx['no_grad']
        torch.save(compact(fx), path)
    run_sampling_sized(ref, 'sampling_noqknorm', SAMPLING, seed = 5, n_each = 2, mod_len = 6, steps = 4, max_length = 40)
    run_text_only(ref, 'text_noqknorm', TEXT, synth.text_batch(4, 257, seed = 3), seed = 3)


if __name__ == '__main__':
    main()
