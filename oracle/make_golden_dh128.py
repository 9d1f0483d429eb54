"""TEST INFRASTRUCTURE ONLY - generates the `dim_head = 128` fixtures from the UNMODIFIED reference (imported as oracle/make_golden.py does;
`TFX_REFERENCE_ROOT=... python -m oracle.make_golden_dh128`).  Writes these fixtures only:

  small_dh128                training step on an interleaved two-type batch (dim 256, 2 heads of 128, depth 4): loss, breakdown, hiddens and
                             final embedding at every HIDDEN_STRIDE-th position (`hidden_rows`), gradient fingerprints
  small_dh128_laser_vres     the same with `attn_laser = True` and `use_value_residual = True` (3 heads: an odd count)
  small_dh128_noqknorm       the same with `qk_rmsnorm = False` (and the names of the parameters left without a gradient)
  sampling_dh128             `sample_many`: greedy text with the reference's top-2 margins, decoded latents
  text_dh128                 `generate_text_only` (greedy, with margins) plus a text-only training step
  state_dict_keys_dh128.json keys, shapes and dtypes of the reference's own state_dict for each of those constructors

Every model gets the non-zero gammas of synth.fill_parameters_, so a q / k norm over 64-wide halves would not match.
"""
from __future__ import annotations

import json
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.reference_loader import load_reference          # noqa: E402
from oracle.make_golden import GOLDEN, compact, count_modalities, run_interleaved, run_sampling_sized, run_text_only     # noqa: E402
from transfusion_pytorch_b200 import synth                   # noqa: E402

BASE = dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)))
TRAINING = dict(
    small_dh128 = dict(BASE, transformer = dict(dim = 256, depth = 4, heads = 2, dim_head = 128)),
    small_dh128_laser_vres = dict(BASE, transformer = dict(dim = 256, depth = 4, heads = 3, dim_head = 128, attn_laser = True, use_value_residual = True)),
    small_dh128_noqknorm = dict(BASE, transformer = dict(dim = 256, depth = 4, heads = 2, dim_head = 128, qk_rmsnorm = False)))
SAMPLING = dict(num_text_tokens = 16, dim_latent = 32, modality_default_shape = (6,), transformer = dict(dim = 128, depth = 2, heads = 1, dim_head = 128))
TEXT = dict(num_text_tokens = 256, transformer = dict(dim = 256, depth = 2, heads = 2, dim_head = 128))
HIDDEN_STRIDE = 8                 # positions kept of the [B, n, D] hidden states: keeps a fixture of a width-256 model near 0.5 MB


def two_type_batch():
    return synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)


def main():
    ref = load_reference()
    built = {}

    def recording(name):
        def build(**kw):
            built[name] = ref.Transfusion(**kw)
            return built[name]
        return types.SimpleNamespace(Transfusion = build)

    listing = {}
    for name, ctor in TRAINING.items():
        batch = two_type_batch()
        times = torch.rand(2, count_modalities(batch), generator = torch.Generator().manual_seed(6))
        run_interleaved(recording(name), name, ctor, batch, times, seed = 2)
        model = built[name]
        path = os.path.join(GOLDEN, f'{name}.pt')
        fx = torch.load(path, weights_only = False)
        rows = torch.arange(0, fx['embed'].shape[1], HIDDEN_STRIDE)
        fx.update(hidden_rows = rows, hiddens = [h[:, rows] for h in fx['hiddens']], embed = fx['embed'][:, rows])
        fx['no_grad'] = sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None)
        torch.save(compact(fx), path)
        listing[name] = {k: [list(v.shape), str(v.dtype)] for k, v in model.state_dict().items()}
    run_sampling_sized(ref, 'sampling_dh128', SAMPLING, seed = 5, n_each = 2, mod_len = 6, steps = 4, max_length = 40)
    run_text_only(ref, 'text_dh128', TEXT, synth.text_batch(4, 257, seed = 3), seed = 3)
    for name, ctor in (('sampling_dh128', SAMPLING), ('text_dh128', TEXT)):
        torch.manual_seed(0)
        listing[name] = {k: [list(v.shape), str(v.dtype)] for k, v in ref.Transfusion(**ctor).state_dict().items()}
    with open(os.path.join(GOLDEN, 'state_dict_keys_dh128.json'), 'w') as f:
        json.dump(listing, f, indent = 0, sort_keys = True)


if __name__ == '__main__':
    main()
