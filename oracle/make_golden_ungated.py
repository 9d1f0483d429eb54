"""TEST INFRASTRUCTURE ONLY - generates the ungated-attention (`attn_kwargs = dict(gate_values = False)`) and wide value-residual fixtures from the
UNMODIFIED reference (imported as oracle/make_golden.py does; `TFX_REFERENCE_ROOT=... python -m oracle.make_golden_ungated`).  Writes these
fixtures only:

  small_ungated              training step on an interleaved two-type batch (depth 4: two U-Net skips), `gate_values = False`: loss, breakdown,
                             hiddens and final embedding at every HIDDEN_STRIDE-th position (`hidden_rows`), gradient fingerprints
  small_ungated_laser_vres   the same with `attn_laser = True` and `use_value_residual = True` (LASER without a gate: out = log(o))
  small_ungated_noqknorm     the same as small_ungated with `qk_rmsnorm = False` (the general attention kernels)
  small_vres_h32             dim 128, 32 heads of 64, `use_value_residual` and LASER, gated: the mix columns of the QKVG gate tile are 32-63
  small_wide1536_vres        dim 1536, 24 heads of 64, `use_value_residual`, depth 2; also every HIDDEN_COL_STRIDE-th column (`hidden_cols`)
  sampling_ungated           `sample_many` of an ungated model: greedy text with the reference's top-2 margins, decoded latents
  state_dict_keys_ungated.json  keys, shapes and dtypes of the reference's own state_dict for each constructor above and for ungated / value-
                             residual models at 18, 24 and 32 heads

Noise is injected and times are pinned as in the other make_golden_* scripts.
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
from oracle.make_golden import GOLDEN, compact, count_modalities, run_interleaved, run_sampling_sized     # noqa: E402
from transfusion_pytorch_b200 import synth                   # noqa: E402

BASE = dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)))
UNGATED = dict(gate_values = False)
TRAINING = dict(
    small_ungated = dict(BASE, transformer = dict(dim = 128, depth = 4, heads = 4, attn_kwargs = UNGATED)),
    small_ungated_laser_vres = dict(BASE, transformer = dict(dim = 128, depth = 4, heads = 4, attn_kwargs = UNGATED, attn_laser = True, use_value_residual = True)),
    small_ungated_noqknorm = dict(BASE, transformer = dict(dim = 128, depth = 4, heads = 4, attn_kwargs = UNGATED, qk_rmsnorm = False)),
    small_vres_h32 = dict(BASE, transformer = dict(dim = 128, depth = 4, heads = 32, attn_laser = True, use_value_residual = True)),
    small_wide1536_vres = dict(BASE, transformer = dict(dim = 1536, depth = 2, heads = 24, use_value_residual = True)))
SAMPLING = dict(num_text_tokens = 16, dim_latent = 32, modality_default_shape = (6,), transformer = dict(dim = 128, depth = 2, heads = 2, attn_kwargs = UNGATED))
# state-dict listings only: the head counts above 16 with and without the gate
LISTED = dict(
    ungated_h18_vres = dict(num_text_tokens = 64, dim_latent = 32, transformer = dict(dim = 512, depth = 2, heads = 18, attn_kwargs = UNGATED, use_value_residual = True)),
    vres_h24 = dict(num_text_tokens = 64, dim_latent = 32, transformer = dict(dim = 1536, depth = 2, heads = 24, use_value_residual = True)),
    ungated_h24 = dict(num_text_tokens = 64, dim_latent = 32, transformer = dict(dim = 1536, depth = 2, heads = 24, attn_kwargs = UNGATED)),
    vres_h32 = dict(num_text_tokens = 64, dim_latent = 32, transformer = dict(dim = 2048, depth = 2, heads = 32, use_value_residual = True)),
    ungated_h32_vres = dict(num_text_tokens = 64, dim_latent = 32, transformer = dict(dim = 2048, depth = 2, heads = 32, attn_kwargs = UNGATED, use_value_residual = True)))
HIDDEN_STRIDE = 4                 # positions kept of the [B, n, D] hidden states
HIDDEN_COL_STRIDE = 7             # columns kept at width 1536 (as in oracle/make_golden_wide.py)


def two_type_batch():
    return synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)


def listing_of(model):
    return {k: [list(v.shape), str(v.dtype)] for k, v in model.state_dict().items()}


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
        if ctor['transformer']['dim'] > 512:
            cols = torch.arange(0, fx['embed'].shape[2], HIDDEN_COL_STRIDE)
            fx.update(hidden_rows = rows, hidden_cols = cols, hiddens = [h[:, rows][..., cols] for h in fx['hiddens']], embed = fx['embed'][:, rows][..., cols])
        else:
            fx.update(hidden_rows = rows, hiddens = [h[:, rows] for h in fx['hiddens']], embed = fx['embed'][:, rows])
        fx['no_grad'] = sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None)
        torch.save(compact(fx), path)
        listing[name] = listing_of(model)
    run_sampling_sized(ref, 'sampling_ungated', SAMPLING, seed = 5, n_each = 2, mod_len = 6, steps = 4, max_length = 40)
    for name, ctor in dict(sampling_ungated = SAMPLING, **LISTED).items():
        torch.manual_seed(0)
        listing[name] = listing_of(ref.Transfusion(**ctor))
    with open(os.path.join(GOLDEN, 'state_dict_keys_ungated.json'), 'w') as f:
        json.dump(listing, f, indent = 0, sort_keys = True)


if __name__ == '__main__':
    main()
