"""TEST INFRASTRUCTURE ONLY - generates the model-width 1536 / 2048 fixtures from the UNMODIFIED reference (imported as oracle/make_golden.py does;
`TFX_REFERENCE_ROOT=... python -m oracle.make_golden_wide`).  Writes these fixtures only:

  small_wide1536             training step on an interleaved two-type batch (dim 1536, depth 2, 8 heads of 64): loss, breakdown, hiddens and
                             final embedding at every HIDDEN_STRIDE-th position (`hidden_rows`) and every HIDDEN_COL_STRIDE-th column
                             (`hidden_cols`), gradient fingerprints
  small_wide2048             the same at dim 2048 with 16 heads of 128, so the attention's inner width is 2048 as well
  small_wide2048_laser_vres  the same with `attn_laser = True` and `use_value_residual = True`
  sampling_wide2048          `sample_many` at dim 2048: greedy text with the reference's top-2 margins, decoded latents
  state_dict_keys_wide.json  keys, shapes and dtypes of the reference's own state_dict for each of those constructors

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
TRAINING = dict(
    small_wide1536 = dict(BASE, transformer = dict(dim = 1536, depth = 2, heads = 8, dim_head = 64)),
    small_wide2048 = dict(BASE, transformer = dict(dim = 2048, depth = 2, heads = 16, dim_head = 128)),
    small_wide2048_laser_vres = dict(BASE, transformer = dict(dim = 2048, depth = 2, heads = 16, dim_head = 128, attn_laser = True, use_value_residual = True)))
SAMPLING = dict(num_text_tokens = 16, dim_latent = 32, modality_default_shape = (6,), transformer = dict(dim = 2048, depth = 2, heads = 4, dim_head = 64))
HIDDEN_STRIDE = 8                 # positions kept of the [B, n, D] hidden states
HIDDEN_COL_STRIDE = 7             # and columns: 7 is coprime to the 4 columns a lane owns and the 128 of a chunk, so the kept columns fall on
                                  # every lane and every chunk; keeps a width-2048 fixture near 0.4 MB


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
        cols = torch.arange(0, fx['embed'].shape[2], HIDDEN_COL_STRIDE)
        fx.update(hidden_rows = rows, hidden_cols = cols, hiddens = [h[:, rows][..., cols] for h in fx['hiddens']], embed = fx['embed'][:, rows][..., cols])
        fx['no_grad'] = sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None)
        torch.save(compact(fx), path)
        listing[name] = {k: [list(v.shape), str(v.dtype)] for k, v in model.state_dict().items()}
    run_sampling_sized(ref, 'sampling_wide2048', SAMPLING, seed = 5, n_each = 2, mod_len = 6, steps = 4, max_length = 40)
    torch.manual_seed(0)
    listing['sampling_wide2048'] = {k: [list(v.shape), str(v.dtype)] for k, v in ref.Transfusion(**SAMPLING).state_dict().items()}
    with open(os.path.join(GOLDEN, 'state_dict_keys_wide.json'), 'w') as f:
        json.dump(listing, f, indent = 0, sort_keys = True)


if __name__ == '__main__':
    main()
