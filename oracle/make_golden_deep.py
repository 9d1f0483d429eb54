"""TEST INFRASTRUCTURE ONLY - generates the deep-model fixtures from the UNMODIFIED reference (imported as oracle/make_golden.py does;
`TFX_REFERENCE_ROOT=... python -m oracle.make_golden_deep`).  Every fixture is at dim 128, heads 2, and goes past the ten layers the deferred
AttentionResidual backward assembles in one launch.  Writes these fixtures only:

  small_deep12   depth 12, interleaved text and two modality types, injected noise and times: loss, breakdown, the final embedding, every
                 hidden state at the positions `hidden_rows` (every third), gradient fingerprints
  small_deep13   depth 13 (odd): the middle layer of the later half has no U-Net skip
  text_deep12    depth 12 text-only model: loss, gradient fingerprints, greedy generate_text_only tokens with the reference's top-2 margins
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.reference_loader import load_reference          # noqa: E402
from oracle.make_golden import GOLDEN, compact, count_modalities, run_interleaved, run_text_only        # noqa: E402
from transfusion_pytorch_b200 import synth                   # noqa: E402


def deep_ctor(depth):
    return dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)), transformer = dict(dim = 128, depth = depth, heads = 2))


# (name, depth, batch seed, packed tokens per sample): one text-only sample and one with both modality types
INTERLEAVED = [('small_deep12', 12, 118, 64), ('small_deep13', 13, 93, 72)]


def deep_batch(seed, total_len):
    return synth.config4_batch(2, seed = seed, total_len = total_len, dims = (32, 16), text_vocab = 64)


def deep_times(batch, seed):
    return torch.rand(2, count_modalities(batch), generator = torch.Generator().manual_seed(100 + seed))


HIDDEN_STRIDE = 3             # every hidden state is kept at every third position: the fixtures stay well under 1 MB


def main():
    os.makedirs(GOLDEN, exist_ok = True)
    ref = load_reference()
    for name, depth, seed, total_len in INTERLEAVED:
        batch = deep_batch(seed, total_len)
        run_interleaved(ref, name, deep_ctor(depth), batch, deep_times(batch, seed), seed = seed)
        path = os.path.join(GOLDEN, f'{name}.pt')
        fx = torch.load(path, weights_only = False)
        rows = torch.arange(0, fx['hiddens'][0].shape[1], HIDDEN_STRIDE)
        fx['hidden_rows'] = rows
        fx['hiddens'] = [h[:, rows] for h in fx['hiddens']]            # [B, len(rows), D] per hidden state, x0 first
        torch.save(compact(fx), path)
    ctor = dict(num_text_tokens = 256, transformer = dict(dim = 128, depth = 12, heads = 2))
    run_text_only(ref, 'text_deep12', ctor, synth.text_batch(4, 129, seed = 12), seed = 12, prompt_len = 16, gen_len = 32)


if __name__ == '__main__':
    main()
