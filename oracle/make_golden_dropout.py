"""TEST INFRASTRUCTURE ONLY - generates tests/golden/small_dropout.pt from the UNMODIFIED reference (imported as oracle/make_golden.py
does; `TFX_REFERENCE_ROOT=... python -m oracle.make_golden_dropout`).

FFN dropout (`ff_kwargs = dict(dropout = p)`, T.py:845-850) with a pinned mask: on the instantiated reference model, every
`FeedForward.net[2]` (the nn.Dropout after GEGLU) is replaced by a module that multiplies by the counter-based mask of its layer
(oracle/dropout_mask.py, the restatement of csrc/dropout.cuh) for a fixed key.  Everything else - flat packing, injected flow noise,
loss, backward - is the reference's own `run_interleaved` path.  Writes this one fixture only.
"""
from __future__ import annotations

import os
import sys
import types
from unittest import mock

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.reference_loader import load_reference          # noqa: E402
from oracle.make_golden import GOLDEN, compact, run_interleaved        # noqa: E402
from oracle.dropout_mask import ffn_mask                    # noqa: E402
from transfusion_pytorch_b200 import synth                   # noqa: E402

NAME = 'small_dropout'
CTOR = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), transformer = dict(dim = 128, depth = 2, heads = 2, ff_kwargs = dict(dropout = 0.2)))
KEY = (0xA4093822, 0x299F31D0)
SEED = 1


def times_for(batch):
    return torch.rand(len(batch), 2, generator = torch.Generator().manual_seed(5))


class _PinnedDropout(torch.nn.Module):
    """stands in for nn.Dropout(p) of the FeedForward of `layer`: x [b, n, inner] (the reference's padded layout) times keep / (1 - p), with
    the packed row of (b, i) = cu[b] + i taken from the sequence lengths the reference's own packing produced for this forward (`lens`)"""

    def __init__(self, layer, p, lens):
        super().__init__()
        self.layer, self.p, self.lens = layer, p, lens

    def forward(self, x):
        B, n, inner = x.shape
        # the first packing of the batch is the training forward's; the transformer sees every sample but its last token (T.py:3136, 3144)
        lens = [n_tok - 1 for n_tok in self.lens[0]]
        assert len(lens) == B and max(lens) == n, (lens, x.shape)
        cu = np.concatenate([[0], np.cumsum(lens)])
        m = torch.zeros(B, n, inner)
        for b in range(B):
            m[b, :lens[b]] = ffn_mask(KEY, self.p, self.layer, np.arange(cu[b], cu[b + 1]), inner)
        return x * m


def main():
    ref = load_reference()
    batch = synth.dropout_batch()
    times = times_for(batch)
    p = CTOR['transformer']['ff_kwargs']['dropout']
    mp = sys.modules['transfusion_pytorch.modality_processing']
    assemble, lens = mp.assemble_batch, []

    def recording_assemble(*a, **kw):                # the reference's per-sample token counts (total_lens), [sos] / [eos] included
        out = assemble(*a, **kw)
        lens.append([int(v) for v in out[4]])
        return out

    def build(**kw):
        model = ref.Transfusion(**kw)
        for layer, (_, _, ff, _) in enumerate(model.transformer.layers):
            assert isinstance(ff.fn.net[2], torch.nn.Dropout) and ff.fn.net[2].p == p
            ff.fn.net[2] = _PinnedDropout(layer, p, lens)
        return model

    with mock.patch.object(mp, 'assemble_batch', recording_assemble):
        run_interleaved(types.SimpleNamespace(Transfusion = build), NAME, CTOR, batch, times, seed = SEED)
    path = os.path.join(GOLDEN, f'{NAME}.pt')
    fx = torch.load(path, weights_only = False)
    fx.update(dropout_key = KEY, ff_dropout = p)
    torch.save(compact(fx), path)

if __name__ == '__main__':
    main()
