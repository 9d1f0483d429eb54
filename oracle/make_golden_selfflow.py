"""TEST INFRASTRUCTURE ONLY - generates tests/golden/small_selfflow*.pt from the UNMODIFIED reference wrapper `SelfMaskedRepTraining`
(T.py:3452-3569), imported as oracle/make_golden.py does (`TFX_REFERENCE_ROOT=... python -m oracle.make_golden_selfflow`).

The wrapper runs in training mode on a ragged batch (its padded [b, n] layout has pad positions, which the cosine mean counts), with
prob_uncond = 0 and the flow noise of both forwards injected: the flat strategy draws one randn_like per modality type, the student's first,
then the teacher's.  The asymmetric-dropout case uses a `use_flex_attn` model: `Attention.dropout` stays the identity (on CUDA the reference
takes the flex_attention branch, which applies none) and every student `FeedForward.net[2]` multiplies by the restated mask of its layer
(oracle/dropout_mask.py), as oracle/make_golden_dropout.py does; the teacher's rate is 0.  Each fixture keeps the loss, the student and Self-Flow
losses, the gradient fingerprints of the student's and the head's parameters and the reference wrapper's state-dict keys.
"""
from __future__ import annotations

import os
import sys
from unittest import mock

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.reference_loader import load_reference          # noqa: E402
from oracle.make_golden import GOLDEN, compact, grad_fingerprint, noise_for        # noqa: E402
from oracle.dropout_mask import ffn_mask                    # noqa: E402
from transfusion_pytorch_b200 import synth                   # noqa: E402

CTOR = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0., transformer = dict(dim = 128, depth = 2, heads = 2))
CASES = {
    'small_selfflow': dict(use_asymmetric_dropout = False, student_layer = -3),
    'small_selfflow_last': dict(use_asymmetric_dropout = False, student_layer = -1),
    'small_selfflow_tokens': dict(use_asymmetric_dropout = False, student_layer = 0),
    'small_selfflow_drop': dict(use_asymmetric_dropout = True, student_dropout_rate = 0.1, teacher_dropout_rate = 0., student_layer = -3),
}
KEY = (0x51F7F10E, 0x0BADCAFE)
SEED = 3
HEAD_SEED = 8


def ctor_for(name):
    if name == 'small_selfflow_drop':
        return dict(CTOR, transformer = dict(CTOR['transformer'], use_flex_attn = True))
    return CTOR


def times_for(batch):
    return torch.rand(len(batch), 2, generator = torch.Generator().manual_seed(5))


def noise_seed(side, k):
    """seed of the k-th modality type's noise of the student (side 0) or the teacher (side 1)"""
    return 9000 + 500 * side + k + 17 * SEED


class _PinnedDropout(torch.nn.Module):
    """nn.Dropout(p) of the FeedForward of `layer`: x [b, n, inner] times the restated mask of packed row b * n + i (every sample is fed at
    length n in the padded layout)"""

    def __init__(self, layer, p):
        super().__init__()
        self.layer, self.p = layer, p

    def forward(self, x):
        B, n, inner = x.shape
        return x * ffn_mask(KEY, self.p, self.layer, np.arange(B * n), inner).reshape(B, n, inner)


def main():
    ref = load_reference()
    batch = synth.dropout_batch()
    times = times_for(batch)
    for name, kw in CASES.items():
        torch.manual_seed(0)
        model = ref.Transfusion(**ctor_for(name), modality_processing = 'flat')
        synth.fill_parameters_(model, seed = SEED)
        drop = kw['use_asymmetric_dropout']
        if drop:
            for layer, (_, attn, ff, _) in enumerate(model.transformer.layers):
                attn.fn.dropout = torch.nn.Identity()
                ff.fn.net[2] = _PinnedDropout(layer, kw['student_dropout_rate'])
        wrapper = ref.SelfMaskedRepTraining(model, **kw)
        synth.fill_parameters_(wrapper.student_predict_head, seed = HEAD_SEED)
        if drop:
            for _, _, ff, _ in wrapper.teacher.ema_model.transformer.layers:
                ff.fn.net[2] = torch.nn.Identity()
        wrapper.train()
        calls = []

        def fake_randn_like(t):
            side = 0 if len(calls) < model.num_modalities else 1
            k = len(calls) - side * model.num_modalities
            calls.append((side, tuple(t.shape)))
            return noise_for(t.shape[0], t.shape[1], noise_seed(side, k)).to(t)

        with mock.patch('torch.randn_like', side_effect = fake_randn_like):
            # the wrapper passes `times = student_times` to the teacher itself, so the times are pinned through the times function
            loss, (student_loss, ssl) = wrapper(batch, num_modalities_to_times_fn = lambda n: times.clone())
        loss.backward()
        assert [s for s, _ in calls] == [0] * model.num_modalities + [1] * model.num_modalities, calls
        grads = grad_fingerprint(wrapper.student)
        grads.update({f'student_predict_head.{k}': v for k, v in grad_fingerprint(wrapper.student_predict_head).items()})
        fx = dict(name = name, ctor = ctor_for(name), wrapper_kwargs = kw, seed = SEED, head_seed = HEAD_SEED, times = times, dropout_key = KEY,
                  noise_shapes = [s for _, s in calls[:model.num_modalities]], loss = loss.detach().double(), student_loss = student_loss.detach().double(),
                  ssl_loss = ssl.detach().double(), grads = grads, state_dict_keys = list(wrapper.state_dict().keys()))
        torch.save(compact(fx), os.path.join(GOLDEN, f'{name}.pt'))
        print(f'{name}: loss {loss.item():.6f} student {student_loss.item():.6f} self-flow {ssl.item():.6f}')


if __name__ == '__main__':
    main()
