"""TEST INFRASTRUCTURE ONLY - the CPU checker for ungated attention (`attn_kwargs = dict(gate_values = False)`, T.py:901-904, 1026-1027: no
to_gates, the attention output goes to to_out without the sigmoid(gate) factor), on top of oracle/dh128_reference.py (which it leaves as it
is), so that it serves both head widths and both qk-norm modes.  Pinned by tests/test_ungated_vres_cpu.py against tests/golden/*ungated*.pt
(outputs of the reference itself, oracle/make_golden_ungated.py).

The head-dim stack multiplies the attention output by sigmoid(F.linear(u, gate weight)), looking the weight up among the model's parameters.
For an ungated model, for the duration of one stack evaluation, every layer is given a stand-in gate weight and the stack's `F.linear` returns
+inf logits for it: sigmoid(+inf) = 1 exactly, so the output is the attention output unchanged and no gradient reaches the stand-in.  Gated
models run the stack as it is.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import oracle.dh128_reference as _dh
from oracle.dh128_reference import HeadDimOracleEngine, HeadDimReference


class _ModelWithGateStandIns:
    """the model as the stack sees it: every attribute of the model, and named_parameters() with a stand-in for each layer's gate weight"""

    def __init__(self, model, stand_in):
        self._model, self._stand_in = model, stand_in

    def __getattr__(self, name):
        return getattr(self._model, name)

    def named_parameters(self):
        yield from self._model.named_parameters()
        for i in range(self._model.transformer.depth):
            yield f'transformer.layers.{i}.1.fn.to_gates.0.weight', self._stand_in


class UngatedReference(HeadDimReference):
    def stack(self, *args, **kwargs):
        if getattr(self.tr, 'gate_values', True):
            return super().stack(*args, **kwargs)
        stand_in, H = torch.empty(0), self.tr.heads

        def linear(x, w, b = None):
            if w is stand_in:
                return torch.full((*x.shape[:-1], H), float('inf'), dtype = x.dtype)
            return F.linear(x, w, b)

        model, fns = self.m, _dh.F
        self.m = _ModelWithGateStandIns(model, stand_in)
        _dh.F = _Functional(linear)
        try:
            return super().stack(*args, **kwargs)
        finally:
            self.m, _dh.F = model, fns


class _Functional:
    """torch.nn.functional with `linear` replaced"""

    def __init__(self, linear):
        self.linear = linear

    def __getattr__(self, name):
        return getattr(F, name)


class UngatedOracleEngine(HeadDimOracleEngine):
    """HeadDimOracleEngine that honours `attn_kwargs = dict(gate_values = False)`.  Injected by the tests: `model._engine = UngatedOracleEngine(model)`."""

    def __init__(self, model):
        super().__init__(model)
        self.ref = UngatedReference(model)
