"""TEST INFRASTRUCTURE ONLY - the CPU checker for `qk_rmsnorm = False` (T.py:949-951: q and k skip their RMSNorms and go straight to RoPE), on
top of oracle/torch_reference.py (which it leaves as it is).  Pinned by tests/test_noqknorm_cpu.py against tests/golden/*noqknorm*.pt (outputs
of the reference itself, oracle/make_golden_noqknorm.py).

TorchReference.stack normalises q and k with the module function `_rms`; for a model without the qk-RMSNorm that function is swapped, for the
duration of one stack evaluation, for one that passes q and k through unchanged (recognised by their gamma parameters) and normalises every
other input (AttentionResidual keys, final norm) as before.
"""
from __future__ import annotations

import oracle.torch_reference as _tr
from oracle.torch_reference import OracleEngine, TorchReference


class NoQkNormReference(TorchReference):
    def stack(self, *args, **kwargs):
        if getattr(self.tr, 'qk_rmsnorm', True):
            return super().stack(*args, **kwargs)
        skip = {id(p) for n, p in self.m.named_parameters() if n.endswith(('.fn.q_norm.gamma', '.fn.k_norm.gamma'))}
        rms = _tr._rms
        _tr._rms = lambda x, gamma: x if id(gamma) in skip else rms(x, gamma)
        try:
            return super().stack(*args, **kwargs)
        finally:
            _tr._rms = rms


class NoQkNormOracleEngine(OracleEngine):
    """OracleEngine that honours `Transformer(qk_rmsnorm = False)`.  Injected by the tests: `model._engine = NoQkNormOracleEngine(model)`."""

    def __init__(self, model):
        super().__init__(model)
        self.ref = NoQkNormReference(model)
