"""TEST INFRASTRUCTURE ONLY - NumPy restatement of the counter-based dropout masks of
transfusion_pytorch_b200/csrc/dropout.cuh (DESIGN.md §5), and a CPU checker that applies them where the kernels do.

    keep(key, site, layer, head, i, j): Philox4x32-10 (Random123), key (key0, key1), counter (j >> 3, i, head, 2 * layer + site);
    the four output words are eight 16-bit uniforms, element j & 7 takes half-word j & 7 (low half first); keep iff u16 >= round(p * 65536).
    Kept values are scaled by 1 / (1 - p); p = 1 drops everything.

Site 1 (FFN, nn.Dropout after GEGLU, T.py:848): i = packed token row (cu[b] + position), j = inner column, head = 0.
Never imported by the product package.
"""
from __future__ import annotations

from unittest import mock

import numpy as np
import torch

SITE_ATTN, SITE_FFN = 0, 1

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: uint32 [..., 4], key: uint32 [..., 2] (broadcast) -> uint32 [..., 4]"""
    c = [np.asarray(ctr, dtype = np.uint32)[..., k].astype(np.uint64) for k in range(4)]
    key = np.asarray(key, dtype = np.uint32)
    k0, k1 = key[..., 0].copy(), key[..., 1].copy()
    with np.errstate(over = 'ignore'):
        for _ in range(10):
            p0, p1 = _M0 * c[0], _M1 * c[2]
            c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0.astype(np.uint64), p1 & _LO, (p0 >> np.uint64(32)) ^ c[3] ^ k1.astype(np.uint64), p0 & _LO]
            k0, k1 = k0 + _W0, k1 + _W1
    return np.stack([x.astype(np.uint32) for x in c], axis = -1)


def threshold(p: float) -> int:
    """p arrives in the kernels as a float32"""
    return 65536 if p >= 1. else int(np.float64(np.float32(p)) * 65536.0 + 0.5)


def scale(p: float) -> float:
    return 0. if p >= 1. else float(np.float32(1.0 / (1.0 - np.float64(np.float32(p)))))


def keep_mask(key, p, site, layer, head, rows, cols):
    """bool [len(rows), len(cols)]: keep bit of (rows[r], cols[c]) for one (site, layer, head)"""
    rows = np.asarray(rows, dtype = np.int64)
    groups = np.unique(np.asarray(cols, dtype = np.int64) >> 3)
    ctr = np.zeros((len(rows), len(groups), 4), dtype = np.uint32)
    ctr[..., 0] = groups[None, :]
    ctr[..., 1] = rows[:, None]
    ctr[..., 2] = head
    ctr[..., 3] = 2 * layer + site
    w = philox4x32_10(ctr, np.asarray(key, dtype = np.uint32))                         # [R, G, 4]
    u16 = np.stack([w & 0xFFFF, w >> 16], axis = -1).reshape(len(rows), len(groups), 8)  # half-word e = element e of the group
    cols = np.asarray(cols, dtype = np.int64)
    g_idx = np.searchsorted(groups, cols >> 3)
    return np.ascontiguousarray(u16[:, g_idx, cols & 7] >= threshold(p))        # (the fancy index alone yields a column-major array)


def ffn_mask(key, p, layer, rows, inner):
    """float32 [len(rows), inner]: keep / (1 - p) of the FFN site for the given packed rows"""
    return torch.from_numpy(keep_mask(key, p, SITE_FFN, layer, 0, rows, np.arange(inner)).astype(np.float32) * np.float32(scale(p)))


def padded_rows(rb):
    """packed row of every (b, i) of the padded [B, n] layout (rows past a sequence's end: -1)"""
    B, n = rb.B, int(rb.seq_lens.max())
    out = np.full((B, n), -1, dtype = np.int64)
    for b in range(B):
        out[b, :rb.seq_lens[b]] = np.arange(rb.cu[b], rb.cu[b + 1])
    return out


class DropoutOracleEngine:
    """oracle.torch_reference.OracleEngine with the FFN dropout of a training forward: the FFN-out Linear of layer l (T.py:849) receives
    gelu(gate) * value times the restated mask.  Accepts the engine's `dropout` / `dropout_key` arguments; a `dropout_key` is required."""

    def __init__(self, model):
        from oracle import torch_reference
        self._tr = torch_reference
        self.inner = torch_reference.OracleEngine(model)
        self.model = model

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def forward(self, rb, latents, eps, *, train, dropout = False, dropout_key = None, **kw):
        tr = self.model.transformer
        p = tr.ff_dropout_p(train, dropout)
        if p == 0.:
            return self.inner.forward(rb, latents, eps, train = train, **kw)
        assert dropout_key is not None and not torch.is_tensor(dropout_key), 'the CPU checker needs an explicit (k0, k1) dropout key'
        rows = padded_rows(rb)
        valid = rows >= 0
        masks = {}
        for layer in range(tr.depth):
            m = torch.zeros(rows.shape + (tr.ff_inner,))
            m[torch.from_numpy(valid)] = ffn_mask(dropout_key, p, layer, rows[valid], tr.ff_inner)
            masks[self.model.get_parameter(f'transformer.layers.{layer}.2.fn.net.3.weight')] = m
        real_F = self._tr.F

        class _F:                                       # torch.nn.functional with the FFN-out Linear seeing the dropped hidden
            def __getattr__(self, name):
                return getattr(real_F, name)

            @staticmethod
            def linear(x, w, b = None):
                for wk, m in masks.items():
                    if w is wk:
                        x = x * m
                return real_F.linear(x, w, b)

        with mock.patch.object(self._tr, 'F', _F()):
            return self.inner.forward(rb, latents, eps, train = train, **kw)
