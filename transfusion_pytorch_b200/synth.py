"""Deterministic synthetic workloads (BASELINE.json `configs`, SURVEY.md section 8(d)) and deterministic
parameter fill.  Everything is drawn from CPU `torch.Generator`s so that the reference (oracle side,
this container) and the CUDA path (GPU box) see bit-identical inputs and weights without shipping
them.  No dependency on the reference or on `oracle/`.
"""
from __future__ import annotations

import zlib
import torch


def _gen(seed: int) -> torch.Generator:
    g = torch.Generator(device = 'cpu')
    g.manual_seed(int(seed))
    return g


def fill_parameters_(module: torch.nn.Module, seed: int = 0, scale: float = 1.0) -> None:
    """Overwrite every parameter / persistent buffer with values that depend only on (name, shape, seed).

    The reference zero-initialises most of the conditioning path (transfusion.py:659-669, 783), which
    would hide bugs (SURVEY.md section 7, hard part 6) - so parity fixtures randomise everything, with
    magnitudes chosen to keep activations O(1).
    """
    sd = module.state_dict()
    for name in sorted(sd.keys()):
        t = sd[name]
        if not t.is_floating_point():
            continue
        g = _gen(zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1 & 0xFFFFFFFF))
        if name.endswith('rotary_emb.freqs'):
            continue                                      # keep the analytic RoPE frequencies
        shape = tuple(t.shape)
        r = torch.randn(shape, generator = g, dtype = torch.float32)
        if name.endswith('to_time_cond.0.weights'):
            v = r                                         # N(0,1) fourier frequencies, as the reference draws them
        elif t.ndim == 2:
            fan_in = shape[1]
            v = r * (scale / fan_in ** 0.5)
            if 'text_embed' in name:
                v = r * scale
        elif name.endswith('to_ada_ln_zero.bias'):
            v = r * 0.5 - 1.0
        elif name.endswith('pseudo_queries'):
            v = r * 0.5
        else:
            v = r * 0.2                                   # gammas, layerscales, biases: O(0.2) perturbation
        t.copy_(v.to(t.dtype))
    module.load_state_dict(sd)


def posemb_batch(seed: int = 77, dim_latent: int = 32, text_vocab: int = 64):
    """three ragged samples with 2-D latents of different (h, w) per instance: the axial positional embedding fixture (tests/golden/small_posemb.pt)"""
    g = _gen(seed)
    txt = lambda n: torch.randint(0, text_vocab, (n,), generator = g)
    lat = lambda h, w: torch.randn(h, w, dim_latent, generator = g)
    return [[txt(5), lat(2, 3), txt(4), lat(3, 2), txt(3)], [txt(7), lat(4, 2), txt(2)], [lat(1, 5), txt(6)]]


def config2_sample(seed: int, dim_latent: int = 384, text_vocab: int = 256,
                   text_lens = (200, 200, 99), span_len: int = 256):
    """One sample of the graded shape: [text200, latent 256xdl, text200, latent 256xdl, text99]
    -> 1025 positions after [sos]/[eos] and the 2x6 meta tokens -> n = 1024 after the shift."""
    g = _gen(1000003 * (seed + 1))
    out = []
    for i, tl in enumerate(text_lens):
        out.append(torch.randint(0, text_vocab, (tl,), generator = g))
        if i < len(text_lens) - 1:
            out.append(torch.randn(span_len, dim_latent, generator = g))
    return out


def config2_batch(batch: int, seed: int = 0, **kw):
    return [config2_sample(seed * 100003 + b, **kw) for b in range(batch)]


def config2_times(batch: int, seed: int = 0, num_modalities: int = 2) -> torch.Tensor:
    return torch.rand(batch, num_modalities, generator = _gen(77 + seed))


def small_sample(seed: int, dim_latent: int = 32, text_vocab: int = 64):
    """Small ragged sample: short text runs and spans of different lengths (parity-test sizes)."""
    g = _gen(424243 * (seed + 1))
    def ri(lo, hi):
        return int(torch.randint(lo, hi + 1, (1,), generator = g))
    out = [torch.randint(0, text_vocab, (ri(3, 20),), generator = g)]
    for _ in range(ri(1, 3)):
        out.append(torch.randn(ri(2, 40), dim_latent, generator = g))
        out.append(torch.randint(0, text_vocab, (ri(1, 25),), generator = g))
    return out


def small_batch(batch: int, seed: int = 0, **kw):
    return [small_sample(seed * 7919 + b, **kw) for b in range(batch)]


def dropout_batch(dim_latent: int = 32, text_vocab: int = 64, seed: int = 11):
    """Three interleaved samples, text | modality | text | modality | text, of odd packed lengths (37, 43 and 45 tokens with [sos] / [eos]
    and the modality delimiters): the FFN-dropout fixture, tests/golden/small_dropout.pt."""
    g = _gen(seed)
    shapes = [(5, 7, 4, 9, 3), (8, 12, 1, 6, 6), (2, 5, 11, 13, 4)]       # text, latents, text, latents, text
    return [[torch.randint(0, text_vocab, (n,), generator = g) if k % 2 == 0 else torch.randn(n, dim_latent, generator = g) for k, n in enumerate(s)]
            for s in shapes]


def config4_sample(seed: int, total_len: int = 1025, dims = (384, 192), text_vocab: int = 256):
    """Two modality types, many short alternating spans (span-mask stress), padded with text so that the
    packed length is exactly `total_len` after [sos]/[eos] and meta tokens."""
    g = _gen(9176 * (seed + 1))
    def pick(opts):
        return opts[int(torch.randint(0, len(opts), (1,), generator = g))]
    parts, used = [], 2                                    # sos + eos
    for i in range(8):
        tl = int(torch.randint(8, 41, (1,), generator = g))
        mtype = i % 2
        ml = pick((16, 32, 64, 96)) if mtype == 0 else pick((8, 24, 48))
        meta = 3 + len(str(ml))                            # [meta] digits [som] ... [eom]
        if used + tl + ml + meta + 8 > total_len:
            break
        parts.append(torch.randint(0, text_vocab, (tl,), generator = g))
        parts.append((mtype, torch.randn(ml, dims[mtype], generator = g)))
        used += tl + ml + meta
    parts.append(torch.randint(0, text_vocab, (total_len - used,), generator = g))
    return parts


def config4_batch(batch: int, seed: int = 0, **kw):
    return [config4_sample(seed * 65537 + b, **kw) for b in range(batch)]


def text_batch(batch: int, seq: int, vocab: int = 256, seed: int = 0) -> torch.Tensor:
    return torch.randint(0, vocab, (batch, seq), generator = _gen(31337 + seed))


def recon_batch(dims = (32, 16), text_vocab: int = 64, seed: int = 23):
    """Four interleaved samples with 3, 0, 1 and 2 modality instances of two types and ragged lengths (1 to 33 rows): the reconstruction-loss
    fixtures (tests/golden/small_recon*.pt)."""
    g = _gen(seed)
    txt = lambda n: torch.randint(0, text_vocab, (n,), generator = g)
    lat = lambda t, n: (t, torch.randn(n, dims[t], generator = g))
    return [[txt(4), lat(0, 5), txt(3), lat(1, 31), txt(2), lat(0, 33), txt(5)],
            [txt(9)],
            [txt(6), lat(1, 1), txt(4)],
            [lat(0, 12), txt(7), lat(1, 7), txt(3)]]


def recon_times(seed: int = 29) -> torch.Tensor:
    """times of `recon_batch`: one per instance slot, with one time near 0 and one near 1"""
    t = torch.rand(4, 3, generator = _gen(seed))
    t[0, 0], t[3, 1] = 0.02, 0.97
    return t


def modality_batch(batch: int = 3, length: int = 9, dim: int = 32, seed: int = 41) -> torch.Tensor:
    """[batch, length, dim] modalities for `forward_modality` (reconstruction / velocity fixtures)"""
    return torch.randn(batch, length, dim, generator = _gen(seed))


class StandInEncoder(torch.nn.Module):
    """Small deterministic modality encoder (a fixed Linear then tanh) standing in for a VAE encoder in the reconstruction-loss fixtures"""

    def __init__(self, dim_in: int, dim_latent: int, seed: int = 51):
        super().__init__()
        self.proj = torch.nn.Linear(dim_in, dim_latent)
        with torch.no_grad():
            self.proj.weight.copy_(torch.randn(dim_latent, dim_in, generator = _gen(seed)) * dim_in ** -0.5)
            self.proj.bias.copy_(torch.randn(dim_latent, generator = _gen(seed + 1)) * 0.1)

    def forward(self, x):
        return torch.tanh(self.proj(x))


class StandInDecoder(torch.nn.Module):
    """Decoder paired with `StandInEncoder`: a fixed Linear from the latent back to the modality's width"""

    def __init__(self, dim_latent: int, dim_out: int, seed: int = 53):
        super().__init__()
        self.proj = torch.nn.Linear(dim_latent, dim_out)
        with torch.no_grad():
            self.proj.weight.copy_(torch.randn(dim_out, dim_latent, generator = _gen(seed)) * dim_latent ** -0.5)
            self.proj.bias.copy_(torch.randn(dim_out, generator = _gen(seed + 1)) * 0.1)

    def forward(self, x):
        return self.proj(x)
