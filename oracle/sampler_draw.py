"""TEST INFRASTRUCTURE ONLY - NumPy restatement of the tempered token draw of transfusion_pytorch_b200/csrc/decode.cu
(`sample_tokens_k`, include/tfx_b200.h `tfx_sample_tokens`).

    h = mix64(seed ^ mix64((step << 40) ^ (s << 20) ^ c))          splitmix64 finaliser, wrapping uint64 arithmetic
    u = ((h >> 41) + 1/2) 2^-23                                       exact in fp32, in [2^-24, 1 - 2^-24]
    y_c = logit_c / T - log(-log u)                                   over the ids min-p keeps (taken over all V logits, T.py:574-578),
                                                                      then restricted to ids < vlimit (T.py:2697); the token is argmax y
step is counters[1] (0 without counters), s the sample, c the vocabulary id.  u is bit for bit the kernel's; the Gumbel value and y are
float64 here, fp32 in the kernel (`draw_error` states the difference).
Never imported by the product package.
"""
from __future__ import annotations

import numpy as np

_K0, _K1, _K2 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)
U_BITS = 23


def mix64(z):
    z = np.asarray(z, dtype = np.uint64)
    with np.errstate(over = 'ignore'):
        z = z + _K0
        z = (z ^ (z >> np.uint64(30))) * _K1
        z = (z ^ (z >> np.uint64(27))) * _K2
    return z ^ (z >> np.uint64(31))


def draw_hash(seed, step, s, c):
    """uint64 hash of (seed, step, sample, id); arguments broadcast"""
    seed, step, s, c = (np.asarray(a, dtype = np.uint64) for a in (seed, step, s, c))
    return mix64(seed ^ mix64((step << np.uint64(40)) ^ (s << np.uint64(20)) ^ c))


def uniform(h):
    """the kernel's u (an fp32 value, exact in float64)"""
    k = (np.asarray(h, dtype = np.uint64) >> np.uint64(64 - U_BITS)).astype(np.float64)
    return (k + 0.5) * 2.0 ** -U_BITS


def gumbel(u):
    return -np.log(-np.log(u))


def kept(logits, temperature, min_p, vlimit):
    """bool [..., V]: the ids a tempered draw may pick.  logits: the fp32 row(s); temperature, min_p: as the kernel receives them (fp32).
    p_c >= min_p p_max  <=>  x_c - max x >= log(min_p), x = logits / T over all V; then ids >= vlimit are dropped (vlimit 0: none).
    -inf logits are never picked (their y is -inf)."""
    x = np.asarray(logits, dtype = np.float64) / np.float64(np.float32(temperature))
    mx = x.max(-1, keepdims = True)
    mp = np.float64(np.float32(min_p))
    keep = np.isfinite(x)
    if mp > 0:
        keep &= x - mx >= np.log(mp)
    if vlimit > 0:
        keep[..., vlimit:] = False
    return keep


def draw_values(logits, temperature, seed, step, samples):
    """(y, g) float64 [S, V]: y = logit / T + Gumbel of every id of the rows of `samples` (before any filter)"""
    logits = np.asarray(logits, dtype = np.float64)
    V = logits.shape[-1]
    g = gumbel(uniform(draw_hash(seed, step, np.asarray(samples)[:, None], np.arange(V)[None, :])))
    return logits / np.float64(np.float32(temperature)) + g, g


def draw_error(x_over_t, g):
    """bound on |y_fp32 - y_float64| of one candidate: x * fp32(1 / T) rounds twice (2^-23 |x / T|), each logf is within 1 ulp (-log u
    to 2^-23 relative, so the Gumbel value to 2^-23 (1 + |g|)), and the sum rounds once (2^-24 |y|); doubled"""
    return 2.0 ** -22 * (np.abs(x_over_t) + np.abs(g) + 1.0)
