"""Shared helpers of the tests: rebuild the exact inputs the golden fixtures were generated from (parity tests), and the comparison /
sentinel plumbing of the float64 kernel tests (Checks, guarded outputs, bit-exact untouched checks, the GEMM cluster-mode fixture)."""
import os

import numpy as np
import pytest
import torch

from transfusion_pytorch_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
BF16, F32 = torch.bfloat16, torch.float32
SENT = -77.5                          # exact in bf16 and fp32

# fp32 accumulation of the wgmma main loop, relative to |A| |B|^T: 1.6e-6 is the bound measured over K <= 2752 = 43 k-blocks of 64
# (5.4e-7 there, test_block_epilogues_gpu.py).  Rounding errors of random-sign sums grow like the square root of their length, so the bound
# grows with sqrt(kb / 43) above that.  Measured on an H100 80GB HBM3 (700 W power limit), worst over the files that use it: 7.0e-7 at 64
# k-blocks (gemm_resid, K = 4096; 0.36 of c_acc(64)), 7.4e-7 at 86 (gemm_resid, K = 5504; 0.33), 6.8e-7 at 128 and 8.3e-7 at 172 (the gemm_store
# replay, where the dgrad du = dvg W1 of the d1536 and d2048 models runs them; 0.25 and 0.26), 1.4e-6 at 384 (the d2048 conditioning dgrad; 0.29).
C_ACC0, KB0 = 1.6e-6, 43


def c_acc(kb):
    """the accumulator bound of a GEMM work item that runs kb k-blocks of 64"""
    return C_ACC0 * max(1., (kb / KB0) ** 0.5)


def show_c_acc(shown, kb, measured):
    """keep a measured accumulator error (relative to |A| |B|^T) as the file's worst, and past KB0 k-blocks also per k-block count"""
    keys = ['c_acc (measured)'] + ([f'c_acc (measured) at kb = {kb}'] if kb > KB0 else [])
    for k in keys:
        shown[k] = max(shown.get(k, 0.), measured)


# ------------------------------------------------------------------------------------------------ float64 kernel tests
class Checks:
    """collects every comparison of a test, prints its worst err / bound and fails at the end with all the violations.
    `shown`: the calling module's dict of worst err / bound per check name, printed at the end of the module."""

    def __init__(self, what, shown):
        self.what, self.shown, self.bad = what, shown, []

    def __call__(self, name, got, ref, bound, row0 = 0):
        """row0: the first row of got / ref / bound when they are a row chunk of the output (for the failure report)"""
        got = got.double()
        err = (got - ref).abs()
        ratio = (err / bound.clamp_min(1e-300)).nan_to_num(nan = float('inf'))
        r = ratio.max().item() if ratio.numel() else 0.
        self.shown[name] = max(self.shown.get(name, 0.), r)
        print(f'{self.what} {name}: worst err / bound {r:.3g}')
        if not torch.isfinite(got).all():
            self.bad.append(f'{name}: non-finite values')
        elif r > 1:
            i = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
            at = (int(i[0]) + row0,) + tuple(int(x) for x in i[1:])
            self.bad.append(f'{name}: {int((ratio > 1).sum())} values off, worst err / bound {r:.3e} at {at} '
                            f'(got {got[i].item():.6e}, ref {ref[i].item():.6e})')

    def true(self, name, ok):
        if not ok:
            self.bad.append(name)

    def done(self):
        assert not self.bad, f'{self.what}:\n  ' + '\n  '.join(self.bad)


def gen(seed):
    return torch.Generator(device = 'cuda').manual_seed(seed)


def guarded(rows, cols, dtype):
    """a sentinel-filled [rows + 1, cols] buffer and its first `rows` rows; the last row is a guard the kernel must not touch"""
    buf = torch.full((rows + 1, cols), SENT, device = 'cuda', dtype = dtype)
    return buf, buf[:rows]


def same_bits(a, b):
    view = {BF16: torch.int16, F32: torch.int32}
    return torch.equal(a.contiguous().view(view[a.dtype]), b.contiguous().view(view[b.dtype]))


def untouched(t):
    return same_bits(t, torch.full_like(t, SENT))


@pytest.fixture(params = [1, 2], ids = ['single', 'paired'])
def cluster_mode(ops, request):
    """GEMM launches as independent CTAs (default) and as 2-CTA clusters sharing the B tile by TMA multicast"""
    assert ops.lib.tfx_gemm_set_cluster_mode(request.param) == 0
    yield request.param
    ops.lib.tfx_gemm_set_cluster_mode(1)


# ------------------------------------------------------------------------------------------------ parity tests


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, f'{name}.pt'), weights_only = False)


def golden_inputs(name):
    """(batch, times) exactly as oracle/make_golden.py built them."""
    if name in ('small_one_modality', 'small_laser_vres', 'small_velocity', 'small_clean'):
        return synth.small_batch(3, seed = 1, dim_latent = 32, text_vocab = 64)
    if name == 'small_posemb':
        return synth.posemb_batch()
    if name == 'small_two_modalities':
        return synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)
    if name == 'config2_b2':
        return synth.config2_batch(2, seed = 4)
    if name == 'config4_d8':
        return synth.config4_batch(2, seed = 31)
    raise KeyError(name)


def golden_noise(fx, batch, dim_latents):
    """Per-type noise tensors in the order the reference's flat strategy drew them (one randn_like per type,
    types in order of first appearance)."""
    order = []
    for s in batch:
        for p in s:
            t = p[0] if isinstance(p, tuple) else (0 if (torch.is_tensor(p) and p.is_floating_point()) else None)
            if t is not None and t not in order:
                order.append(t)
    noise = [None] * len(dim_latents)
    for k, t in enumerate(order):
        rows, dl = fx['noise_shapes'][k]
        assert dl == dim_latents[t]
        noise[t] = torch.randn(rows, dl, generator = torch.Generator().manual_seed(9000 + k + 17 * fx['seed']))
    return noise


def grad_fingerprint(named_grads):
    out = {}
    for name, g in named_grads:
        g = g.detach().float().reshape(-1).cpu()
        proj = torch.randn(g.numel(), generator = torch.Generator().manual_seed(1234))
        out[name] = dict(stats = torch.stack([g.sum(), g.abs().sum(), (g * proj).sum(), g.norm()]).double(), head = g[:8].clone())
    return out


def unpack_rows(packed, rb, width = None):
    """packed [M, d] -> padded [B, n_max, d] like the reference's batch layout"""
    n_max = int(rb.seq_lens.max())
    d = packed.shape[1] if width is None else width
    out = packed.new_zeros((rb.B, n_max, d))
    for b in range(rb.B):
        out[b, :rb.seq_lens[b]] = packed[rb.cu[b]:rb.cu[b + 1], :d]
    return out


def flatten_sample(model, sample):
    """[('t', id) ...] / [('m', (type, latents))] items of one sample (list of text tensors and (type, latents) tuples)"""
    items = []
    for p in sample:
        if torch.is_tensor(p):
            items += [('t', int(v)) for v in p.reshape(-1).tolist()]
        else:
            items.append(('m', (p[0], p[1].detach().float().cpu())))
    return items


def compare_sampling(model, out, fx, bound, lat_tol):
    """Compare `sample_many` output with a reference fixture that carries the reference's top-2 logit margins per sampled token.

    Text must be IDENTICAL up to the first sampled token whose reference margin is below `bound` (the stated bf16 logit-noise bound): a
    mismatch at a larger margin fails; at a smaller one the sample has legitimately diverged (greedy decoding of two near-tied logits) and
    the comparison of that sample stops there.  Every modality decoded before that point must match within `lat_tol` of its max magnitude.
    Returns a per-sample report: dict(matched = sampled tokens that agree, total = sampled tokens in the fixture, diverged_at = index or None,
    margin = reference margin at the divergence, latent_err = [relative errors of the compared modalities])."""
    import copy
    report = []
    forced = fx['kw'].get('force_modality_at_start')
    for i, (ours, ref) in enumerate(zip(out, fx['samples'])):
        prep = model.prepare_prompt_sample(copy.deepcopy(fx['prompts'][i]), forced)[0]
        n_prompt = len(flatten_sample(model, prep))
        a, b = flatten_sample(model, ours), flatten_sample(model, ref)
        margins = fx['margins'][i]
        g, rep = 0, dict(matched = 0, total = len(margins), diverged_at = None, margin = None, latent_err = [])
        prev_mod = False
        for j, (x, y) in enumerate(zip(a, b)):
            sampled = j >= n_prompt and y[0] == 't' and not prev_mod            # the [eom] right after a decoded modality is appended, not sampled
            if x[0] != y[0]:
                assert sampled or (j >= n_prompt and x[0] == 't' and y[0] == 'm'), f'sample {i}: structure differs at item {j} inside the prompt'
            if y[0] == 'm' and x[0] == 'm':
                assert x[1][0] == y[1][0] and x[1][1].shape == y[1][1].shape, f'sample {i}: modality type / shape differs at item {j}'
                if j >= n_prompt:
                    err = ((x[1][1] - y[1][1]).abs().max() / y[1][1].abs().max().clamp(min = 1e-9)).item()
                    rep['latent_err'].append(err)
                    assert err < lat_tol, f'sample {i}: decoded modality at item {j} differs by {err:.3e} of its max magnitude'
                else:
                    assert torch.equal(x[1][1], y[1][1])
                prev_mod = True
                continue
            if x == y:
                if sampled:
                    g += 1; rep['matched'] += 1
                prev_mod = False
                continue
            # first difference
            assert j >= n_prompt, f'sample {i}: prompt token {j} differs'
            assert sampled, f'sample {i}: non-sampled token at item {j} differs: {x} vs {y}'
            assert margins[g] < bound, f'sample {i}: sampled token {g} differs ({x} vs {y}) although the reference margin {margins[g]:.4f} >= {bound}'
            rep['diverged_at'], rep['margin'] = g, margins[g]
            break
        else:
            assert len(a) == len(b), f'sample {i}: lengths differ without a token mismatch'
        report.append(rep)
    return report
