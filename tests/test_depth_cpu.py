"""CPU: models deeper than ten layers.  The oracle restatement (oracle/torch_reference.py) is pinned against the deep fixtures, which are outputs of
the reference itself (oracle/make_golden_deep.py), and the depth limit is checked where models are built."""
import os
import re

import pytest
import torch

from helpers import load_golden, golden_noise
from oracle.make_golden_deep import INTERLEAVED, deep_batch
from test_oracle_cpu import REL, build, check_grads
from transfusion_pytorch_b200 import Transfusion, synth
from transfusion_pytorch_b200.transfusion import MAX_DEPTH, MODEL_DIMS, Transformer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('name,depth,seed,total_len', INTERLEAVED, ids = [c[0] for c in INTERLEAVED])
def test_oracle_matches_reference_deep(name, depth, seed, total_len):
    fx = load_golden(name)
    assert fx['ctor']['transformer']['depth'] == depth and len(fx['hiddens']) == depth + 1
    model = build(fx)
    batch = deep_batch(seed, total_len)
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = golden_noise(fx, batch, model.dim_latents))
    rb = model._last_batch
    assert rb.modality_positions == fx['modality_positions'] and rb.total_tokens == fx['total_tokens']
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < REL
    assert abs(bd.text.item() - fx['text_loss'].item()) / fx['text_loss'].item() < REL
    assert len(bd.flow) == 2 and all(abs(a.item() - b.item()) / b.item() < REL for a, b in zip(bd.flow, fx['flow_losses']))
    st = model._engine.state
    rows = fx['hidden_rows']                 # the fixture keeps every hidden state at these positions
    for l, h in enumerate(fx['hiddens']):
        for b in range(rb.B):
            keep = rows < int(rb.seq_lens[b])
            assert torch.allclose(st['hiddens'][l][b, rows[keep]], h[b, keep], atol = 2e-4, rtol = 1e-4), f'hidden {l} sample {b}'
    emb = st['embed']
    for b in range(rb.B):
        n = int(rb.seq_lens[b])
        assert torch.allclose(emb[b, :n], fx['embed'][b, :n], atol = 2e-4, rtol = 1e-4), f'embedding sample {b}'
    loss.backward()
    check_grads(model, fx, 1e-3)


def test_oracle_matches_reference_text_deep12():
    fx = load_golden('text_deep12')
    model = build(fx)
    text = synth.text_batch(4, 129, seed = 12)
    loss = model(text)
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < REL
    loss.backward()
    check_grads(model, fx, 1e-3)
    gen = model.generate_text_only(text[:, :fx['prompt_len']], fx['gen_len'], temperature = 0.)
    assert torch.equal(gen.cpu(), fx['generated'])


def test_depth_limit():
    assert MAX_DEPTH == 64
    with open(os.path.join(ROOT, 'include', 'tfx_b200.h')) as f:
        assert int(re.search(r'#define TFX_MAX_DEPTH (\d+)', f.read()).group(1)) == MAX_DEPTH       # the kernels' bound is the same number
    t = Transformer(128, depth = 64, heads = 2)
    assert len(t.layers) == 64 and sum(l[0] is not None for l in t.layers) == 32
    with pytest.raises(NotImplementedError, match = 'depth 65 > 64'):
        Transformer(128, depth = 65, heads = 2)
    with pytest.raises(NotImplementedError, match = 'depth'):
        Transfusion(num_text_tokens = 16, transformer = dict(dim = 128, depth = 65, heads = 2))


def test_width_and_head_limits():
    """the accepted widths are the widths the row kernels dispatch (the case labels of TFX_DISPATCH_NCH, D = 128 * NCH) and the widths the
    README lists; other widths and head counts the attention kernels do not take are rejected where the model is built"""
    with open(os.path.join(ROOT, 'transfusion_pytorch_b200', 'csrc', 'common.cuh')) as f:
        src = f.read()
    macro = src[src.index('#define TFX_DISPATCH_NCH'):]
    macro = macro[:macro.index('} while (0)')]
    dispatched = {128 * int(n) for n in re.findall(r'case (\d+):', macro)}
    assert dispatched == set(MODEL_DIMS) and len(MODEL_DIMS) == len(dispatched)
    with open(os.path.join(ROOT, 'README.md')) as f:
        line = re.search(r'width \(`dim`\) ([\d, or]+) with', f.read()).group(1)
    assert {int(w) for w in re.findall(r'\d+', line)} == set(MODEL_DIMS)
    for D in MODEL_DIMS:
        Transformer(D, depth = 1, heads = 2)
    Transformer(128, depth = 1, heads = 32)
    with pytest.raises(NotImplementedError, match = 'dim 640'):
        Transformer(640, depth = 2, heads = 2)
    with pytest.raises(NotImplementedError, match = 'dim 896'):
        Transformer(896, depth = 2, heads = 2)
    for heads in (3, 34, 0):
        with pytest.raises(NotImplementedError, match = f'heads {heads} '):
            Transformer(128, depth = 2, heads = heads)
