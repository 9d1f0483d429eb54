"""GPU: the bounded-logit attention fast path on sequences long enough that its K / V and Q / dO rings wrap many times
(32 key tiles per 128-row query tile, up to 64 query steps per key tile, odd step counts), checked as the fast-path test checks it."""
import pytest

from test_ops_gpu import ops  # noqa: F401  (module fixture)
from test_ops_gpu import test_attention_tcgen05_fast_path_vs_dense as fast_path_vs_dense

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('lens,spans', [([4096], [(0, 1000, 300), (0, 2500, 700)]),            # 64 query steps for the first key tile
                                        ([4000, 1000], [(0, 100, 2000), (1, 300, 500)])])      # 63 / 16 steps: odd counts, ring slots reused unevenly
def test_attention_fast_path_long_sequences(ops, lens, spans):
    fast_path_vs_dense(ops, lens, spans)
