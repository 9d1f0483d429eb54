"""GPU: the 256 x 128 cooperative tile of tfx_gemm_store against the 128 x 128 ping-pong tile (bit for bit: same wgmma instructions, same
shared-memory data, same k order, same epilogue code), split-K wgrads at the engine's shapes against fp64, and the launch geometry that
tfx_gemm_store_items reports and engine.wgrad_splits builds on."""
import ctypes
import json

import pytest
import torch

from transfusion_pytorch_b200 import _lib
from transfusion_pytorch_b200.engine import wgrad_splits

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
WIDE, PINGPONG = 2, 3                # tfx_gemm_set_wide_mode


@pytest.fixture(scope = 'module')
def ops():
    o = _lib.Ops()
    yield o
    o.lib.tfx_gemm_set_wide_mode(1)


def _operand(mat, mn, pad = 8):
    """mat [MN, K] -> (stored tensor, row pitch): [MN][K] or, MN-major, [K][MN]; pitches padded to a multiple of `pad` elements"""
    rows, K = mat.shape
    if mn:
        t = torch.zeros(K, (rows + pad - 1) // pad * pad, device = 'cuda', dtype = BF16); t[:, :rows] = mat.t()
    else:
        t = torch.zeros(rows, (K + pad - 1) // pad * pad, device = 'cuda', dtype = BF16); t[:, :K] = mat
    return t, t.shape[1]


def _both(ops, launch):
    """run `launch` (which returns its outputs, freshly initialised) with the wide and with the ping-pong tile"""
    res = []
    for mode in (WIDE, PINGPONG):
        assert ops.lib.tfx_gemm_set_wide_mode(mode) == 0
        res.append(launch())
        torch.cuda.synchronize()
    ops.lib.tfx_gemm_set_wide_mode(1)
    return res


@pytest.mark.parametrize('a_mn,b_mn', [(0, 0), (0, 1), (1, 1), (1, 0)])
@pytest.mark.parametrize('M,N,K', [(131072, 512, 320), (1000, 1365, 1088), (257, 1408, 192), (1000, 390, 640)])
def test_wide_tile_bit_identical(ops, a_mn, b_mn, M, N, K):
    g = torch.Generator(device = 'cuda').manual_seed(M + N + K)
    A = torch.randn(M, K, device = 'cuda', generator = g).to(BF16)
    B = torch.randn(N, K, device = 'cuda', generator = g).to(BF16)
    (a, lda), (b, ldb) = _operand(A, a_mn), _operand(B, b_mn)
    Np8 = (N + 7) // 8 * 8
    bias = torch.randn(N, device = 'cuda', generator = g)

    # fp32 and bf16 outputs, bias, alpha != 1
    def full():
        out, outb = torch.zeros(M, N, device = 'cuda'), torch.zeros(M, Np8, device = 'cuda', dtype = BF16)
        ops.gemm_store(a, lda, a_mn, b, ldb, b_mn, M, N, K, out, N, outb, Np8, bias, None, 0.37, 0, 1)
        return out, outb
    (w32, wb), (p32, pb) = _both(ops, full)
    assert torch.equal(w32, p32) and torch.equal(wb, pb)
    ref = 0.37 * (A.float() @ B.float().t()) + bias
    assert torch.allclose(w32, ref, atol = 5e-2, rtol = 1e-3)

    # fp32 accumulate through per-row offsets: rows permuted, some skipped (-1), pitch N + 3 so that most rows are not 16-byte aligned
    pitch = N + 3
    perm = torch.randperm(M, device = 'cuda', generator = g)
    off = perm * pitch
    off[torch.rand(M, device = 'cuda', generator = g) < 0.1] = -1
    init = torch.randn(M * pitch, device = 'cuda', generator = g)
    def rows():
        flat = init.clone()
        ops.gemm_store(a, lda, a_mn, b, ldb, b_mn, M, N, K, flat, 0, None, 0, None, off, 1.0, 1, 1)
        return flat
    fw, fp = _both(ops, rows)
    assert torch.equal(fw, fp)
    keep = off >= 0
    got = fw.view(M, pitch)[perm[keep], :N]
    assert torch.allclose(got, init.view(M, pitch)[perm[keep], :N] + (A.float() @ B.float().t())[keep], atol = 5e-2, rtol = 1e-3)
    skipped = torch.ones(M, dtype = torch.bool, device = 'cuda'); skipped[perm[keep]] = False
    assert torch.equal(fw.view(M, pitch)[skipped], init.view(M, pitch)[skipped])

    # bf16 output only
    def bf16_only():
        outb = torch.zeros(M, Np8, device = 'cuda', dtype = BF16)
        ops.gemm_store(a, lda, a_mn, b, ldb, b_mn, M, N, K, None, 0, outb, Np8, None, None, 1.0, 0, 1)
        return outb
    bw, bp = _both(ops, bf16_only)
    assert torch.equal(bw, bp)


# the engine's wgrads over 131072 tokens: dW[n_out, n_in] += dY^T X into rows of the flat gradient buffer
WGRADS = [(2816, 512), (512, 1365), (1664, 512), (512, 512)]


@pytest.mark.parametrize('n_out,n_in', WGRADS)
def test_split_k_wgrad_matches_fp64(ops, n_out, n_in):
    T = 131072
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    s = wgrad_splits(n_out, n_in, T, sms)
    g = torch.Generator(device = 'cuda').manual_seed(n_out * 7 + n_in)
    dy = torch.randn(T, n_out, device = 'cuda', generator = g).to(BF16)
    x = torch.randn(T, n_in, device = 'cuda', generator = g).to(BF16)
    xs, ldx = _operand(x.t(), 1)                         # stored [T][n_in padded]
    base = 5                                             # row r starts at base + r * n_in: for n_in = 1365 three rows in four are unaligned
    off = base + torch.arange(n_out, device = 'cuda', dtype = torch.int64) * n_in
    init = torch.randn(base + n_out * n_in, device = 'cuda', generator = g)
    ref = (dy.double().t() @ x.double()) + init[base:].double().view(n_out, n_in)
    # the fp32 accumulator of a work item adds T / s unit-variance products in sequence; its error grows about linearly with that length
    # (H100: max |error| ~2.2e-6 per token of the item for these inputs, e.g. 0.096 at 3 splits, where |dW| ~ sqrt(T) = 362)
    tol = 4e-6 * T / s
    for mode in (1, PINGPONG):                           # the engine's selection (the wide tile here) and the ping-pong tile, same split count
        assert ops.lib.tfx_gemm_set_wide_mode(mode) == 0
        flat = init.clone()
        ops.gemm_store(dy, n_out, 1, xs, ldx, 1, n_out, n_in, T, flat, 0, None, 0, None, off, 1.0, 1, s)
        torch.cuda.synchronize()
        err = (flat[base:].double().view(n_out, n_in) - ref).abs().max().item()
        assert err < tol, (mode, s, err)
    ops.lib.tfx_gemm_set_wide_mode(1)


def test_store_items_match_the_launch(ops, tmp_path):
    """the reported geometry is what runs: kernel (wide or ping-pong) and grid size of the launch, read from a profiler trace"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cases = [(131072, 512, 2816, 0, 1, 1), (131072, 1408, 512, 0, 1, 1), (2816, 512, 131072, 1, 1, 3), (512, 1365, 65536, 1, 1, 64), (300, 390, 520, 0, 0, 1)]
    want = []
    for M, N, K, amn, bmn, s in cases:
        geo = (ctypes.c_int * 4)()
        assert ops.lib.tfx_gemm_store_items(M, N, K, amn, bmn, s, geo) == 0
        items, kb, tile_m, s_eff = geo
        assert (items, kb, tile_m, s_eff) == _lib.gemm_store_items(M, N, K, amn, bmn, s)
        kbt = (K + 63) // 64
        assert 1 <= s_eff <= s and kb == -(-kbt // s_eff) and (s_eff - 1) * kb < kbt
        assert items == -(-M // tile_m) * -(-N // 128) * s_eff
        assert tile_m == (256 if kb >= 16 else 128)     # default selection: long work items take the wide tile
        want.append((tile_m, min(items, sms)))
    g = torch.Generator(device = 'cuda').manual_seed(3)
    with torch.profiler.profile(activities = [torch.profiler.ProfilerActivity.CUDA]) as prof:
        for M, N, K, amn, bmn, s in cases:
            pad8 = lambda x: (x + 7) // 8 * 8
            a = torch.randn(K if amn else M, pad8(M if amn else K), device = 'cuda', generator = g).to(BF16)
            b = torch.randn(K if bmn else N, pad8(N if bmn else K), device = 'cuda', generator = g).to(BF16)
            out = torch.zeros(M, N, device = 'cuda')
            ops.gemm_store(a, a.shape[1], amn, b, b.shape[1], bmn, M, N, K, out, N, None, 0, None, None, 1.0, 1, s)
        torch.cuda.synchronize()
    trace = tmp_path / 'trace.json'
    prof.export_chrome_trace(str(trace))
    kern = [e for e in json.loads(trace.read_text())['traceEvents'] if e.get('cat') == 'kernel' and 'gemm_sm90' in e.get('name', '')]
    got = [(256 if 'wide' in e['name'] else 128, e['args']['grid'][0]) for e in sorted(kern, key = lambda e: e['ts'])]
    assert got == want


@pytest.mark.parametrize('n_out,n_in', WGRADS + [(1408, 512), (512, 1408)])
def test_wgrad_splits_fill_one_or_two_waves(ops, n_out, n_in):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for T in (131072, 65536, 16384):
        s = wgrad_splits(n_out, n_in, T, sms)
        items, kb, tile_m, s_eff = _lib.gemm_store_items(n_out, n_in, T, 1, 1, s)
        assert s_eff == s and kb >= 16
        assert items <= 2 * sms, (T, s, items)           # at most two waves of the persistent grid
        assert items >= 0.6 * sms or kb == 16, (T, s, items)    # and most of one, unless the items are already as short as allowed
