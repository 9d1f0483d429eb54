"""GPU: the fused GEMM epilogues at sizes that give every CTA several work items (three or four, so both consumer
warpgroups of a CTA take turns and some CTAs end on an odd item), against a plain PyTorch fp32 reference."""
import pytest
import torch

from transfusion_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


@pytest.fixture(params = [1, 2], ids = ['single', 'paired'])
def cluster_mode(ops, request):
    assert ops.lib.tfx_gemm_set_cluster_mode(request.param) == 0
    yield request.param
    ops.lib.tfx_gemm_set_cluster_mode(1)


def _rope_ref(x, pos, freqs):                       # interleaved pairs (x0, x1) -> (x0 c - x1 s, x1 c + x0 s)
    ang = (pos[:, None].float() * freqs).repeat_interleave(2, dim = -1)
    x2 = x.reshape(*x.shape[:-1], 32, 2)
    rot = torch.stack((-x2[..., 1], x2[..., 0]), dim = -1).flatten(-2)
    return x * ang.cos()[:, None] + rot * ang.sin()[:, None]


def test_gemm_qkvg_several_items_per_cta(ops, cluster_mode):
    M, H, D = 5000, 8, 512                           # 40 x 13 tiles
    g = torch.Generator(device = 'cuda').manual_seed(11)
    HI, NQ = H * 64, 3 * H * 64 + 128
    u = torch.randn(M, D, device = 'cuda', generator = g).to(BF16)
    W = torch.zeros(NQ, D, device = 'cuda', dtype = BF16)
    W[:3 * HI + 2 * H] = (torch.randn(3 * HI + 2 * H, D, device = 'cuda', generator = g) / D ** 0.5).to(BF16)
    gq, gk = (torch.randn(64, device = 'cuda', generator = g) * 0.3 for _ in range(2))
    pos = torch.randint(0, 900, (M,), device = 'cuda', generator = g, dtype = torch.int32)
    freqs = 1. / (10000 ** (torch.arange(0, 64, 2, device = 'cuda').float() / 64))
    t, tt = torch.empty(1024, 32, 2, device = 'cuda'), torch.empty(32, 1024, 2, device = 'cuda')
    ops.rope_table(freqs, t, tt, 1024, 32)
    q, k, v = (torch.zeros(M, HI, device = 'cuda', dtype = BF16) for _ in range(3))
    gates, mix = torch.zeros(M, H, device = 'cuda'), torch.zeros(M, H, device = 'cuda')
    inv = torch.zeros(M, 2 * H, device = 'cuda')
    ops.gemm_qkvg(u, D, W, D, M, H, D, q, k, v, gates, inv, gq, gk, pos, tt, 1024, None, mix)
    y = u.float() @ W.float().t()
    rms = lambda x, gm: torch.nn.functional.normalize(x, dim = -1) * 8. * (gm + 1.)
    qr = _rope_ref(rms(y[:, :HI].reshape(M, H, 64), gq), pos, freqs).reshape(M, HI)
    kr = _rope_ref(rms(y[:, HI:2 * HI].reshape(M, H, 64), gk), pos, freqs).reshape(M, HI)
    torch.cuda.synchronize()
    assert torch.allclose(q.float(), qr, atol = 6e-2, rtol = 2e-2) and torch.allclose(k.float(), kr, atol = 6e-2, rtol = 2e-2)
    assert torch.allclose(v.float(), y[:, 2 * HI:3 * HI], atol = 3e-2, rtol = 2e-2)
    assert torch.allclose(gates, y[:, 3 * HI:3 * HI + H], atol = 2e-2, rtol = 1e-2)
    assert torch.allclose(mix, y[:, 3 * HI + H:3 * HI + 2 * H], atol = 2e-2, rtol = 1e-2)
    assert torch.allclose(inv, 1. / y[:, :2 * HI].reshape(M, 2 * H, 64).norm(dim = -1), rtol = 1e-2, atol = 1e-4)


def test_gemm_resid_several_items_per_cta(ops, cluster_mode):
    M, N, nc = 20000, 512, 6                         # 157 x 4 tiles
    g = torch.Generator(device = 'cuda').manual_seed(12)
    bias = torch.randn(N, device = 'cuda', generator = g) * 0.2
    x_res = torch.randn(M, N, device = 'cuda', generator = g)
    cond_row = torch.randint(-1, nc, (M,), device = 'cuda', generator = g, dtype = torch.int32)
    zg = torch.rand(nc, 2 * N, device = 'cuda', generator = g)
    ls = torch.randn(N, device = 'cuda', generator = g) * 0.3
    cr = cond_row.long().clamp(min = 0)
    scale = torch.where((cond_row >= 0)[:, None], zg[cr, N:], ls + 1.)
    # attention output projection: fp32 residual out, bf16 branch output saved for backward
    K = 512
    A = torch.randn(M, K, device = 'cuda', generator = g).to(BF16)
    W = (torch.randn(N, K, device = 'cuda', generator = g) / K ** 0.5).to(BF16)
    x_out = torch.zeros(M, N, device = 'cuda'); yb = torch.zeros(M, N, device = 'cuda', dtype = BF16)
    ops.gemm_resid(A, K, None, 0, 0, W, K, M, N, K, bias, x_res, x_out, None, yb, cond_row, zg[:, N:], 2 * N, ls)
    yy = A.float() @ W.float().t() + bias
    torch.cuda.synchronize()
    assert torch.allclose(yb.float(), yy, atol = 6e-2, rtol = 2e-2)
    assert torch.allclose(x_out, x_res + yy * scale, atol = 4e-2, rtol = 1e-2)
    # feed-forward output projection: K = 1408, residual kept as bf16 only
    K = 1408
    A = torch.randn(M, K, device = 'cuda', generator = g).to(BF16)
    W = (torch.randn(N, K, device = 'cuda', generator = g) / K ** 0.5).to(BF16)
    xb = torch.zeros(M, N, device = 'cuda', dtype = BF16)
    ops.gemm_resid(A, K, None, 0, 0, W, K, M, N, K, bias, x_res, None, xb, yb, cond_row, zg[:, N:], 2 * N, ls)
    yy = A.float() @ W.float().t() + bias
    torch.cuda.synchronize()
    assert torch.allclose(yb.float(), yy, atol = 6e-2, rtol = 2e-2)
    assert torch.allclose(xb.float(), x_res + yy * scale, atol = 6e-2, rtol = 2e-2)


def test_gemm_geglu_several_items_per_cta(ops, cluster_mode):
    M, D, inner = 2900, 512, 1365                    # 23 x 22 tiles
    g = torch.Generator(device = 'cuda').manual_seed(13)
    Ip = (inner + 63) // 64 * 64
    W1 = torch.randn(2 * inner, D, device = 'cuda', generator = g) / D ** 0.5
    b1 = torch.randn(2 * inner, device = 'cuda', generator = g) * 0.3
    u = torch.randn(M, D, device = 'cuda', generator = g).to(BF16)
    Wp = torch.zeros(2 * Ip, D, device = 'cuda'); bp = torch.zeros(2 * Ip, device = 'cuda')
    col = torch.arange(Ip, device = 'cuda')
    valid = col < inner
    tile, j = col // 64, col % 64
    Wp[(tile * 128 + j)[valid]] = W1[col[valid]]; Wp[(tile * 128 + 64 + j)[valid]] = W1[inner + col[valid]]
    bp[(tile * 128 + j)[valid]] = b1[col[valid]]; bp[(tile * 128 + 64 + j)[valid]] = b1[inner + col[valid]]
    vg = torch.zeros(M, 2 * Ip, device = 'cuda', dtype = BF16); h = torch.zeros(M, Ip, device = 'cuda', dtype = BF16)
    ops.gemm_geglu(u, D, Wp.to(BF16), D, bp, M, 2 * Ip, D, vg, h)
    pre = u.float() @ W1.to(BF16).float().t() + b1
    val, gate = pre[:, :inner], pre[:, inner:]
    torch.cuda.synchronize()
    assert torch.allclose(h[:, :inner].float(), torch.nn.functional.gelu(gate) * val, atol = 6e-2, rtol = 3e-2) and (h[:, inner:] == 0).all()
    vgf = vg.float().reshape(M, Ip // 64, 2, 64)
    assert torch.allclose(vgf[:, :, 0].reshape(M, Ip)[:, :inner], val, atol = 6e-2, rtol = 2e-2)
    assert torch.allclose(vgf[:, :, 1].reshape(M, Ip)[:, :inner], gate, atol = 6e-2, rtol = 2e-2)
