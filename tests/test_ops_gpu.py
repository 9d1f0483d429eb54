"""GPU: individual C-ABI kernels against a plain PyTorch fp32 reference of the same op."""
import math

import numpy as np
import pytest
import torch

from transfusion_pytorch_b200 import _lib
from transfusion_pytorch_b200.modality_processing import RaggedBatch, build_tiles

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


def dense_attention(q, k, v, gates, kv_limit, cu, scale, cap):
    out = torch.zeros_like(q, dtype = F32)
    H = q.shape[1] // 64
    for b in range(len(cu) - 1):
        s, e = cu[b], cu[b + 1]
        qq, kk, vv = (t[s:e].float().reshape(e - s, H, 64).transpose(0, 1) for t in (q, k, v))
        sim = torch.einsum('hid,hjd->hij', qq * scale, kk)
        sim = torch.tanh(sim / cap) * cap
        j = torch.arange(s, e, device = q.device)
        mask = j[None, :] <= kv_limit[s:e, None]
        sim = sim.masked_fill(~mask[None], -1e30)
        o = torch.einsum('hij,hjd->hid', sim.softmax(-1), vv)
        o = o * torch.sigmoid(gates[s:e].t())[..., None]
        out[s:e] = o.transpose(0, 1).reshape(e - s, H * 64)
    return out


def make_rb(lens, spans):
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    M = int(cu[-1])
    kv = np.arange(M, dtype = np.int32); qf = np.arange(M, dtype = np.int32)
    for b, off, ln in spans:
        kv[cu[b] + off: cu[b] + off + ln] = cu[b] + off + ln - 1
        qf[cu[b] + off: cu[b] + off + ln] = cu[b] + off
    z = np.zeros(M, dtype = np.int32)
    rb = RaggedBatch(B = len(lens), M = M, seq_lens = np.asarray(lens, dtype = np.int64), cu = cu, full_lens = np.asarray(lens), text_id = z, label = z, kv_limit = kv,
                     rope_pos = z, cond_row = z, slot = z, n_cond = 0, cond_times = np.zeros(0, np.float32), n_types = 0, type_rows = [], row_token = np.zeros(0, np.int32),
                     row_time = np.zeros(0, np.float32), latents = [], instances = [], modality_positions = [], total_tokens = M, n_type_tokens = [])
    build_tiles(rb, qf)
    return rb


@pytest.mark.parametrize('lens,spans', [([1024, 1024], [(0, 206, 256), (0, 668, 256), (1, 100, 700)]), ([77, 130, 5], [(0, 10, 40), (1, 64, 64), (1, 128, 2)]), ([64], [])])
def test_attention_forward_backward_vs_dense(ops, lens, spans):
    H, cap, scale = 4, 50., 0.125
    rb = make_rb(lens, spans)
    M = rb.M
    g = torch.Generator(device = 'cuda').manual_seed(1)
    q, k, v = (torch.randn(M, H * 64, device = 'cuda', generator = g).to(BF16) * 2 for _ in range(3))
    gates = torch.randn(M, H, device = 'cuda', generator = g)
    dev = lambda a: torch.from_numpy(a).cuda()
    kvl = dev(rb.kv_limit)
    o = torch.zeros(M, H * 64, device = 'cuda', dtype = BF16); lse = torch.zeros(H, M, device = 'cuda')
    ops.attn_fwd(q, k, v, H * 64, H * 64, H * 64, gates, H, kvl, dev(rb.tile_q0), dev(rb.tile_qend), dev(rb.tile_kv0), dev(rb.tile_kvend), len(rb.tile_q0), o, H * 64, lse, M, scale, cap, None)
    qf, kf, vf, gf = (t.float().requires_grad_(True) for t in (q, k, v, gates))
    ref = dense_attention(qf, kf, vf, gf, kvl.long(), rb.cu.tolist(), scale, cap)
    torch.cuda.synchronize()
    assert torch.allclose(o.float(), ref, atol = 3e-2, rtol = 3e-2)
    do = torch.randn(M, H * 64, device = 'cuda', generator = g).to(BF16)
    ref.backward(do.float())
    dop = torch.zeros_like(do); dsum = torch.zeros(H, M, device = 'cuda'); dsum2 = torch.zeros(M, H, device = 'cuda')
    ops.attn_bwd_prep(do, o, gates, dop, dsum, dsum2, None, M, H)
    dq = torch.zeros(M, H * 64, device = 'cuda'); dk = torch.zeros(M, H * 64, device = 'cuda'); dv = torch.zeros(M, H * 64, device = 'cuda', dtype = BF16)
    ops.attn_bwd(q, k, v, dop, H * 64, H * 64, H * 64, H * 64, lse, dsum, kvl, dev(rb.kt_kv0), dev(rb.kt_kvend), dev(rb.kt_q0), dev(rb.kt_qend), len(rb.kt_kv0), dq, dk, dv, H * 64,
                 M, H, scale, cap, None)
    torch.cuda.synchronize()
    for ours, want, name in ((dq, qf.grad, 'dq'), (dk, kf.grad, 'dk'), (dv.float(), vf.grad, 'dv')):
        err = (ours - want).abs().max().item() / want.abs().max().item()
        assert err < 4e-2, (name, err)
    dgate_ref = gf.grad
    dgate = (1 - torch.sigmoid(gates)) * dsum2
    assert (dgate - dgate_ref).abs().max().item() / dgate_ref.abs().max().item() < 4e-2


@pytest.mark.parametrize('lens,spans', [([1024, 1024], [(0, 206, 256), (0, 668, 256), (1, 100, 700)]), ([77, 130, 5, 300], [(0, 10, 40), (1, 64, 64), (1, 128, 2), (3, 120, 150)]), ([64], []),
                                        ([128, 129, 127], [(1, 0, 129)]), ([640] * 6 + [385, 1000, 257], [(b, 100, 300) for b in range(6)] + [(7, 100, 800)]),
                                        ([385, 1000, 257, 640, 129, 900, 31], [(1, 100, 800), (3, 0, 640), (5, 300, 77), (5, 500, 300)])])
def test_attention_tcgen05_fast_path_vs_dense(ops, lens, spans):
    """bounded-logit wgmma forward and backward (attention_sm90.cu): RMS-normalised q/k as the QKVG epilogue produces them"""
    H, cap, scale = 4, 50., 0.125
    rb = make_rb(lens, spans)
    M = rb.M
    g = torch.Generator(device = 'cuda').manual_seed(1)
    def unit(x):
        x = x.reshape(M, H, 64)
        return (torch.nn.functional.normalize(x, dim = -1) * 8.).reshape(M, H * 64).to(BF16)
    q, k = (unit(torch.randn(M, H * 64, device = 'cuda', generator = g)) for _ in range(2))
    q[: M // 2] = k[: M // 2]                       # aligned q/k: logits reach the bound (|s| = 8)
    v = (torch.randn(M, H * 64, device = 'cuda', generator = g) * 2).to(BF16)
    gates = torch.randn(M, H, device = 'cuda', generator = g)
    dev = lambda a: torch.from_numpy(a).cuda()
    kvl = dev(rb.kv_limit)
    fp = torch.zeros(8, device = 'cuda')
    zeros = torch.zeros(64, device = 'cuda')
    ops.attn_fast_params(zeros, zeros, 64, scale, cap, fp)
    torch.cuda.synchronize()
    assert fp[0].item() == 1.0 and 8.0 <= fp[1].item() <= 8.2
    o = torch.zeros(M, H * 64, device = 'cuda', dtype = BF16); lse = torch.zeros(H, M, device = 'cuda')
    ops.attn_fwd_tc(q, k, v, H * 64, H * 64, H * 64, gates, H, kvl, dev(rb.t2_q0), dev(rb.t2_qend), dev(rb.t2_kv0), dev(rb.t2_kvend), len(rb.t2_q0), o, H * 64, lse, M, 0, scale, cap, fp)
    ref = dense_attention(q.float(), k.float(), v.float(), gates, kvl.long(), rb.cu.tolist(), scale, cap)
    # the general kernel must skip when the fast flag is set, and agree when run
    o2 = torch.zeros_like(o); lse2 = torch.zeros_like(lse)
    ops.attn_fwd(q, k, v, H * 64, H * 64, H * 64, gates, H, kvl, dev(rb.tile_q0), dev(rb.tile_qend), dev(rb.tile_kv0), dev(rb.tile_kvend), len(rb.tile_q0), o2, H * 64, lse2, M, scale, cap, fp)
    torch.cuda.synchronize()
    assert (o2 == 0).all()
    ops.attn_fwd(q, k, v, H * 64, H * 64, H * 64, gates, H, kvl, dev(rb.tile_q0), dev(rb.tile_qend), dev(rb.tile_kv0), dev(rb.tile_kvend), len(rb.tile_q0), o2, H * 64, lse2, M, scale, cap, None)
    torch.cuda.synchronize()
    assert torch.allclose(o.float(), ref, atol = 3e-2, rtol = 3e-2)
    assert torch.allclose(lse, lse2, atol = 2e-3, rtol = 1e-4)
    assert torch.allclose(o.float(), o2.float(), atol = 2e-2, rtol = 2e-2)
    # ---- backward: fast kernel vs autograd of the dense reference and vs the general kernel
    qf, kf, vf, gf = (t.float().requires_grad_(True) for t in (q, k, v, gates))
    ref = dense_attention(qf, kf, vf, gf, kvl.long(), rb.cu.tolist(), scale, cap)
    do = torch.randn(M, H * 64, device = 'cuda', generator = g).to(BF16)
    ref.backward(do.float())
    dop = torch.zeros_like(do); dsum = torch.zeros(H, M, device = 'cuda'); dsum2 = torch.zeros(M, H, device = 'cuda')
    dq = torch.full((M, H * 64), 7., device = 'cuda')              # cleared by the prep kernel
    ops.attn_bwd_prep(do, o, gates, dop, dsum, dsum2, dq, M, H)
    dk = torch.zeros(M, H * 64, device = 'cuda'); dv = torch.zeros(M, H * 64, device = 'cuda', dtype = BF16)
    ops.attn_bwd_tc(q, k, v, dop, H * 64, H * 64, H * 64, H * 64, lse, dsum, kvl, dev(rb.k2_kv0), dev(rb.k2_kvend), dev(rb.k2_q0), dev(rb.k2_qend), dev(rb.k2_order), len(rb.k2_kv0), dq, dk, dv, H * 64,
                    M, H, scale, cap, fp)
    dq2 = torch.zeros(M, H * 64, device = 'cuda'); dk2 = torch.zeros(M, H * 64, device = 'cuda'); dv2 = torch.zeros(M, H * 64, device = 'cuda', dtype = BF16)
    ops.attn_bwd(q, k, v, dop, H * 64, H * 64, H * 64, H * 64, lse, dsum, kvl, dev(rb.kt_kv0), dev(rb.kt_kvend), dev(rb.kt_q0), dev(rb.kt_qend), len(rb.kt_kv0), dq2, dk2, dv2, H * 64,
                 M, H, scale, cap, None)
    # relaunch on dirty outputs (dq accumulates and is cleared by the caller, dk / dv are overwritten)
    dq3 = torch.zeros(M, H * 64, device = 'cuda'); dk3 = torch.full((M, H * 64), 3., device = 'cuda'); dv3 = torch.zeros(M, H * 64, device = 'cuda', dtype = BF16)
    for _ in range(2):
        dq3.zero_()
        ops.attn_bwd_tc(q, k, v, dop, H * 64, H * 64, H * 64, H * 64, lse, dsum, kvl, dev(rb.k2_kv0), dev(rb.k2_kvend), dev(rb.k2_q0), dev(rb.k2_qend), dev(rb.k2_order), len(rb.k2_kv0), dq3, dk3, dv3,
                        H * 64, M, H, scale, cap, fp)
    torch.cuda.synchronize()
    for ours, gen, want, name in ((dq, dq2, qf.grad, 'dq'), (dk, dk2, kf.grad, 'dk'), (dv.float(), dv2.float(), vf.grad, 'dv'),
                                  (dq3, dq2, qf.grad, 'dq_relaunch'), (dk3, dk2, kf.grad, 'dk_relaunch'), (dv3.float(), dv2.float(), vf.grad, 'dv_relaunch')):
        err = (ours - want).abs().max().item() / want.abs().max().item()
        err2 = (ours - gen).abs().max().item() / want.abs().max().item()
        assert err < 4e-2 and err2 < 4e-2, (name, err, err2)
    # large gammas: the fast path must decline
    ops.attn_fast_params(zeros + 2.0, zeros + 2.0, 64, scale, cap, fp)
    torch.cuda.synchronize()
    assert fp[0].item() == 0.0


def test_ce_and_mse_heads_vs_torch(ops):
    M, V = 500, 390
    g = torch.Generator(device = 'cuda').manual_seed(3)
    logits = torch.randn(M, 392, device = 'cuda', generator = g) * 3
    labels = torch.randint(-1, V, (M,), device = 'cuda', generator = g, dtype = torch.int32)
    dl = torch.zeros(M, 392, device = 'cuda', dtype = BF16); acc = torch.zeros(1, device = 'cuda', dtype = torch.float64); nv = torch.zeros(1, device = 'cuda', dtype = torch.int32)
    ops.ce_fwd_bwd(logits, 392, labels, V, 0, 0.25, dl, 392, acc, nv, M)
    lg = logits[:, :V].clone().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(lg, labels.long(), ignore_index = -1, reduction = 'sum')
    (ref * 0.25).backward()
    torch.cuda.synchronize()
    assert abs(acc.item() - ref.item()) / ref.item() < 1e-5 and nv.item() == int((labels >= 0).sum())
    assert torch.allclose(dl[:, :V].float(), lg.grad, atol = 2e-3, rtol = 1e-2) and (dl[:, V:] == 0).all()

