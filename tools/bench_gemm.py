#!/usr/bin/env python
"""Times the wgmma GEMM family alone on the shapes of the b128 train step (M = 131072 tokens, d = 512, heads 8, FFN inner 1365 -> 1408 / 2816).
TFX_LIB=<path to a libtfx_b200 build> selects a library variant (A/B experiments).  --dump DIR writes each case's outputs as
DIR/<case>.<tensor>.npy, so that two builds can be compared bit for bit (split-K cases accumulate with atomics and are not written)."""
import argparse, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transfusion_pytorch_b200 import _lib
if os.environ.get('TFX_LIB'):
    _lib.LIB_PATH = os.environ['TFX_LIB']

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--dump', default = None, metavar = 'DIR', help = 'write the outputs of every non-split-K case to DIR/*.npy')
    ap.add_argument('--tiles', action = 'store_true', help = 'the plain-store (dgrad / wgrad) shapes of the train step with the 256 x 128 '
                    'cooperative tile and the 128 x 128 ping-pong tile alternated (tfx_gemm_set_wide_mode); with --dump both outputs per case')
    args = ap.parse_args()
    ops = _lib.Ops()
    M, D, Ip, H = int(os.environ.get('TOKENS', 131072)), 512, 1408, 8
    HI, NQ, n_cond = H * 64, 3 * H * 64 + 128, 128
    bf = torch.bfloat16
    g = torch.Generator(device = 'cuda').manual_seed(0)
    r = lambda *s: (torch.randn(*s, device = 'cuda', generator = g) * 0.05).to(bf)
    u, w1, b1 = r(M, D), r(2 * Ip, D), torch.zeros(2 * Ip, device = 'cuda')
    vg, h = torch.empty(M, 2 * Ip, device = 'cuda', dtype = bf), torch.empty(M, Ip, device = 'cuda', dtype = bf)
    w2 = r(D, Ip); dy = r(M, D); dh = torch.empty(M, Ip, device = 'cuda', dtype = bf); du = torch.empty(M, D, device = 'cuda', dtype = bf)
    gw = torch.zeros(2 * Ip, D, device = 'cuda')
    # QKVG: to_qk | to_v | to_gates (2 heads per 128-column tile) + qk-RMSNorm + RoPE
    wq = r(NQ, D)
    q, k, v = (torch.empty(M, HI, device = 'cuda', dtype = bf) for _ in range(3))
    gates, qk_inv = torch.empty(M, H, device = 'cuda'), torch.empty(M, 2 * H, device = 'cuda')
    gq, gk = (torch.randn(64, device = 'cuda', generator = g) * 0.3 for _ in range(2))
    pos = (torch.arange(M, device = 'cuda') % 1024).to(torch.int32)             # positions of packed 1024-token sequences
    freqs = 1. / (10000 ** (torch.arange(0, 64, 2, device = 'cuda').float() / 64))
    rope_t, rope_tt = torch.empty(1024, 32, 2, device = 'cuda'), torch.empty(32, 1024, 2, device = 'cuda')
    ops.rope_table(freqs, rope_t, rope_tt, 1024, 32)
    # RESID as the engine calls it: to_out (fp32 residual in / out, bf16 branch output saved) and ffn_out (bf16 hidden state out)
    att, wo, w2r = r(M, HI), r(D, HI), r(D, Ip)
    bias2 = torch.randn(D, device = 'cuda', generator = g) * 0.1
    x_a = torch.randn(M, D, device = 'cuda', generator = g)
    x_b, x_cb = torch.empty(M, D, device = 'cuda'), torch.empty(M, D, device = 'cuda', dtype = bf)
    yA, yF = (torch.empty(M, D, device = 'cuda', dtype = bf) for _ in range(2))
    cond_row = torch.randint(-1, n_cond, (M,), device = 'cuda', generator = g, dtype = torch.int32)
    zg = torch.rand(n_cond, 2 * D, device = 'cuda', generator = g)
    ls = torch.randn(D, device = 'cuda', generator = g) * 0.1
    drop_key = torch.tensor([0x1234567, 0x7654321], device = 'cuda', dtype = torch.int32)      # FFN dropout p = 0.1 (csrc/dropout.cuh)
    cases = {   # name: (launch, algorithmic FLOPs, outputs to dump)
        'qkvg   [131072 x 1664 x 512]': (lambda: ops.gemm_qkvg(u, D, wq, D, M, H, D, q, k, v, gates, qk_inv, gq, gk, pos, rope_tt, 1024, None, None),
                                         2.0 * M * NQ * D, dict(q = q, k = k, v = v, gates = gates, qk_inv = qk_inv)),
        # `gate_values = False` without the value residual: no gate tile (N = 3 HI)
        'qkvg ungated [131072 x 1536 x 512]': (lambda: ops.gemm_qkvg(u, D, wq, D, M, H, D, q, k, v, None, qk_inv, gq, gk, pos, rope_tt, 1024, None, None),
                                               2.0 * M * 3 * HI * D, dict(q = q, k = k, v = v, qk_inv = qk_inv)),
        'resid  [131072 x 512 x 512]': (lambda: ops.gemm_resid(att, HI, None, 0, 0, wo, HI, M, D, HI, None, x_a, x_b, None, yA, cond_row, zg[:, D:], 2 * D, ls),
                                        2.0 * M * D * HI, dict(x_out = x_b, y = yA)),
        'resid  [131072 x 512 x 1408]': (lambda: ops.gemm_resid(h, Ip, None, 0, 0, w2r, Ip, M, D, Ip, bias2, x_b, None, x_cb, yF, cond_row, zg[:, :D], 2 * D, ls),
                                         2.0 * M * D * Ip, dict(x_out_bf16 = x_cb, y = yF)),
        'geglu  [131072 x 2816 x 512]': (lambda: ops.gemm_geglu(u, D, w1, D, b1, M, 2 * Ip, D, vg, h), 2.0 * M * 2 * Ip * D, dict(vg = vg, h = h)),
        'geglu_drop [131072 x 2816 x 512]': (lambda: ops.gemm_geglu_drop(u, D, w1, D, b1, M, 2 * Ip, D, vg, h, drop_key, 0.1, 0), 2.0 * M * 2 * Ip * D,
                                             dict(vg = vg, h = h)),
        'store  [131072 x 2816 x 512]': (lambda: ops.gemm_store(u, D, 0, w1, D, 0, M, 2 * Ip, D, None, 0, vg, 2 * Ip, None, None, 1.0, 0, 1), 2.0 * M * 2 * Ip * D,
                                         dict(out = vg)),
        'dgrad  [131072 x 1408 x 512]': (lambda: ops.gemm_store(dy, D, 0, w2, Ip, 1, M, Ip, D, None, 0, dh, Ip, None, None, 1.0, 0, 1), 2.0 * M * Ip * D, dict(out = dh)),
        'dgrad  [131072 x 512 x 2816]': (lambda: ops.gemm_store(vg, 2 * Ip, 0, w1, D, 1, M, D, 2 * Ip, None, 0, du, D, None, None, 1.0, 0, 1), 2.0 * M * 2 * Ip * D,
                                         dict(out = du)),
        'wgrad  [2816 x 512 x 131072]': (lambda: ops.gemm_store(vg, 2 * Ip, 1, u, D, 1, 2 * Ip, D, M, gw, D, None, 0, None, None, 1.0, 1, 20), 2.0 * M * 2 * Ip * D, {}),
    }
    big = torch.empty(256 << 20, dtype = torch.uint8, device = 'cuda')
    tag = os.path.basename(os.environ.get('TFX_LIB', 'default'))
    if args.dump:
        os.makedirs(args.dump, exist_ok = True)
    if args.tiles:
        return compare_tiles(ops, M, D, Ip, big, args.dump)
    for name, (fn, fl, outs) in cases.items():
        for _ in range(3): fn()
        ts = []
        for _ in range(10):
            big.zero_()                                    # flush L2
            e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        med = sorted(ts)[5]
        print(f'{tag:36s} {name}: median {med:8.1f} us  min {min(ts):8.1f} us  {fl / med / 1e6:7.1f} TFLOP/s')
        if args.dump:
            case = name.split()[0] + '_' + name.split('[')[1].rstrip(']').replace(' x ', 'x')
            for tn, t in outs.items():
                a = t.cpu()
                np.save(os.path.join(args.dump, f'{case}.{tn}.npy'), (a.view(torch.int16) if a.dtype == bf else a).numpy())
def compare_tiles(ops, M, D, Ip, big, dump):
    """tfx_gemm_store at the train step's long-K shapes (and two short-K ones) with each tile; the wgrads use the split count the engine picks
    (`engine.wgrad_splits`, default mode) for both tiles and write rows of the flat gradient buffer as the engine does (the [512 x 1365] rows
    start 1365 floats apart, so three in four are not 16-byte aligned)"""
    from transfusion_pytorch_b200.engine import wgrad_splits
    bf = torch.bfloat16
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device = 'cuda').manual_seed(1)
    r = lambda *s: (torch.randn(*s, device = 'cuda', generator = g) * 0.05).to(bf)
    NQ, inner = 3 * 8 * 64 + 128, 1365
    cases = {}      # name: (launch, algorithmic FLOPs, output, split-K)
    def dgrad(N, K):
        a, b, out = r(M, K), r(K, N), torch.empty(M, N, device = 'cuda', dtype = bf)      # dY [M, K] x W stored [K][N] (MN-major)
        cases[f'dgrad [{M} x {N} x {K}]'] = (lambda: ops.gemm_store(a, K, 0, b, N, 1, M, N, K, None, 0, out, N, None, None, 1.0, 0, 1), 2.0 * M * N * K, out, 1)
    def wgrad(n_out, n_in):
        s = wgrad_splits(n_out, n_in, M, sms)
        a, b = r(M, n_out), r(M, (n_in + 63) // 64 * 64)
        flat = torch.zeros(n_out * n_in + 4, device = 'cuda')
        rows = torch.arange(n_out, device = 'cuda', dtype = torch.int64) * n_in + 4    # offset 4: the first row aligned, as no real one needs to be
        cases[f'wgrad [{n_out} x {n_in} x {M}] splits {s}'] = (lambda: ops.gemm_store(a, n_out, 1, b, b.shape[1], 1, n_out, n_in, M, flat, 0, None, 0, None, rows,
                                                                                     1.0, 1, s), 2.0 * M * n_out * n_in, flat, s)
    dgrad(D, 2 * Ip); wgrad(2 * Ip, D); wgrad(D, inner); dgrad(D, NQ); wgrad(NQ, D); wgrad(D, D); dgrad(2 * Ip // 2, D); dgrad(D, D)
    modes = {'wide': 2, 'pingpong': 3}
    for name, (fn, fl, out, s) in cases.items():
        res, ts = {}, {m: [] for m in modes}
        for m, code in modes.items():                       # warm-up, and the output of each tile from a zeroed destination
            ops.lib.tfx_gemm_set_wide_mode(code)
            out.zero_(); fn(); torch.cuda.synchronize()
            res[m] = out.clone()
            for _ in range(2): fn()
        for _ in range(10):
            for m, code in modes.items():
                ops.lib.tfx_gemm_set_wide_mode(code)
                big.zero_()                                 # flush L2
                e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
                e0.record(); fn(); e1.record(); torch.cuda.synchronize()
                ts[m].append(e0.elapsed_time(e1) * 1e3)
        ops.lib.tfx_gemm_set_wide_mode(1)
        med = {m: sorted(t)[5] for m, t in ts.items()}
        same = 'bit-identical' if torch.equal(res['wide'], res['pingpong']) else f'max |diff| {(res["wide"].float() - res["pingpong"].float()).abs().max().item():.3g}'
        print(f'{name:44s} ' + '  '.join(f'{m} {med[m]:7.1f} us ({fl / med[m] / 1e6:5.1f} TFLOP/s)' for m in modes)
              + f'  wide/pingpong {med["wide"] / med["pingpong"]:.3f}  outputs {same}' + (' (split-K atomics)' if s > 1 else ''), flush = True)
        if dump:
            case = name.split()[0] + '_' + name.split('[')[1].split(']')[0].replace(' x ', 'x')
            for m, t in res.items():
                a = t.cpu()
                np.save(os.path.join(dump, f'{case}.{m}.npy'), (a.view(torch.int16) if a.dtype == bf else a).numpy())


if __name__ == '__main__':
    main()
