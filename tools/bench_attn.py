#!/usr/bin/env python
"""Times the bounded-logit wgmma attention kernels alone on the config-2 shape (--batch x 1024 tokens, 8 heads, two 256-token spans per sample).
TFX_LIB=<path to a libtfx_b200 build> selects a library variant (used for A/B experiments on the kernel).  --dump DIR writes o, lse (forward) and
dq, dk, dv (one backward after the prep kernel) from the seeded inputs as DIR/<tensor>.npy, so that two builds can be compared tensor by tensor."""
import argparse, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transfusion_pytorch_b200 import _lib
if os.environ.get('TFX_LIB'):
    _lib.LIB_PATH = os.environ['TFX_LIB']
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
from test_ops_gpu import make_rb

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type = int, default = 128, help = '1024-token sequences (the benchmark runs 128)')
    ap.add_argument('--dump', default = None, metavar = 'DIR', help = 'write o, lse, dq, dk, dv to DIR/*.npy')
    args = ap.parse_args()
    ops = _lib.Ops()
    B, H, cap, scale = args.batch, 8, 50., 0.125
    lens = [1024] * B
    spans = [(b, off, 256) for b in range(B) for off in (206, 668)]
    rb = make_rb(lens, spans)
    M = rb.M
    g = torch.Generator(device = 'cuda').manual_seed(1)
    unit = lambda x: (torch.nn.functional.normalize(x.reshape(M, H, 64), dim = -1) * 8.).reshape(M, H * 64).to(torch.bfloat16)
    q, k = unit(torch.randn(M, H * 64, device = 'cuda', generator = g)), unit(torch.randn(M, H * 64, device = 'cuda', generator = g))
    v = torch.randn(M, H * 64, device = 'cuda', generator = g).to(torch.bfloat16)
    gates = torch.randn(M, H, device = 'cuda', generator = g)
    dev = lambda a: torch.from_numpy(a).cuda()
    kvl = dev(rb.kv_limit)
    t2 = [dev(x) for x in (rb.t2_q0, rb.t2_qend, rb.t2_kv0, rb.t2_kvend)]
    k2 = [dev(x) for x in (rb.k2_kv0, rb.k2_kvend, rb.k2_q0, rb.k2_qend, rb.k2_order)]
    fp = torch.zeros(8, device = 'cuda'); z = torch.zeros(64, device = 'cuda')
    ops.attn_fast_params(z, z, 64, scale, cap, fp)
    o = torch.zeros(M, H * 64, device = 'cuda', dtype = torch.bfloat16); lse = torch.zeros(H, M, device = 'cuda')
    do = torch.randn(M, H * 64, device = 'cuda', generator = g).to(torch.bfloat16)
    dop = torch.zeros_like(do); dsum = torch.zeros(H, M, device = 'cuda'); dsum2 = torch.zeros(M, H, device = 'cuda')
    dq = torch.zeros(M, H * 64, device = 'cuda'); dk = torch.zeros_like(dq); dv = torch.zeros_like(o)
    def fwd(): ops.attn_fwd_tc(q, k, v, H * 64, H * 64, H * 64, gates, H, kvl, *t2, len(rb.t2_q0), o, H * 64, lse, M, 0, scale, cap, fp)
    def bwd(): ops.attn_bwd_tc(q, k, v, dop, H * 64, H * 64, H * 64, H * 64, lse, dsum, kvl, *k2, len(rb.k2_kv0), dq, dk, dv, H * 64, M, H, scale, cap, fp)
    fwd()
    ops.attn_bwd_prep(do, o, gates, dop, dsum, dsum2, dq, M, H)       # D = rowsum(dO o) and the gate-scaled dO, as the engine feeds the backward
    big = torch.empty(256 << 20, dtype = torch.uint8, device = 'cuda')
    pairs = float((rb.kv_limit.astype('int64') - rb.cu[:-1].repeat(rb.seq_lens) + 1).sum())
    flops = dict(fwd = 4.0 * pairs * 64 * H, bwd = 10.0 * pairs * 64 * H)
    for name, fn in (('fwd', fwd), ('bwd', bwd)):
        for _ in range(3): fn()
        ts = []
        for _ in range(10):
            big.zero_()                                    # flush L2
            e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        med = sorted(ts)[5]
        print(f'{os.environ.get("TFX_LIB", "default"):24s} B={B} {name:7s}: median {med:8.1f} us  min {min(ts):8.1f} us  {flops[name] / med / 1e6:7.1f} TFLOP/s algorithmic')
    if args.dump:
        os.makedirs(args.dump, exist_ok = True)
        dq.zero_(); bwd(); torch.cuda.synchronize()
        for tn, t in dict(o = o, lse = lse, dq = dq, dk = dk, dv = dv).items():
            a = t.cpu()
            np.save(os.path.join(args.dump, f'{tn}.npy'), (a.view(torch.int16) if a.dtype == torch.bfloat16 else a).numpy())
if __name__ == '__main__':
    main()
