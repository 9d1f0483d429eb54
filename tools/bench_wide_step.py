#!/usr/bin/env python
"""Training-step cost at model widths 1536 and 2048: the resident step bench.py times (`DataParallelTrainer.step_packed`, CUDA-graph replay) on
config-2-style batches (1024-token samples), each shape in a process of its own and the shapes alternated round by round; and, from one eager step
under torch.profiler, the time of the row-kernel family (the kernels of rowops.cu that TFX_DISPATCH_NCH instantiates per width) with the achieved
HBM rate of the kernels whose traffic is fixed by the shapes.  The bytes are what the algorithm has to move, counted below; the AttentionResidual
bytes are tools/bench_depth.py's.  Prints the card, its power limit and max SM clock first, and the peak device memory of each shape.

    python tools/bench_wide_step.py                     # 1536 x depth 16 x 4 samples, 2048 x depth 8 x 2 samples; plus 1024 x 24 x 6 as the anchor
    python tools/bench_wide_step.py --shapes 2048x8x2   # width x depth x batch"""
import argparse, os, subprocess, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from bench_depth import arm, ares_bytes_per_token       # noqa: E402

DEFAULT = '1024x24x6,1536x16x4,2048x8x2'
ROW_KERNELS = ('adaln_fwd_k', 'adaln_bwd_k', 'resid_bwd_k', 'rmsnorm_fwd_k', 'rmsnorm_bwd_k', 'attn_res_fwd_k', 'attn_res_bwd2_k', 'attn_res_bwd_finish_k',
               'embed_assemble_k', 'embed_bwd_k', 'scatter_add_rows_k', 'clean_flow_fwd_k', 'clean_flow_bwd_k', 'rep_cos_fwd_bwd_k')


def row_bytes(name, D):
    """HBM bytes per token row of one launch (None: traffic depends on the call's options)"""
    return {'adaln_fwd_k': 4 * D + 2 * D + 8,            # x fp32 in, u bf16 out, mean / rstd
            'adaln_bwd_k': 4 * D + 4 * D + 8 * D + 8,    # du, x in; dx read-modify-write; stats
            'resid_bwd_k': 4 * D + 2 * D + 2 * D,        # dx fp32, y bf16 in; dy bf16 out
            'rmsnorm_bwd_k': 4 * D + 4 * D + 4 * D}.get(name)


def eager_profile(trainer, rb, lat, M, D, depth):
    trainer.cuda_graph = False
    trainer.step_packed(rb, lat)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities = [torch.profiler.ProfilerActivity.CUDA]) as prof:
        trainer.step_packed(rb, lat)
        torch.cuda.synchronize()
    fam, calls, total = {}, {}, 0.
    for e in prof.key_averages():
        t = e.device_time_total / 1e3 if hasattr(e, 'device_time_total') else e.cuda_time_total / 1e3
        total += t
        for k in ROW_KERNELS:
            if k + '<' in e.key or e.key.startswith(k) or ('::' + k) in e.key:
                fam[k] = fam.get(k, 0.) + t
                calls[k] = calls.get(k, 0) + e.count
                break
    trainer.cuda_graph = True
    fwd_b, bwd_b = ares_bytes_per_token(D, depth)
    rates = {}
    for k, t in fam.items():
        rb_ = row_bytes(k, D)
        if rb_ is not None and t > 0:
            rates[k] = rb_ * M * calls[k] / t / 1e6
    if fam.get('attn_res_fwd_k'):
        rates['attn_res_fwd_k'] = fwd_b * M / fam['attn_res_fwd_k'] / 1e6
    bwd_t = fam.get('attn_res_bwd2_k', 0.) + fam.get('attn_res_bwd_finish_k', 0.)
    if bwd_t:
        rates['attn_res_bwd'] = bwd_b * M / bwd_t / 1e6
    return fam, calls, rates, total


def one(spec, steps, r):
    D, depth, B = (int(v) for v in spec.split('x'))
    torch.cuda.reset_peak_memory_stats()
    model, trainer, rb, lat = arm(D, depth, B)
    M = rb.M
    for _ in range(4):                                   # two eager steps, the capture, one replay
        trainer.step_packed(rb, lat)
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
        e0.record(); trainer.step_packed(rb, lat); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    med = ts[len(ts) // 2]
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    params = sum(p.numel() for p in model.parameters())
    print(f'round {r}  d {D:5d} depth {depth:3d} tokens {M:6d} ({params / 1e9:.2f} B parameters): step median {med:8.2f} ms (min {ts[0]:.2f}, '
          f'{steps} replays)  {M / med * 1e3:9.0f} tok/s  peak {peak:.1f} GiB', flush = True)
    if r == 0:
        fam, calls, rates, total = eager_profile(trainer, rb, lat, M, D, depth)
        row = sum(fam.values())
        print(f'  eager step: kernels {total:.2f} ms, row kernels {row:.2f} ms ({100 * row / total:.1f} %)')
        for k in ROW_KERNELS:
            if k in fam:
                rate = f'  {rates[k]:6.0f} GB/s' if k in rates else ''
                print(f'    {k:24s} {fam[k]:8.3f} ms / {calls[k]:4d} launches{rate}')
        if 'attn_res_bwd' in rates:
            print(f'    {"AttentionResidual bwd":24s} (bwd2 + fold) {rates["attn_res_bwd"]:6.0f} GB/s')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default = DEFAULT, help = 'comma-separated width x depth x batch (1024-token samples)')
    ap.add_argument('--steps', type = int, default = 10)
    ap.add_argument('--rounds', type = int, default = 2)
    ap.add_argument('--one', default = None, help = 'run one shape in this process (used by the alternation)')
    ap.add_argument('--round', type = int, default = 0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_wide_step.py times the H100 path: it needs a GPU'
    if args.one is not None:
        return one(args.one, args.steps, args.round)
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output = True, text = True).stdout.strip()
    print(f'card (name, power limit, max SM clock): {q}', flush = True)
    for r in range(args.rounds):
        for spec in args.shapes.split(','):
            subprocess.run([sys.executable, os.path.abspath(__file__), '--one', spec, '--round', str(r), '--steps', str(args.steps)], check = True)


if __name__ == '__main__':
    main()
