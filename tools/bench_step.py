#!/usr/bin/env python
"""Cost of model options in the resident training step, on the path bench.py times (`DataParallelTrainer.step_packed`, CUDA-graph replay).
Each positional argument is one arm, WIDTHxDEPTHxBATCH[:key=value,...] with BATCH in 1024-token samples; the keys are `dim_head` (default 64),
`heads` (default width // dim_head), `qk_rmsnorm` (0 / 1), `gated` (0 / 1: `attn_kwargs = dict(gate_values = ...)`), `vres` (0 / 1:
`use_value_residual`), `dropout` (`ff_kwargs = dict(dropout = p)`), `recon` (`reconstruction_loss_weight`) and `data` (config2, the default,
or config4).  Each arm runs in a process of its own, so its device memory is returned before the next
starts, and the arms alternate in the order given for --rounds rounds.  Prints the card, its power limit and max SM clock once, then per arm
the median and minimum step time of --steps replays, tokens, tokens/s, peak device memory and the SM clock after the arm.

--kernels adds, in round 0, one eager step with CUDA events around every entry-point launch (`Ops.timing`): each entry point's summed time and
launch count, and the achieved HBM rate of those whose traffic is fixed by the shapes (the bytes the algorithm moves, counted by `row_bytes`
and `ares_bytes_per_token` below, over event time).  A launch shorter than the host's time per call (few tokens) is timed at that host
time, so there the ms are upper bounds and the GB/s lower bounds.

    python tools/bench_step.py 512x8x128 512x8x128:qk_rmsnorm=0 --kernels
    python tools/bench_step.py 512x8x128 512x8x128:gated=0 2048x8x16:heads=32 2048x8x16:heads=32,vres=1
    python tools/bench_step.py 512x8x128:data=config4 512x8x128:data=config4,recon=0.1"""
import argparse, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transfusion_pytorch_b200 import Transfusion, synth
from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
from transfusion_pytorch_b200.modality_processing import pack_batch

KEYS = ('dim_head', 'heads', 'qk_rmsnorm', 'gated', 'vres', 'dropout', 'recon', 'data')
DATA = {'config2': dict(dim_latent = 384, modality_default_shape = (256,)),
        'config4': dict(dim_latent = (384, 192), modality_default_shape = ((4,), (2,)))}
CHUNK = 10                    # later layers per deferred-assembly launch (rowops.cu BWD2_CHUNK)
ARES = {'attn_residual_fwd_h16': 0, 'attn_residual_bwd2': 1}      # which of ares_bytes_per_token's (fwd, bwd) the entry point's launches move


def parse_arm(spec):
    """'WIDTHxDEPTHxBATCH[:key=value,...]' -> (Transfusion kwargs, batch kind, batch size in samples); needs no GPU"""
    shape, _, opts = spec.partition(':')
    D, depth, B = (int(v) for v in shape.split('x'))
    kv = dict(o.split('=', 1) for o in opts.split(',')) if opts else {}
    if set(kv) - set(KEYS):
        raise ValueError(f'{spec}: unknown key(s) {sorted(set(kv) - set(KEYS))}; the keys are {", ".join(KEYS)}')
    dim_head = int(kv.get('dim_head', 64))
    tr = dict(dim = D, depth = depth, dim_head = dim_head, heads = int(kv.get('heads', D // dim_head)))
    for key in ('qk_rmsnorm', 'gated', 'vres'):
        if key in kv and kv[key] not in ('0', '1'):
            raise ValueError(f'{spec}: {key} is 0 or 1')
    if 'qk_rmsnorm' in kv:
        tr['qk_rmsnorm'] = kv['qk_rmsnorm'] == '1'
    if 'gated' in kv:
        tr['attn_kwargs'] = dict(gate_values = kv['gated'] == '1')
    if 'vres' in kv:
        tr['use_value_residual'] = kv['vres'] == '1'
    if 'dropout' in kv:
        tr['ff_kwargs'] = dict(dropout = float(kv['dropout']))
    data = kv.get('data', 'config2')
    if data not in DATA:
        raise ValueError(f'{spec}: data is one of {", ".join(DATA)}')
    ctor = dict(num_text_tokens = 256, **DATA[data], transformer = tr)
    if 'recon' in kv:
        ctor['reconstruction_loss_weight'] = float(kv['recon'])
    return ctor, data, B


def row_bytes(name, D):
    """HBM bytes per token row of one launch (None: traffic depends on the call's options)"""
    return {'adaln_fwd': 4 * D + 2 * D + 8,              # x fp32 in, u bf16 out, mean / rstd
            'adaln_bwd': 4 * D + 4 * D + 8 * D + 8,      # du, x in; dx read-modify-write; stats
            'resid_bwd': 4 * D + 2 * D + 2 * D,          # dx fp32, y bf16 in; dy bf16 out
            'rmsnorm_bwd': 4 * D + 4 * D + 4 * D}.get(name)


def ares_bytes_per_token(D, L):
    """HBM bytes per token of the AttentionResidual kernels of one train step (bf16 hiddens, deferred backward)"""
    fwd = sum((i + 2) * 2 * D + 4 * D + 2 * D + 4 for i in range(L))                      # hiddens in; x_out fp32 + bf16, lse out
    bwd = 0
    for i in range(L):
        n_later = L - 1 - i
        extra = max(0, -(-n_later // CHUNK) - 1)                                         # further chunks re-read h and read-modify-write G
        bwd += 4 + 12 * n_later + 8 * D + (i + 2) * 2 * D + n_later * 4 * D + 4 * D + 12 * (i + 1) + extra * (2 * D + 8 * D)
    extra0 = max(0, -(-L // CHUNK) - 1)
    bwd += 12 * L + 2 * D + L * 4 * D + 4 * D + extra0 * (2 * D + 8 * D)                  # x0 assembly
    return fwd, bwd


def step_bytes(name, D, depth, M, launches):
    """HBM bytes all launches of one entry point move in a step of M tokens (None: traffic depends on the call's options)"""
    if name in ARES:
        return ares_bytes_per_token(D, depth)[ARES[name]] * M
    b = row_bytes(name, D)
    return None if b is None else b * M * launches


def smi(query):
    return subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                          capture_output = True, text = True).stdout.strip()


def kernel_times(model, trainer, rb, lat, D, depth):
    """one eager step with events around every launch: print each entry point's summed ms, launches, share and, where fixed, GB/s"""
    ops = model.engine.ops
    ops.timing = {}
    e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
    e0.record(); trainer.step_packed_eager(rb, lat); e1.record(); torch.cuda.synchronize()
    rows = sorted(((sum(a.elapsed_time(b) for a, b, _ in calls), len(calls), name) for name, calls in ops.timing.items()), reverse = True)
    ops.timing = None
    total = sum(t for t, _, _ in rows)
    print(f'  eager step {e0.elapsed_time(e1):.2f} ms; timed entry points {total:.2f} ms ({100 * total / e0.elapsed_time(e1):.1f} % of it):')
    for t, n, name in rows:
        by = step_bytes(name, D, depth, rb.M, n)
        print(f'    {name:28s} {t:8.3f} ms / {n:4d} launches {100 * t / total:5.1f} %' + (f'  {by / t / 1e6:6.0f} GB/s' if by else ''))


def run_arm(spec, steps, r, kernels):
    ctor, data, B = parse_arm(spec)
    torch.manual_seed(0)
    model = Transfusion(**ctor).cuda()
    synth.fill_parameters_(model, seed = 0)
    model.train()
    trainer = DataParallelTrainer(model, lr = 1e-4, cuda_graph = True)
    model.engine.ensure_attached()
    if data == 'config2':
        batch, times = synth.config2_batch(B, seed = 1), synth.config2_times(B, seed = 1)
    else:
        batch = synth.config4_batch(B, seed = 1)
        nm = max(sum(isinstance(p, tuple) for p in s) for s in batch)
        times = torch.rand(B, nm, generator = torch.Generator().manual_seed(1))
    samples = [[torch.tensor([model.sos_id]), *s, torch.tensor([model.eos_id])] for s in batch]
    rb = pack_batch(samples, times, model, return_loss = True, return_embed = False)
    lat = model._latents_to_device(rb)
    model.engine.upload(rb)
    for _ in range(4):                                   # two eager steps, the capture, one replay
        trainer.step_packed(rb, lat)
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
        e0.record(); trainer.step_packed(rb, lat); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    med, M = ts[len(ts) // 2], rb.M
    print(f'round {r} {spec}: median {med:.2f} ms  min {ts[0]:.2f} ms ({steps} replays)  tokens {M}  {M / med * 1e3:.0f} tok/s  '
          f'peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB  SM clock after: {smi("clocks.sm")}', flush = True)
    if kernels:
        kernel_times(model, trainer, rb, lat, ctor['transformer']['dim'], ctor['transformer']['depth'])


def main():
    ap = argparse.ArgumentParser(description = __doc__, formatter_class = argparse.RawDescriptionHelpFormatter)
    ap.add_argument('arms', nargs = '*', metavar = 'ARM', help = 'WIDTHxDEPTHxBATCH[:key=value,...]')
    ap.add_argument('--steps', type = int, default = 10)
    ap.add_argument('--rounds', type = int, default = 2)
    ap.add_argument('--kernels', action = 'store_true', help = 'per-entry-point times of one eager step, in round 0')
    ap.add_argument('--one', default = None, metavar = 'ARM', help = 'run one arm in this process (used by the alternation)')
    ap.add_argument('--round', type = int, default = 0)
    args = ap.parse_args()
    for spec in args.arms + ([args.one] if args.one else []):
        parse_arm(spec)
    if not args.arms and args.one is None:
        ap.error('give at least one arm')
    assert torch.cuda.is_available(), 'bench_step.py times the H100 path: it needs a GPU'
    if args.one is not None:
        return run_arm(args.one, args.steps, args.round, args.kernels and args.round == 0)
    print(f'card (name, power limit, max SM clock): {smi("name,power.limit,clocks.max.sm")}', flush = True)
    for r in range(args.rounds):
        for spec in args.arms:
            subprocess.run([sys.executable, os.path.abspath(__file__), '--one', spec, '--round', str(r), '--steps', str(args.steps)]
                           + ['--kernels'] * args.kernels, check = True)


if __name__ == '__main__':
    main()
