#!/usr/bin/env python
"""Cost of `dim_head = 128` in the resident training step: config 2 (d 512, depth 8, 1024-token samples) at --batch 128 on the path bench.py
times (`DataParallelTrainer.step_packed`, CUDA-graph replay), with heads = 4 x dim_head 128 against heads = 8 x dim_head 64 (the same inner
width 512 and the same FLOPs), alternated round by round; each arm runs in a process of its own, so its device memory is returned before the
other starts.  At dim_head 128 every layer runs the general running-maximum attention kernels (there is no bounded-logit wgmma kernel for
it).  Also times, per entry point, the attention-related kernels of one eager step of each arm (CUDA events around every launch).  Prints the
card, its power limit and SM clocks, the median / minimum step time per round and arm, and the per-kernel totals."""
import argparse, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transfusion_pytorch_b200 import Transfusion, synth
from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
from transfusion_pytorch_b200.modality_processing import pack_batch

KERNELS = ('attn_fast_params', 'attn_fwd_tc', 'attn_fwd', 'attn_fwd_d128', 'attn_bwd_tc', 'attn_bwd', 'attn_bwd_d128', 'attn_bwd_prep', 'attn_bwd_prep_d128',
           'gemm_qkvg', 'gemm_qkvg_d128', 'qk_bwd_pack', 'qk_bwd_pack_d128')
ARMS = {'d128': dict(heads = 4, dim_head = 128), 'd64': dict(heads = 8, dim_head = 64)}


def arm(name, B, seed = 0):
    ctor = dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), transformer = dict(dim = 512, depth = 8, **ARMS[name]))
    torch.manual_seed(0)
    model = Transfusion(**ctor).cuda()
    synth.fill_parameters_(model, seed = seed)
    model.train()
    trainer = DataParallelTrainer(model, lr = 1e-4, cuda_graph = True)
    model.engine.ensure_attached()
    batch, times = synth.config2_batch(B, seed = 1), synth.config2_times(B, seed = 1)
    samples = [[torch.tensor([model.sos_id]), *s, torch.tensor([model.eos_id])] for s in batch]
    rb = pack_batch(samples, times, model, return_loss = True, return_embed = False)
    lat = model._latents_to_device(rb)
    model.engine.upload(rb)
    for _ in range(4):                               # two eager steps, the capture, one replay
        trainer.step_packed(rb, lat)
    torch.cuda.synchronize()
    return model, trainer, rb, lat


def kernel_times(model, trainer, rb, lat):
    """ms per entry point (summed over the step's launches) of one eager step"""
    ops = model.engine.ops
    ops.timing = {}
    trainer.step_packed_eager(rb, lat)
    torch.cuda.synchronize()
    t = {n: sum(e0.elapsed_time(e1) for e0, e1, _ in calls) for n, calls in ops.timing.items()}
    n = {n: len(calls) for n, calls in ops.timing.items()}
    ops.timing = None
    return t, n


def one(name, batch, steps, r, kernels):
    model, trainer, rb, lat = arm(name, batch)
    ts = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
        e0.record(); trainer.step_packed(rb, lat); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    q = subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())], capture_output = True, text = True).stdout.strip()
    print(f'round {r} {name} ({ARMS[name]}): median {ts[len(ts) // 2]:.2f} ms  min {ts[0]:.2f} ms  ({steps} replayed steps, batch {batch}; SM clock after: {q})')
    if kernels:
        t, n = kernel_times(model, trainer, rb, lat)
        print(f'  eager step, {name}: ' + '  '.join(f'{k} {t[k]:.2f} ms / {n[k]}' for k in KERNELS if k in t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type = int, default = 128)
    ap.add_argument('--steps', type = int, default = 10)
    ap.add_argument('--rounds', type = int, default = 2)
    ap.add_argument('--arm', default = None, choices = list(ARMS), help = 'run one arm in this process (used by the alternation)')
    ap.add_argument('--round', type = int, default = 0)
    args = ap.parse_args()
    if args.arm is not None:
        return one(args.arm, args.batch, args.steps, args.round, kernels = args.round == 0)
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output = True, text = True).stdout.strip()
    print(f'card (name, power limit, max SM clock): {q}', flush = True)
    for r in range(args.rounds):
        for a in ARMS:
            subprocess.run([sys.executable, os.path.abspath(__file__), '--arm', a, '--round', str(r), '--batch', str(args.batch), '--steps', str(args.steps)], check = True)


if __name__ == '__main__':
    main()
