#!/usr/bin/env python
"""Cost of the reconstruction loss in the resident training step, on the path bench.py times (`DataParallelTrainer.step_packed`, CUDA-graph
replay): config 2 (d 512, depth 8, one modality type, 1024-token samples) or config 4 (two modality types, many short spans) at --batch 128
with `reconstruction_loss_weight = --weight`.  bench.py's own model has no reconstruction loss; run this with --weight 0 and --weight 0.1
alternately to compare.  Prints the card, its power limit and the median and minimum step time of each of --rounds rounds."""
import argparse, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transfusion_pytorch_b200 import Transfusion, synth
from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
from transfusion_pytorch_b200.modality_processing import pack_batch


def arm(config, w_r, B, seed = 0):
    tr = dict(dim = 512, depth = 8)
    if config == 2:
        ctor = dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), transformer = tr)
        batch, times = synth.config2_batch(B, seed = 1), synth.config2_times(B, seed = 1)
    else:
        ctor = dict(num_text_tokens = 256, dim_latent = (384, 192), modality_default_shape = ((4,), (2,)), transformer = tr)
        batch = synth.config4_batch(B, seed = 1)
        nm = max(sum(isinstance(p, tuple) for p in s) for s in batch)
        times = torch.rand(B, nm, generator = torch.Generator().manual_seed(1))
    torch.manual_seed(0)
    model = Transfusion(**ctor, reconstruction_loss_weight = w_r).cuda()
    synth.fill_parameters_(model, seed = seed)
    model.train()
    trainer = DataParallelTrainer(model, lr = 1e-4, cuda_graph = True)
    model.engine.ensure_attached()
    samples = [[torch.tensor([model.sos_id]), *s, torch.tensor([model.eos_id])] for s in batch]
    rb = pack_batch(samples, times, model, return_loss = True, return_embed = False)
    lat = model._latents_to_device(rb)
    model.engine.upload(rb)
    for _ in range(4):                               # two eager steps, the capture, one replay
        trainer.step_packed(rb, lat)
    torch.cuda.synchronize()
    return lambda: trainer.step_packed(rb, lat)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', type = int, choices = (2, 4), default = 2)
    ap.add_argument('--weight', type = float, default = 0.1)
    ap.add_argument('--batch', type = int, default = 128)
    ap.add_argument('--steps', type = int, default = 10)
    ap.add_argument('--rounds', type = int, default = 2)
    args = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output = True, text = True).stdout.strip()
    print(f'card: {q}')
    step = arm(args.config, args.weight, args.batch)
    for r in range(args.rounds):
        ts = []
        for _ in range(args.steps):
            e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
            e0.record(); step(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        print(f'round {r} config {args.config} recon weight {args.weight:.2f}: median {ts[len(ts) // 2]:.2f} ms  min {ts[0]:.2f} ms  ({args.steps} steps, batch {args.batch})')

if __name__ == '__main__':
    main()
