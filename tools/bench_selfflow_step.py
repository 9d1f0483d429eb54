#!/usr/bin/env python
"""Cost of Self-Flow training: config 2 (d 512, depth 8, 1024-token samples) eager training steps - forward, backward, torch.optim.Adam - of the
plain model against the same model wrapped in `SelfMaskedRepTraining` (defaults: student layer -3, teacher layer -1, no asymmetric dropout,
which needs `use_flex_attn`), with `update_teacher()` after each wrapped step.  The two arms share one model and alternate round by round in
one process.  Prints the card, its power limit and the median and minimum step time per round and batch size."""
import argparse, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transfusion_pytorch_b200 import Transfusion, SelfMaskedRepTraining, synth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type = int, nargs = '+', default = [32, 128])
    ap.add_argument('--steps', type = int, default = 8)
    ap.add_argument('--rounds', type = int, default = 5)
    args = ap.parse_args()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output = True, text = True).stdout.strip()
    print(f'card: {q}')
    torch.manual_seed(0)
    model = Transfusion(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), transformer = dict(dim = 512, depth = 8)).cuda()
    synth.fill_parameters_(model, seed = 0)
    wrapper = SelfMaskedRepTraining(model, use_asymmetric_dropout = False).cuda().train()
    opt = torch.optim.Adam(wrapper.parameters(), lr = 1e-5)

    def plain(batch, times):
        loss = model(batch, times = times)
        loss.backward()
        opt.step(); opt.zero_grad()

    def wrapped(batch, times):
        loss, _ = wrapper(batch, times = times)
        loss.backward()
        opt.step(); opt.zero_grad()
        wrapper.update_teacher()

    for B in args.batch:
        batch, times = synth.config2_batch(B, seed = 1), synth.config2_times(B, seed = 1)
        for fn in (plain, wrapped, plain, wrapped):         # warm-up: workspaces, algorithm choices
            fn(batch, times)
        torch.cuda.synchronize()
        for r in range(args.rounds):
            for name, fn in (('plain', plain), ('self-flow', wrapped)):
                ts = []
                for _ in range(args.steps):
                    e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
                    e0.record(); fn(batch, times); e1.record(); torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1))
                ts.sort()
                print(f'round {r} batch {B} {name}: median {ts[len(ts) // 2]:.2f} ms  min {ts[0]:.2f} ms  ({args.steps} steps)', flush = True)


if __name__ == '__main__':
    main()
