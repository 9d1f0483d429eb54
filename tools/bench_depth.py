#!/usr/bin/env python
"""Training-step cost of deeper models: the resident step bench.py times (`DataParallelTrainer.step_packed`, CUDA-graph replay) on config-2-style
batches (1024-token samples, one 256-row modality per sample) at several (width, depth) pairs, and, from one eager step under torch.profiler, the time
of the AttentionResidual kernel family (forward, deferred backward, parameter-gradient fold) with its achieved HBM rate.  The bytes are what the
algorithm has to move, counted from shapes by `ares_bytes_per_token` below.  Prints the card and its power limit first.

    python tools/bench_depth.py                   # the default list: (512, 8) as the anchor, (512, 16), (768, 12), (1024, 24), (1024, 32)
    python tools/bench_depth.py --shapes 512x8x32 # width x depth x batch (1024-token samples)"""
import argparse, gc, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transfusion_pytorch_b200 import Transfusion, synth
from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
from transfusion_pytorch_b200.modality_processing import pack_batch

DEFAULT = '512x8x64,512x16x64,768x12x32,1024x24x6,1024x32x4'
CHUNK = 10                    # later layers per deferred-assembly launch (rowops.cu BWD2_CHUNK)


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


def arm(D, depth, B):
    ctor = dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), transformer = dict(dim = D, depth = depth, heads = D // 64))
    batch, times = synth.config2_batch(B, seed = 1), synth.config2_times(B, seed = 1)
    torch.manual_seed(0)
    model = Transfusion(**ctor).cuda()
    synth.fill_parameters_(model, seed = 0)
    model.train()
    trainer = DataParallelTrainer(model, lr = 1e-4, cuda_graph = True)
    model.engine.ensure_attached()
    samples = [[torch.tensor([model.sos_id]), *s, torch.tensor([model.eos_id])] for s in batch]
    rb = pack_batch(samples, times, model, return_loss = True, return_embed = False)
    lat = model._latents_to_device(rb)
    model.engine.upload(rb)
    return model, trainer, rb, lat


def eager_profile(model, trainer, rb, lat):
    """one eager step (outside the graph) under the profiler: AttentionResidual family time and the whole step's kernel time, in ms"""
    trainer.cuda_graph = False
    trainer.step_packed(rb, lat)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities = [torch.profiler.ProfilerActivity.CUDA]) as prof:
        trainer.step_packed(rb, lat)
        torch.cuda.synchronize()
    fam = {'fwd': 0., 'bwd': 0.}
    total = 0.
    for e in prof.key_averages():
        t = e.device_time_total / 1e3 if hasattr(e, 'device_time_total') else e.cuda_time_total / 1e3
        total += t
        if 'attn_res_fwd_k' in e.key:
            fam['fwd'] += t
        elif 'attn_res_bwd' in e.key:
            fam['bwd'] += t
    trainer.cuda_graph = True
    return fam, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default = DEFAULT, help = 'comma-separated width x depth x batch')
    ap.add_argument('--steps', type = int, default = 10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_depth.py times the H100 path: it needs a GPU'
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output = True, text = True).stdout.strip()
    print(f'card: {q}')
    for spec in args.shapes.split(','):
        D, depth, B = (int(v) for v in spec.split('x'))
        torch.cuda.reset_peak_memory_stats()
        model, trainer, rb, lat = arm(D, depth, B)
        M = rb.M
        for _ in range(4):                               # two eager steps, the capture, one replay
            trainer.step_packed(rb, lat)
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.steps):
            e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
            e0.record(); trainer.step_packed(rb, lat); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        med = ts[len(ts) // 2]
        fam, total = eager_profile(model, trainer, rb, lat)
        bf, bb = ares_bytes_per_token(D, depth)
        ares = fam['fwd'] + fam['bwd']
        print(f'd {D:5d} depth {depth:3d} tokens {M:6d}: step {med:8.2f} ms (min {ts[0]:.2f})  {M / med * 1e3:10.0f} tok/s  |  eager kernels {total:8.2f} ms, '
              f'AttentionResidual {ares:7.2f} ms ({100 * ares / total:4.1f} %): fwd {fam["fwd"]:6.2f} ms {bf * M / fam["fwd"] / 1e6:6.0f} GB/s, '
              f'bwd {fam["bwd"]:6.2f} ms {bb * M / fam["bwd"] / 1e6:6.0f} GB/s  (fwd {bf / 1e6:.2f} MB/token, bwd {bb / 1e6:.2f} MB/token), '
              f'peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB', flush = True)
        del model, trainer, rb, lat
        gc.collect()                                     # the engine and the captured graph hold reference cycles
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
