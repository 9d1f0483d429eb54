"""GPU: model widths 1536 and 2048 (NCH 12 and 16 of TFX_DISPATCH_NCH) end to end.

- Every row-kernel entry point at both widths against float64, through the per-kernel tests of the narrower widths (same inputs, row counts and
  bounds; their width lists stop at 1024): adaLN forward / backward with and without condition rows, the branch-gate backward, final RMSNorm
  forward / backward, token assemble / embedding backward / scatter-add / clean-flow rows, the Self-Flow cosine loss, and the
  AttentionResidual forward and deferred backward at depths that cross the 10-layer chunks of the backward assembly.
- The fused GEMM epilogues and the GEGLU backward at both widths against float64, through the bodies of tests/test_block_epilogues_gpu.py
  (same row count and bounds, the accumulator bound grown with the k-loop as helpers.c_acc states): gemm_resid in its attention-out,
  text-only, FFN-out, bf16-only and U-Net skip forms, whose FFN-out and skip products run 48 to 86 k-blocks over 12 and 16 N tiles, at HI
  below D (8 heads) and HI = D (32 heads); gemm_geglu with and without dropout over 64 and 86 value / gate tile pairs; geglu_bwd with and
  without dropout at 512 and 704 threads per block, with the colsum_f32 bias sums.
- Whole training steps against the reference's own outputs (oracle/make_golden_wide.py) at the parity bounds of tests/test_parity_gpu.py, the
  sampler against the reference under the greedy-margin rule, the captured `step_packed` graph against the eager step, and `torch.optim.Adam`
  steps against the fp32 checker."""
import copy

import pytest
import torch

import test_attn_residual_gpu as ares
import test_aux_kernels_gpu as aux
import test_block_epilogues_gpu as epi
import test_norm_kernels_gpu as norm
import test_selfflow_gpu as selfflow
from helpers import cluster_mode, compare_sampling, golden_noise, grad_fingerprint, load_golden, unpack_rows  # noqa: F401  (cluster_mode: a fixture)
from transfusion_pytorch_b200 import Transfusion, _lib, synth
from transfusion_pytorch_b200.transfusion import MODEL_DIMS
from oracle.dh128_reference import HeadDimOracleEngine

pytestmark = pytest.mark.gpu
WIDE = (1536, 2048)
EPI_CONFIGS = [(1536, 8), (2048, 32)]                    # (D, H): HI = 64 H below D and equal to D
# Measured on an H100 80GB HBM3 (700 W power limit), worst err / bound of the fused-epilogue checks at both widths: bf16 outputs 0.984 - 0.996
# (the cast's rounding, which the bound states exactly); gemm_resid x_out 0.18 - 0.38 (the accumulator at 64 and 86 k-blocks: 7.0e-7 and
# 7.4e-7 of |u| |W|^T); geglu_bwd dbias 0.012 - 0.014.  Per case: gemm_resid 0.1 s and +1.4 / +2.0 GiB of device memory at D = 1536 / 2048,
# gemm_geglu 3.0 - 3.7 s and +4.3 / +5.8 GiB (its float64 reference in two row chunks), geglu_bwd 3.2 / 3.7 s and +6.4 / +8.6 GiB.
LOSS_REL, HID_REL, GRAD_REL = 1e-3, 2e-2, 6e-2           # tests/test_parity_gpu.py
MARGIN_BOUND, LATENT_TOL = 0.1, 5e-2                     # tests/test_dh128_gpu.py


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


def test_wide_widths_are_dispatched():
    assert set(WIDE) <= set(MODEL_DIMS)


# ------------------------------------------------------------------------------------------------ row kernels vs float64
@pytest.mark.parametrize('D', WIDE)
def test_adaln_fwd_vs_float64(ops, D):
    norm.test_adaln_fwd_vs_float64(ops, D)


@pytest.mark.parametrize('D', WIDE)
def test_adaln_bwd_vs_float64(ops, D):
    norm.test_adaln_bwd_vs_float64(ops, D)


@pytest.mark.parametrize('D', WIDE)
def test_resid_bwd_vs_float64(ops, D):
    epi.test_resid_bwd_vs_float64(ops, D)


@pytest.mark.parametrize('D', WIDE)
def test_rmsnorm_fwd_vs_float64(ops, D):
    norm.test_rmsnorm_fwd_vs_float64(ops, D)


@pytest.mark.parametrize('D', WIDE)
def test_rmsnorm_bwd_vs_float64(ops, D):
    norm.test_rmsnorm_bwd_vs_float64(ops, D)


@pytest.mark.parametrize('D', WIDE)
def test_embed_bwd_vs_float64(ops, D):
    norm.test_embed_bwd_vs_float64(ops, D)


@pytest.mark.parametrize('D', WIDE)
def test_embed_scatter_clean_flow(ops, D):
    aux.test_embed_scatter_clean_flow(ops, D)


@pytest.mark.parametrize('D', WIDE)
def test_rep_cos_kernel_against_float64(ops, D):
    selfflow.test_rep_cos_kernel_against_float64(ops, D)


@pytest.mark.parametrize('D', WIDE)
@pytest.mark.parametrize('L1', [1, 10, 11, 21, 65])
def test_attn_residual_fwd_vs_float64(ops, D, L1):
    ares.test_attn_residual_fwd_vs_float64(ops, D, L1)


@pytest.mark.parametrize('D', WIDE)
@pytest.mark.parametrize('depth', [1, 10, 11, 21, 64])
def test_attn_residual_backward_vs_float64(ops, D, depth):
    ares.test_attn_residual_backward_vs_float64(ops, D, depth)


# ------------------------------------------------------------------------------------------------ fused GEMM epilogues vs float64
@pytest.mark.parametrize('D,H', EPI_CONFIGS, ids = [f'd{d}h{h}' for d, h in EPI_CONFIGS])
def test_gemm_resid_vs_float64(ops, cluster_mode, D, H):
    epi.test_gemm_resid_vs_float64(ops, cluster_mode, D, H, False)


@pytest.mark.parametrize('D,H', EPI_CONFIGS, ids = [f'd{d}h{h}' for d, h in EPI_CONFIGS])
def test_gemm_geglu_vs_float64(ops, cluster_mode, D, H):
    epi.test_gemm_geglu_vs_float64(ops, cluster_mode, D, H, False)


@pytest.mark.parametrize('D', WIDE)
def test_geglu_bwd_vs_float64(ops, D):
    epi.test_geglu_bwd_vs_float64(ops, D)


# ------------------------------------------------------------------------------------------------ whole model
def build(ctor, seed, dev = 'cuda'):
    torch.manual_seed(0)
    model = Transfusion(**ctor)
    synth.fill_parameters_(model, seed = seed)
    model = model.to(dev).eval()
    if dev == 'cpu':
        model._engine = HeadDimOracleEngine(model)
    return model


def rel_max(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp(min = 1e-9)).item()


def check_grads(model, fx):
    fp = grad_fingerprint((n, p.grad) for n, p in model.named_parameters() if p.grad is not None)
    assert set(fx['grads']) <= set(fp)
    for k, v in fx['grads'].items():
        ref_n = max(v['stats'][3].item(), 1e-12)
        assert abs(fp[k]['stats'][2].item() - v['stats'][2].item()) / ref_n < GRAD_REL, k
        assert abs(fp[k]['stats'][3].item() - v['stats'][3].item()) / ref_n < GRAD_REL, k


def two_type_batch():
    return synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)


@pytest.mark.parametrize('name', ['small_wide1536', 'small_wide2048', 'small_wide2048_laser_vres'])
def test_train_step_matches_reference(name):
    """the reference's own outputs: loss, breakdown, hidden states, gradient fingerprints"""
    fx = load_golden(name)
    model = build(fx['ctor'], fx['seed'])
    batch = two_type_batch()
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = golden_noise(fx, batch, model.dim_latents))
    rb = model._last_batch
    assert rb.modality_positions == fx['modality_positions'] and rb.total_tokens == fx['total_tokens']
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < LOSS_REL
    assert abs(bd.text.item() - fx['text_loss'].item()) / fx['text_loss'].item() < LOSS_REL
    assert all(abs(a.item() - b.item()) / b.item() < LOSS_REL for a, b in zip(bd.flow, fx['flow_losses']))
    st = model.engine.state
    rows = fx['hidden_rows']
    cols = fx['hidden_cols']
    for l, h in enumerate(fx['hiddens'] + [fx['embed']]):
        ours = unpack_rows(st['hid'][l] if l < len(fx['hiddens']) else st['out'], rb)
        for b in range(rb.B):
            k = rows < int(rb.seq_lens[b])
            assert rel_max(ours[b, rows[k]][:, cols], h[b, k]) < HID_REL, f'hidden {l} sample {b}'
    loss.backward()
    assert sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is None) == fx['no_grad']
    check_grads(model, fx)


def test_sample_many_matches_reference():
    fx = load_golden('sampling_wide2048')
    model = build(fx['ctor'], fx['seed'])
    out = model.sample_many(copy.deepcopy(fx['prompts']), init_modality_noise = fx['noise'], **fx['kw'])
    rep = compare_sampling(model, out, fx, bound = MARGIN_BOUND, lat_tol = LATENT_TOL)
    assert len(rep) == len(fx['samples']) and all(len(r['latent_err']) >= 1 for r in rep)


def ctor_wide(dim, **tr):
    return dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0., transformer = dict(dim = dim, depth = 2, **tr))


def small_inputs(B = 3, seed = 1):
    batch = synth.small_batch(B, seed = seed, dim_latent = 32, text_vocab = 64)
    nm = max(sum(torch.is_tensor(p) and p.is_floating_point() for p in s) for s in batch)
    times = torch.rand(B, nm, generator = torch.Generator().manual_seed(5))
    rows = sum(p.shape[0] for s in batch for p in s if torch.is_tensor(p) and p.is_floating_point())
    return batch, times, rows


def test_step_packed_graph_replay_follows_eager_step():
    """the captured resident step at dim 2048 (conditioning tables, packed weights, flat gradient / Adam / EMA buffers, split-K wgrads) replays the
    eager step: same losses and parameters over several steps"""
    from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
    from transfusion_pytorch_b200.modality_processing import pack_batch
    batch, times, _ = small_inputs(4, seed = 3)
    results = []
    for use_graph in (False, True):
        model = build(ctor_wide(2048, heads = 16, dim_head = 128), 7).train()
        trainer = DataParallelTrainer(model, lr = 1e-4, cuda_graph = use_graph)
        model.engine.ensure_attached()
        samples = [[torch.tensor([model.sos_id]), *s, torch.tensor([model.eos_id])] for s in batch]
        rb = pack_batch(samples, times, model, return_loss = True, return_embed = False)
        lat = model._latents_to_device(rb)
        model.engine.upload(rb)
        losses = [float(trainer.step_packed(rb, lat)) for _ in range(5)]
        torch.cuda.synchronize()
        results.append((losses, model.engine.flat.clone()))
        if use_graph:
            assert any(g.graph is not None for g in trainer._graphs.values()), 'the step was never captured'
    (l0, p0), (l1, p1) = results
    assert all(abs(a - b) / abs(a) < 2e-3 for a, b in zip(l0, l1)), (l0, l1)
    assert (p1 - p0).abs().max().item() < 2e-3 * p0.abs().max().item() + 2e-4


@pytest.mark.parametrize('dim,tr', [(1536, dict(heads = 8)), (2048, dict(heads = 16, dim_head = 128))], ids = ['d1536', 'd2048'])
def test_adam_steps_track_the_checker(dim, tr):
    """three `torch.optim.Adam` steps on the engine's gradients follow the same steps on the fp32 checker's"""
    batch, times, rows = small_inputs()
    losses = {}
    for dev in ('cuda', 'cpu'):
        model = build(ctor_wide(dim, **tr), 3, dev).train()
        opt = torch.optim.Adam(model.parameters(), lr = 1e-4)
        losses[dev] = []
        for step in range(3):
            noise = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(40 + step))]
            loss = model(batch, times = times, noise = noise)
            loss.backward()
            opt.step()
            opt.zero_grad()
            losses[dev].append(loss.item())
    assert all(abs(a - b) / abs(b) < LOSS_REL for a, b in zip(losses['cuda'], losses['cpu'])), losses
