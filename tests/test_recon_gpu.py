"""GPU (H100): the reconstruction loss (MP.py:177-194, T.py:3420-3431; forward_modality T.py:2836-2856) and forward_modality's velocity term.

  * tfx_mse_recon_fwd_bwd against float64 of the reference's formula on ragged instances; with rscale = 0 its dpred is tfx_mse_fwd_bwd's, bit for bit
  * train steps against the reference's fixtures tests/golden/small_recon*.pt (oracle/make_golden_recon.py), at the tolerances of test_parity_gpu.py
  * a config-4 step against the host checker (oracle/recon_reference.py)
  * launch invariance: reconstruction_loss_weight = 0 launches what a model without the loss launches; a decoder's term launches nothing
  * CUDA-graph replay of batches with the same shape signature but another instance split and other times follows the eager steps"""
import numpy as np
import pytest
import torch

from helpers import load_golden, golden_noise, grad_fingerprint, unpack_rows
from transfusion_pytorch_b200 import Transfusion, _lib, synth
from transfusion_pytorch_b200.modality_processing import pack_batch
from oracle.recon_reference import ReconOracleEngine

pytestmark = pytest.mark.gpu

LOSS_REL, HID_REL, GRAD_REL = 1e-3, 2e-2, 6e-2


@pytest.fixture(scope = 'module')
def ops():
    torch.cuda.init()
    o = _lib.Ops()
    _lib.check(o.lib.tfx_init(0), 'tfx_init')
    return o


def _model(ctor, seed, **extra):
    torch.manual_seed(0)
    model = Transfusion(**ctor, **extra).cuda()
    synth.fill_parameters_(model, seed = seed)
    model.eval()
    return model


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def check_grads(model, fx):
    fp = grad_fingerprint((n, p.grad) for n, p in model.named_parameters() if p.grad is not None)
    assert set(fx['grads']) <= set(fp)
    for k, v in fx['grads'].items():
        ref_n = max(v['stats'][3].item(), 1e-12)
        assert abs(fp[k]['stats'][2].item() - v['stats'][2].item()) / ref_n < GRAD_REL, k
        assert abs(fp[k]['stats'][3].item() - v['stats'][3].item()) / ref_n < GRAD_REL, k


# ------------------------------------------------------------------------------------------------ kernel
def _ragged(dl, vel, seed):
    g = torch.Generator().manual_seed(seed)
    lens = [1, 31, 33, 1100] + torch.randint(1, 21, (300,), generator = g).tolist()
    lens = [lens[k] for k in torch.randperm(len(lens), generator = g).tolist()]
    n_inst, S = len(lens), sum(lens)
    t_inst = torch.rand(n_inst, generator = g, dtype = torch.float64)
    t_inst[:4] = torch.tensor([1e-3, 0.999, 0., 1.], dtype = torch.float64)
    row_inst = torch.repeat_interleave(torch.arange(n_inst), torch.tensor(lens))
    inst_w = torch.zeros(S, dtype = torch.float64)
    inst_w[:n_inst] = 1. / (n_inst * torch.tensor(lens, dtype = torch.float64))
    x, e, p = (torch.randn(S, dl, generator = g, dtype = torch.float64) for _ in range(3))
    ema = torch.randn(S, dl, generator = g, dtype = torch.float64) if vel else None
    return lens, t_inst[row_inst], row_inst, inst_w, x, e, p, ema


@pytest.mark.parametrize('dl', [16, 32, 384])
@pytest.mark.parametrize('vel', [False, True])
@pytest.mark.parametrize('b_is_t', [1, 0])
def test_kernel_matches_float64(ops, dl, vel, b_is_t):
    lens, t, row_inst, inst_w, x, e, p, ema = _ragged(dl, vel, seed = dl + 7 * vel + 3 * b_is_t)
    S, dlp = t.shape[0], dl + 8                                       # dpred with padded columns
    dev = lambda a, dt = torch.float32: a.to(dt).cuda().contiguous()
    flow = dev(x) - dev(e)                                            # what tfx_flow_noise computes (fp32)
    g32 = flow if b_is_t else dev(x - e + 0.25 * torch.sin(x))        # forward_modality: g = orig - noise
    ga, gb, rscale = 0.37, 0.11, 0.9
    target = flow if not vel else (ga * flow + gb * dev(ema)) / (ga + gb)
    G = ga if not vel else ga + gb
    pred, t_row, ri, iw = dev(p), dev(t), dev(row_inst, torch.int32), dev(inst_w)
    dpred = torch.full((S, dlp), 7., device = 'cuda', dtype = torch.bfloat16)
    sumsq, inst_sum, type_sum = (torch.zeros(n, device = 'cuda', dtype = torch.float64) for n in (1, S, 1))
    ops.mse_recon_fwd_bwd(pred, dl, target, g32, t_row, b_is_t, ri, iw, dpred, dlp, G, rscale, sumsq, inst_sum, type_sum, S, dl)
    torch.cuda.synchronize()
    # float64 reference formula: recon = noise + p (1 - t) against noised = x t + noise (1 - t) (interleaved) or against orig (forward_modality)
    t64 = t[:, None]
    gg = g32.double().cpu()
    if b_is_t:
        r = (e + p * (1. - t64)) - (x * t64 + e * (1. - t64))
    else:
        r = (e + p * (1. - t64)) - (gg + e)
    d = p - target.double().cpu()
    want_inst = torch.zeros(S, dtype = torch.float64).index_add_(0, row_inst, (r * r).sum(1))
    want_dpred = G * d + rscale * inst_w[row_inst][:, None] * (1. - t64) * r
    n_inst = len(lens)
    got = inst_sum.cpu()
    assert ((got[:n_inst] - want_inst[:n_inst]).abs() <= 1e-5 * want_inst[:n_inst] + 1e-9).all()
    assert (got[n_inst:] == 0).all()
    assert _rel(type_sum.item(), (inst_w[:n_inst] * want_inst[:n_inst]).sum()) < 1e-5
    assert _rel(sumsq.item(), (d * d).sum()) < 1e-5
    dp = dpred[:, :dl].double().cpu()
    assert ((dp - want_dpred).abs() <= 2 ** -8 * want_dpred.abs() + 1e-6 * want_dpred.abs().max()).all()
    assert (dpred[:, dl:].float() == 7.).all(), 'the padded columns are not the kernel\'s'
    # rscale = 0: exactly the dpred of tfx_mse_fwd_bwd
    d0, d1 = torch.zeros(S, dlp, device = 'cuda', dtype = torch.bfloat16), torch.ones(S, dlp, device = 'cuda', dtype = torch.bfloat16)
    acc = torch.zeros(4, device = 'cuda', dtype = torch.float64)
    ops.mse_recon_fwd_bwd(pred, dl, target, g32, t_row, b_is_t, ri, iw, d0, dlp, G, 0., acc[0:1], inst_sum, acc[2:3], S, dl)
    ops.mse_fwd_bwd(pred, dl, target, d1, dlp, G, acc[1:2], S, dl)
    torch.cuda.synchronize()
    assert torch.equal(d0[:, :dl].view(torch.int16), d1[:, :dl].view(torch.int16))
    assert _rel(acc[0].item(), acc[1].item()) < 1e-6


# ------------------------------------------------------------------------------------------------ model vs the reference
@pytest.mark.parametrize('name', ['small_recon', 'small_recon_only', 'small_recon_clean_vel'])
def test_interleaved_train_step_matches_reference(name):
    fx = load_golden(name)
    model = _model(fx['ctor'], fx['seed'])
    kw = {}
    if fx['ema_seed'] is not None:
        batch = synth.small_batch(3, seed = 1, dim_latent = 32, text_vocab = 64)
        ema = model.create_ema(0.99)
        synth.fill_parameters_(ema.ema_model, seed = fx['ema_seed'])
        (r0, d0), (r1, d1) = fx['noise_shapes']                      # student draw, then the teacher's
        noise = [torch.randn(r0, d0, generator = torch.Generator().manual_seed(9000 + 17 * fx['seed']))]
        kw = dict(velocity_consistency_ema_model = ema, velocity_consistency_delta_time = fx['delta'],
                  velocity_consistency_noise = [torch.randn(r1, d1, generator = torch.Generator().manual_seed(9000 + 1 + 17 * fx['seed']))])
    else:
        batch = synth.recon_batch()
        noise = golden_noise(fx, batch, model.dim_latents)
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = noise, **kw)
    assert _rel(loss.item(), fx['loss']) < LOSS_REL
    assert _rel(bd.text.item(), fx['text_loss']) < LOSS_REL
    for a, b in zip(bd.flow, fx['flow_losses']):
        assert _rel(a.item(), b) < LOSS_REL
    if fx['velocity_losses'] is not None:
        for a, b in zip(bd.velocity, fx['velocity_losses']):
            assert _rel(a.item(), b) < 3 * LOSS_REL
    assert [len(r) for r in bd.recon] == [len(r) for r in fx['recon_losses']]
    for ours, ref in zip(bd.recon, fx['recon_losses']):
        for a, b in zip(ours, ref):
            assert _rel(a.item(), b) < LOSS_REL
    rb, st = model._last_batch, model.engine.state
    emb = unpack_rows(st['out'], rb).float().cpu()
    for b in range(rb.B):                                             # the rows of each sample (the reference's padding rows hold values too)
        n = int(rb.seq_lens[b])
        assert (emb[b, :n] - fx['embed'][b, :n]).abs().max() / fx['embed'][b, :n].abs().max() < HID_REL, f'embed sample {b}'
    for l, h in enumerate(fx.get('hiddens', [])):
        ours = unpack_rows(st['hid'][l], rb).float().cpu()
        for b in range(rb.B):
            n = int(rb.seq_lens[b])
            assert (ours[b, :n] - h[b, :n]).abs().max() / h[b, :n].abs().max() < HID_REL, f'hidden {l} sample {b}'
    loss.backward()
    check_grads(model, fx)


def _modality_case(fx, w_r = None):
    encdec = fx['encdec']
    extra = dict(modality_encoder = synth.StandInEncoder(24, 32), modality_decoder = synth.StandInDecoder(32, 24)) if encdec else {}
    ctor = dict(fx['ctor']) if w_r is None else dict(fx['ctor'], reconstruction_loss_weight = w_r)
    model = _model(ctor, fx['seed'], **extra)
    kw = {}
    if fx['ema_seed'] is not None:
        kw = dict(velocity_consistency_ema_model = _model(ctor, fx['ema_seed'], **extra), velocity_consistency_delta_time = fx['delta'])
    x = synth.modality_batch(dim = 24 if encdec else 32)
    (shape,) = fx['noise_shapes']
    noise = torch.randn(int(np.prod(shape[:-1])), shape[-1], generator = torch.Generator().manual_seed(9000 + 17 * fx['seed']))
    return model, x, noise, kw


@pytest.mark.parametrize('name', ['small_recon_mod', 'small_recon_mod_encdec', 'small_recon_mod_vel'])
def test_forward_modality_matches_reference(name):
    fx = load_golden(name)
    model, x, noise, kw = _modality_case(fx)
    loss, (flow, vel, recon) = model.forward_modality(x, times = fx['times'], return_loss_breakdown = True, noise = noise, **kw)
    assert _rel(loss.item(), fx['loss']) < LOSS_REL and _rel(flow.item(), fx['flow_loss']) < LOSS_REL and _rel(recon.item(), fx['recon_loss']) < LOSS_REL
    assert abs(vel.item() - fx['velocity_loss'].item()) <= 3 * LOSS_REL * max(fx['velocity_loss'].item(), 1e-6)
    loss.backward()
    check_grads(model, fx)


def _launches(model, run):
    """entry points in launch order and their non-pointer arguments (tensors by shape / dtype) of one train step"""
    eng = model.engine
    eng.ensure_attached()
    eng.ops.timing, eng.ops.order = {}, []
    loss = run()
    loss.backward()
    torch.cuda.synchronize()
    order, timing = eng.ops.order, eng.ops.timing
    eng.ops.timing = eng.ops.order = None
    def norm(a):
        if torch.is_tensor(a):
            return ('tensor', tuple(a.shape), a.dtype)
        return a if isinstance(a, (int, float, str, type(None))) else type(a).__name__
    return order, {n: [tuple(norm(a) for a in args) for (_, _, args) in calls] for n, calls in timing.items()}, loss


def test_decoder_term_launches_nothing_and_carries_no_gradient():
    """forward_modality through a decoder: the term runs the user decoder under no_grad; the engine's launches and the gradients are those of w_r = 0"""
    fx = load_golden('small_recon_mod_encdec')
    out = []
    for w_r in (0.1, 0.):
        model, x, noise, kw = _modality_case(fx, w_r)
        order, args, loss = _launches(model, lambda: model.forward_modality(x, times = fx['times'], noise = noise))
        out.append((order, args, loss.item(), model.engine.gflat.clone()))
    (o1, a1, l1, g1), (o0, a0, l0, g0) = out
    assert o1 == o0 and a1 == a0 and 'mse_recon_fwd_bwd' not in o1
    assert l1 > l0 and _rel(l1 - l0, 0.1 * fx['recon_loss']) < LOSS_REL
    assert (g1 - g0).abs().max().item() <= 1e-5 * g0.abs().max().item()          # split-K atomics: run-to-run order only


def test_zero_weight_launches_the_kernels_of_a_model_without_the_loss():
    base = dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)), transformer = dict(dim = 128, depth = 2, heads = 2), prob_uncond = 0.)
    batch, times = synth.recon_batch(), synth.recon_times()
    noise = [torch.randn(50, 32, generator = torch.Generator().manual_seed(1)), torch.randn(39, 16, generator = torch.Generator().manual_seed(2))]
    runs = {}
    for w_r in (None, 0., 0.1):
        model = _model(base if w_r is None else dict(base, reconstruction_loss_weight = w_r), 3)
        runs[w_r] = _launches(model, lambda: model(batch, times = times, noise = noise))[:2]
        assert (model._last_batch.inst_w is not None) == bool(w_r)
    assert runs[0.] == runs[None]
    order, args = runs[0.1]
    assert order.count('mse_recon_fwd_bwd') == 2 and 'mse_fwd_bwd' not in order
    assert [n.replace('mse_recon_fwd_bwd', 'mse_fwd_bwd') for n in order] == runs[None][0]


def test_config4_train_step_matches_the_checker():
    ctor = dict(num_text_tokens = 256, dim_latent = (384, 192), modality_default_shape = ((4,), (2,)), reconstruction_loss_weight = 0.1, prob_uncond = 0.,
                transformer = dict(dim = 512, depth = 8))
    batch = synth.config4_batch(2, seed = 31)
    nm = max(sum(isinstance(p, tuple) for p in s) for s in batch)
    times = torch.rand(2, nm, generator = torch.Generator().manual_seed(5))
    rows = [sum(p[1].shape[0] for s in batch for p in s if isinstance(p, tuple) and p[0] == t) for t in (0, 1)]
    noise = [torch.randn(r, d, generator = torch.Generator().manual_seed(3 + t)) for t, (r, d) in enumerate(zip(rows, (384, 192)))]
    model = _model(ctor, 13)
    got, bd = model(batch, times = times, noise = noise, return_breakdown = True)
    torch.manual_seed(0)
    ref = Transfusion(**ctor)
    synth.fill_parameters_(ref, seed = 13)
    ref.eval()
    ref._engine = ReconOracleEngine(ref)
    with torch.no_grad():
        want, bd_ref = ref(batch, times = times, noise = noise, return_breakdown = True)
    assert _rel(got.item(), want.item()) < LOSS_REL
    for ours, theirs in zip(bd.recon, bd_ref.recon):
        assert len(ours) == len(theirs) > 0
        for a, b in zip(ours, theirs):
            assert _rel(a.item(), b.item()) < LOSS_REL


def test_graph_replay_across_instance_splits_follows_eager():
    """capture on one batch, replay on batches with the same shape signature but another instance split and other times"""
    from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
    ctor = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), reconstruction_loss_weight = 0.5, prob_uncond = 0.,
                transformer = dict(dim = 128, depth = 2, heads = 2))
    g = torch.Generator().manual_seed(0)
    txt = lambda n: torch.randint(0, 64, (n,), generator = g)
    lat = lambda n: torch.randn(n, 32, generator = g)
    splits = [(12, 12, 9), (14, 10, 9), (11, 13, 9), (12, 12, 9)]
    batches = [[[txt(4), lat(a), txt(4), lat(b), txt(4)], [txt(3), lat(c), txt(6)]] for a, b, c in splits]
    results = []
    for use_graph in (False, True):
        model = _model(ctor, 7).train()
        trn = DataParallelTrainer(model, lr = 1e-3, cuda_graph = use_graph)
        eng = model.engine
        eng.ensure_attached()
        losses, sigs = [], set()
        for step in range(8):
            batch = batches[step % len(batches)]
            times = torch.rand(2, 2, generator = torch.Generator().manual_seed(100 + step))
            samples = [[torch.tensor([model.sos_id]), *s, torch.tensor([model.eos_id])] for s in batch]
            rb = pack_batch(samples, times, model, return_loss = True, return_embed = False)
            sigs.add(trn._signature(rb, eng))
            lat_d = model._latents_to_device(rb)
            eng.upload(rb)
            noise = [torch.randn(rb.S, 32, generator = torch.Generator().manual_seed(500 + step)).cuda()]
            losses.append(trn.step_packed(rb, lat_d, noise = noise).item())
        assert len(sigs) == 1, 'the batches must share one shape signature'
        results.append((losses, eng.flat.clone()))
        if use_graph:
            assert sum(gr.graph is not None for gr in trn._graphs.values()) == 1, 'the step was never captured'
    (l0, p0), (l1, p1) = results
    assert all(abs(a - b) / abs(a) < 2e-3 for a, b in zip(l0, l1)), (l0, l1)
    assert (p1 - p0).abs().max().item() < 2e-3 * p0.abs().max().item() + 2e-4
