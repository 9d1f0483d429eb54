"""GPU (H100): models deeper than ten layers, up to the depth limit of 64.  The AttentionResidual kernels themselves are held to float64
at every depth and width in tests/test_attn_residual_gpu.py; here:

  * whole models against the reference fixtures of oracle/make_golden_deep.py, at the tolerances of tests/test_parity_gpu.py;
  * one train step at size against the fp32 checker (oracle/torch_reference.py);
  * CUDA-graph replay and Self-Flow at depth 12;
  * depth <= 10 keeps one deferred-backward launch per call."""
import pytest
import torch

from helpers import load_golden, golden_noise, grad_fingerprint, unpack_rows
from oracle.make_golden_deep import INTERLEAVED, deep_batch
from oracle.torch_reference import OracleEngine
from test_dropout_gpu import _launches
from test_parity_gpu import LOSS_REL, build, check_grads, rel_max, HID_REL, GRAD_REL
from test_selfflow_cpu import grads_close
from transfusion_pytorch_b200 import Transfusion, SelfMaskedRepTraining, synth

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- whole model against the reference
@pytest.mark.parametrize('name,depth,seed,total_len', INTERLEAVED, ids = [c[0] for c in INTERLEAVED])
def test_deep_train_step_matches_reference(name, depth, seed, total_len):
    fx = load_golden(name)
    model = build(fx)
    assert model.transformer.depth == depth
    batch = deep_batch(seed, total_len)
    loss, bd = model(batch, times = fx['times'], return_breakdown = True, noise = golden_noise(fx, batch, model.dim_latents))
    rb = model._last_batch
    assert rb.modality_positions == fx['modality_positions'] and rb.total_tokens == fx['total_tokens']
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < LOSS_REL
    assert abs(bd.text.item() - fx['text_loss'].item()) / fx['text_loss'].item() < LOSS_REL
    for a, b in zip(bd.flow, fx['flow_losses']):
        assert abs(a.item() - b.item()) / b.item() < LOSS_REL
    st = model.engine.state
    rows = fx['hidden_rows']                 # the fixture keeps every hidden state at these positions
    for l, h in enumerate(fx['hiddens']):
        ours = unpack_rows(st['hid'][l], rb)
        for b in range(rb.B):
            keep = rows < int(rb.seq_lens[b])
            assert rel_max(ours[b, rows[keep]], h[b, keep]) < HID_REL, f'hidden {l} sample {b}'
    emb = unpack_rows(st['out'], rb)
    for b in range(rb.B):
        n = int(rb.seq_lens[b])
        assert rel_max(emb[b, :n], fx['embed'][b, :n]) < HID_REL
    loss.backward()
    check_grads(model, fx)


def test_deep_text_only_loss_grads_and_greedy_tokens():
    fx = load_golden('text_deep12')
    model = build(fx)
    text = synth.text_batch(4, 129, seed = 12)
    loss = model(text)
    assert abs(loss.item() - fx['loss'].item()) / fx['loss'].item() < LOSS_REL
    loss.backward()
    check_grads(model, fx)
    ref = fx['generated']
    seq = torch.cat((text[:, :fx['prompt_len']], ref), dim = -1)
    with torch.no_grad():
        lg = model.forward_text(seq[:, :-1], return_loss = False).float()
    pred = lg[:, fx['prompt_len'] - 1:].argmax(dim = -1).cpu()
    decided = fx['margins'] >= 0.1
    assert decided.float().mean().item() > 0.5
    assert torch.equal(pred[decided], ref[decided])
    # free-running greedy decode through the kv cache: identical up to the first position whose reference margin is below 0.1
    gen = model.generate_text_only(text[:, :fx['prompt_len']], fx['gen_len'], temperature = 0.).cpu()
    for b in range(gen.shape[0]):
        for j in range(gen.shape[1]):
            if gen[b, j] != ref[b, j]:
                assert fx['margins'][b, j] < 0.1, (b, j)
                break


# ---------------------------------------------------------------------------------------------------- at size against the checker
def _config(D, depth):
    return dict(num_text_tokens = 256, dim_latent = (64, 32), modality_default_shape = ((4,), (2,)), prob_uncond = 0.,
                transformer = dict(dim = D, depth = depth, heads = D // 64))


def _step(model, batch, times, noise):
    loss = model(batch, times = times, noise = noise)
    loss.backward()
    return loss.item(), grad_fingerprint((n, p.grad) for n, p in model.named_parameters() if p.grad is not None)


def _close(got, want, what):
    (lg, fg), (lw, fw) = got, want
    assert abs(lg - lw) / abs(lw) < LOSS_REL, (what, lg, lw)
    grads_close(fg, fw, GRAD_REL)


@pytest.mark.parametrize('D,depth,total_len', [(768, 12, 1024), (1024, 24, 512), (128, 64, 1024)])
def test_deep_train_step_at_size_matches_checker(D, depth, total_len):
    ctor = _config(D, depth)
    batch = synth.config4_batch(2, seed = 41, total_len = total_len, dims = (64, 32))
    nm = max(sum(isinstance(p, tuple) for p in s) for s in batch)
    times = torch.rand(2, nm, generator = torch.Generator().manual_seed(3))
    rows = [sum(p[1].shape[0] for s in batch for p in s if isinstance(p, tuple) and p[0] == t) for t in range(2)]
    noise = [torch.randn(max(r, 1), dl, generator = torch.Generator().manual_seed(10 + t)) for t, (r, dl) in enumerate(zip(rows, (64, 32)))]
    res = {}
    for dev in ('cpu', 'cuda'):
        torch.manual_seed(0)
        model = Transfusion(**ctor)
        synth.fill_parameters_(model, seed = 4)
        model = model.to(dev).eval()
        if dev == 'cpu':
            model._engine = OracleEngine(model)
        res[dev] = _step(model, batch, times, noise)
        del model
        torch.cuda.empty_cache()
    _close(res['cuda'], res['cpu'], 'cuda')


# ---------------------------------------------------------------------------------------------------- paths
DEEP12 = dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0., transformer = dict(dim = 128, depth = 12, heads = 2))


def _model(ctor, seed):
    torch.manual_seed(0)
    model = Transfusion(**ctor)
    synth.fill_parameters_(model, seed = seed)
    return model.cuda()


def test_deep_graph_replay_follows_eager():
    from transfusion_pytorch_b200.data_parallel import DataParallelTrainer
    from transfusion_pytorch_b200.modality_processing import pack_batch
    batch = synth.dropout_batch()
    times = torch.rand(3, 2, generator = torch.Generator().manual_seed(5))
    results = []
    for use_graph in (False, True):
        model = _model(DEEP12, 7).train()
        trn = DataParallelTrainer(model, lr = 1e-3, cuda_graph = use_graph)
        eng = model.engine
        eng.ensure_attached()
        samples = [[torch.tensor([model.sos_id]), *s, torch.tensor([model.eos_id])] for s in batch]
        rb = pack_batch(samples, times, model, return_loss = True, return_embed = False)
        lat = model._latents_to_device(rb)
        eng.upload(rb)
        losses = []
        for step in range(6):
            noise = [torch.randn(52, 32, generator = torch.Generator().manual_seed(500 + step)).cuda()]
            losses.append(trn.step_packed(rb, lat, noise = noise).item())
        results.append((losses, eng.flat.clone()))
        if use_graph:
            assert sum(g.graph is not None for g in trn._graphs.values()) == 1, 'the step was never captured'
    (l0, p0), (l1, p1) = results
    assert all(abs(a - b) / abs(a) < 2e-3 for a, b in zip(l0, l1)), (l0, l1)
    assert (p1 - p0).abs().max().item() < 2e-3 * p0.abs().max().item() + 2e-4


def test_deep_self_flow_matches_checker():
    from oracle.selfflow_reference import selfflow_loss
    batch = synth.small_batch(3, seed = 1, dim_latent = 32, text_vocab = 64)
    nm = max(sum(torch.is_tensor(p) and p.is_floating_point() for p in s) for s in batch)
    times = torch.rand(3, nm, generator = torch.Generator().manual_seed(5))
    rows = sum(p.shape[0] for s in batch for p in s if torch.is_tensor(p) and p.is_floating_point())
    noise = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(3))]
    tnoise = [torch.randn(rows, 32, generator = torch.Generator().manual_seed(8))]
    res = {}
    for dev in ('cuda', 'cpu'):
        torch.manual_seed(0)
        model = Transfusion(**DEEP12)
        synth.fill_parameters_(model, seed = 4)
        wrapper = SelfMaskedRepTraining(model.to(dev), use_asymmetric_dropout = False, student_layer = -3).to(dev)
        synth.fill_parameters_(wrapper.student_predict_head, seed = 6)
        if dev == 'cuda':
            total, (student, ssl) = wrapper(batch, times = times, noise = noise, teacher_noise = tnoise)
        else:
            total, student, ssl = selfflow_loss(wrapper, batch, times, noise, tnoise)
        total.backward()
        named = [(n, p.grad) for n, p in wrapper.student.named_parameters() if p.grad is not None]
        named += [(f'student_predict_head.{n}', p.grad) for n, p in wrapper.student_predict_head.named_parameters()]
        res[dev] = (total.item(), student.item(), ssl.item(), grad_fingerprint(named))
    for k in range(3):
        assert abs(res['cuda'][k] - res['cpu'][k]) / abs(res['cpu'][k]) < LOSS_REL, (k, res['cuda'][k], res['cpu'][k])
    grads_close(res['cuda'][3], res['cpu'][3], GRAD_REL)


# ---------------------------------------------------------------------------------------------------- launches
def _bwd2_kernels(model, batch, times, noise):
    """(n_later of every attn_residual_bwd2 call, number of attn_res_bwd2_k kernels) of one train step"""
    _, calls = _launches(model, batch, times, noise)
    n_later = [args[7] for args in calls['attn_residual_bwd2']]
    with torch.profiler.profile(activities = [torch.profiler.ProfilerActivity.CUDA]) as prof:
        loss = model(batch, times = times, noise = noise)
        loss.backward()
        torch.cuda.synchronize()
    kernels = sum(e.count for e in prof.key_averages() if 'attn_res_bwd2_k' in e.key)
    return n_later, kernels


@pytest.mark.parametrize('depth', [8, 12])
def test_deferred_backward_launches(depth):
    """depth <= 10: one kernel per attn_residual_bwd2 call, as before chunking; deeper: one per started chunk of 10 later layers"""
    ctor = dict(DEEP12, transformer = dict(DEEP12['transformer'], depth = depth))
    batch = synth.dropout_batch()
    times = torch.rand(3, 2, generator = torch.Generator().manual_seed(5))
    noise = [torch.randn(52, 32, generator = torch.Generator().manual_seed(1))]
    n_later, kernels = _bwd2_kernels(_model(ctor, 3).eval(), batch, times, noise)
    assert sorted(n_later) == sorted(list(range(depth)) + [depth])
    if depth <= 10:
        assert max(n_later) <= 10 and len(n_later) == depth + 1 and kernels == depth + 1
    else:
        assert kernels == sum(max(1, -(-n // 10)) for n in n_later)
