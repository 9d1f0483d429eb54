"""GPU (H100): Self-Flow training (`SelfMaskedRepTraining`) - the fused cosine loss kernel against float64, the wrapper against the reference
fixtures (tests/golden/small_selfflow*.pt) and the CPU checker (oracle/selfflow_reference.py), pad rows that leave the student loss alone,
unchanged launches without the term, and optimizer steps with teacher updates."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden, grad_fingerprint
from test_selfflow_cpu import FIXTURES, selfflow_noise, selfflow_wrapper, grads_close
from test_dropout_gpu import _launches, _model
from transfusion_pytorch_b200 import Transfusion, SelfMaskedRepTraining, _lib, synth
from oracle.selfflow_reference import selfflow_loss

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
LOSS_REL, GRAD_REL = 1e-3, 6e-2          # tests/test_parity_gpu.py


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


def rep_cos(ops, a, b, g, n_mean = None):
    M, D = a.shape
    da = torch.full((M, D), 7., device = 'cuda', dtype = BF16)
    part = torch.zeros(ops.lib.tfx_rep_cos_blocks(M), device = 'cuda', dtype = torch.float64)
    ticket = torch.zeros(1, device = 'cuda', dtype = torch.int32)
    loss = torch.zeros(1, device = 'cuda')
    gd = torch.tensor([g], device = 'cuda')
    ops.rep_cos_fwd_bwd(a, b, 1 if b.dtype == BF16 else 0, gd, n_mean or M, da, part, ticket, loss, M, D)
    torch.cuda.synchronize()
    assert ticket.item() == 0
    return loss, da


@pytest.mark.parametrize('D', [128, 256, 384, 512, 768, 1024])
def test_rep_cos_kernel_against_float64(ops, D):
    """loss and da against float64 `1 - F.cosine_similarity(a, b).mean()` and its autograd gradient, for ragged row counts, bf16 and fp32 teacher
    rows, a zero row (da = g b / (eps |b| n) there, torch's separately clamped norms) and a row shorter than eps"""
    gen = torch.Generator(device = 'cuda').manual_seed(D)
    for M in (1, 37, 1000, 4099):
        a = torch.randn(M, D, device = 'cuda', generator = gen) * 3
        b = torch.randn(M, D, device = 'cuda', generator = gen)
        a[:M // 3] += b[:M // 3] * 2                                     # a spread of cosines, not all near 0
        if M > 2:
            a[1] = 0.
            a[2] *= 1e-10
        for bt in (b.to(BF16), b):
            g = 0.37
            loss, da = rep_cos(ops, a, bt, g)
            aa = a.double().requires_grad_()
            want = 1. - F.cosine_similarity(aa, bt.double(), dim = -1).mean()
            (want * g).backward()
            assert abs(loss.item() - want.item()) < 1e-5 * max(1., abs(want.item())), (M, D, bt.dtype, loss.item(), want.item())
            ref = aa.grad
            err = (da.double() - ref).abs().amax(dim = -1) / ref.abs().amax(dim = -1).clamp(min = 1e-30)
            assert err.max().item() < 1e-2, (M, D, bt.dtype, err.argmax().item())
            again, da2 = rep_cos(ops, a, bt, g)
            assert torch.equal(loss, again) and torch.equal(da, da2)          # deterministic
    loss, _ = rep_cos(ops, torch.zeros(5, D, device = 'cuda'), torch.zeros(5, D, device = 'cuda'), 1.)
    assert loss.item() == 1.


def _run_wrapper(fx, wrapper, steps = 1, opt = None):
    batch = synth.dropout_batch()
    out = []
    for _ in range(steps):
        total, (student, ssl) = wrapper(batch, times = fx['times'], noise = selfflow_noise(fx, 0), teacher_noise = selfflow_noise(fx, 1), dropout_key = fx['dropout_key'])
        out.append((total, student, ssl))
        if opt is not None:
            opt.zero_grad()
            total.backward()
            opt.step()
            wrapper.update_teacher()
    return out


@pytest.mark.parametrize('name', FIXTURES)
def test_wrapper_matches_reference(name):
    fx = load_golden(name)
    wrapper = selfflow_wrapper(fx, 'cuda')
    (total, student, ssl), = _run_wrapper(fx, wrapper)
    for got, want in ((total, fx['loss']), (student, fx['student_loss']), (ssl, fx['ssl_loss'])):
        assert abs(got.item() - want.item()) / abs(want.item()) < LOSS_REL, (got.item(), want.item())
    total.backward()
    named = [(n, p.grad) for n, p in wrapper.student.named_parameters() if p.grad is not None]
    named += [(f'student_predict_head.{n}', p.grad) for n, p in wrapper.student_predict_head.named_parameters()]
    grads_close(grad_fingerprint(named), fx['grads'], GRAD_REL)
    if fx['wrapper_kwargs']['use_asymmetric_dropout']:
        assert wrapper.student.transformer.ff_dropout == 0.1 and wrapper.teacher.ema_model.transformer.ff_dropout == 0.      # set_dropout_ persists


CONFIG2 = dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), prob_uncond = 0., transformer = dict(dim = 512, depth = 8))


def test_config2_against_the_checker():
    batch, times = synth.config2_batch(2, seed = 4), synth.config2_times(2, seed = 4)
    noise = [torch.randn(1024, 384, generator = torch.Generator().manual_seed(3))]
    tnoise = [torch.randn(1024, 384, generator = torch.Generator().manual_seed(8))]
    res = {}
    for dev in ('cuda', 'cpu'):
        torch.manual_seed(0)
        model = Transfusion(**CONFIG2)
        synth.fill_parameters_(model, seed = 4)
        wrapper = SelfMaskedRepTraining(model.to(dev), use_asymmetric_dropout = False).to(dev)
        synth.fill_parameters_(wrapper.student_predict_head, seed = 6)
        if dev == 'cuda':
            total, (student, ssl) = wrapper(batch, times = times, noise = noise, teacher_noise = tnoise)
        else:
            total, student, ssl = selfflow_loss(wrapper, batch, times, noise, tnoise)
        total.backward()
        res[dev] = (total.item(), student.item(), ssl.item(), grad_fingerprint((n, p.grad) for n, p in wrapper.student_predict_head.named_parameters()))
    for k in range(3):
        assert abs(res['cuda'][k] - res['cpu'][k]) / abs(res['cpu'][k]) < LOSS_REL, (k, res['cuda'][k], res['cpu'][k])
    grads_close(res['cuda'][3], res['cpu'][3], GRAD_REL)


def _ssl_grads(wrapper, ssl):
    """gradients of the Self-Flow term alone: the student's (None where it sends none) and the head's"""
    ssl.backward()
    student = {n: p.grad for n, p in wrapper.student.named_parameters()}
    head = {f'student_predict_head.{n}': p.grad for n, p in wrapper.student_predict_head.named_parameters()}
    return student, head


@pytest.mark.parametrize('student_layer, teacher_layer', [(-3, -1), (-1, -1), (0, -1), (-3, -2)])
def test_self_flow_gradient_reaches_the_student_where_its_hidden_state_is(student_layer, teacher_layer):
    """the term alone is backpropagated (the student's own loss is out of the graph, so the engine's backward gets d total = 0 and only g_rep):
    the student's gradients must match the checker's autograd.  Hidden 1 (a layer's assembled x_c gradient), the final norm (d_out) and the
    tokens (dH[0]); teacher_layer = -2 reads the teacher's bf16 hidden state of the last layer"""
    fx = load_golden('small_selfflow')
    fx = dict(fx, wrapper_kwargs = dict(use_asymmetric_dropout = False, student_layer = student_layer, teacher_layer = teacher_layer))
    got, want = {}, {}
    for dev, out in (('cuda', got), ('cpu', want)):
        wrapper = selfflow_wrapper(fx, dev)
        if dev == 'cuda':
            (_, _, ssl), = _run_wrapper(fx, wrapper)
        else:
            _, _, ssl = selfflow_loss(wrapper, synth.dropout_batch(), fx['times'], selfflow_noise(fx, 0), selfflow_noise(fx, 1))
        out['ssl'] = ssl.item()
        out['student'], out['head'] = _ssl_grads(wrapper, ssl)
    assert abs(got['ssl'] - want['ssl']) / abs(want['ssl']) < LOSS_REL, (got['ssl'], want['ssl'])
    reached = {n: g for n, g in want['student'].items() if g is not None and g.abs().max() > 0}
    assert reached and 'text_embed.weight' in reached
    grads_close(grad_fingerprint((n, got['student'][n]) for n in reached), grad_fingerprint(reached.items()), GRAD_REL)
    grads_close(grad_fingerprint(got['head'].items()), grad_fingerprint(want['head'].items()), GRAD_REL)
    scale = max(g.abs().max().item() for g in reached.values())
    for n, g in got['student'].items():                                  # parameters after the student's hidden state get nothing
        if n not in reached and g is not None:
            assert g.abs().max().item() <= 1e-6 * scale, n


def test_pad_rows_leave_the_student_loss_and_gradients_unchanged():
    fx = load_golden('small_selfflow')
    grads = []
    for pad in (False, True):
        torch.manual_seed(0)
        model = Transfusion(**fx['ctor'])
        synth.fill_parameters_(model, seed = fx['seed'])
        model = model.cuda().train()
        rb, _ = model.pack(synth.dropout_batch(), times = fx['times'], return_loss = True, pad_rows = pad)
        assert (rb.M == 3 * 45) == pad
        loss, bd = model.forward_packed(rb, model._latents_to_device(rb), [n.cuda() for n in selfflow_noise(fx, 0)], return_breakdown = True)
        loss.backward()
        grads.append((loss.item(), bd.text.item(), [f.item() for f in bd.flow], {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}))
    (l0, t0, f0, g0), (l1, t1, f1, g1) = grads
    assert abs(l0 - l1) < 1e-5 * abs(l0) and abs(t0 - t1) < 1e-5 * abs(t0) and np.allclose(f0, f1, rtol = 1e-5)
    for n in g0:
        assert (g0[n] - g1[n]).abs().max().item() <= 1e-3 * g0[n].abs().max().item() + 1e-7, n         # split-K order only


def test_without_the_term_a_step_launches_what_a_plain_step_does():
    """rep_loss_weight = 0 and an unwrapped model: the launch list and every non-pointer argument of today's step"""
    fx = load_golden('small_selfflow')
    batch, times = synth.dropout_batch(), fx['times']
    noise = [n.cuda() for n in selfflow_noise(fx, 0)]
    want = _launches(_model(fx['ctor'], fx['seed']).train(), batch, times, noise)
    model = _model(fx['ctor'], fx['seed']).train()
    wrapper = SelfMaskedRepTraining(model, rep_loss_weight = 0., use_asymmetric_dropout = False).cuda()
    eng = model.engine
    eng.ensure_attached()
    eng.ops.timing, eng.ops.order = {}, []
    total, (student, ssl) = wrapper(batch, times = times, noise = noise)
    total.backward()
    torch.cuda.synchronize()
    order, timing = eng.ops.order, eng.ops.timing
    eng.ops.timing = eng.ops.order = None
    assert ssl.item() == 0. and total is student
    assert order == want[0]
    def norm(a):                                                         # as test_dropout_gpu._launches
        if torch.is_tensor(a):
            return ('tensor', tuple(a.shape), a.dtype)
        return a if isinstance(a, (int, float, str, type(None))) else type(a).__name__
    assert {n: [tuple(norm(a) for a in args) for (_, _, args) in calls] for n, calls in timing.items()} == want[1]


def test_adam_steps_with_teacher_updates_track_the_checker():
    fx = load_golden('small_selfflow')
    gpu = selfflow_wrapper(fx, 'cuda')
    cpu = selfflow_wrapper(fx, 'cpu')
    opt_g = torch.optim.Adam(gpu.parameters(), lr = 1e-3)
    opt_c = torch.optim.Adam(cpu.parameters(), lr = 1e-3)
    p0 = [p.detach().cpu().clone() for p in cpu.student_predict_head.parameters()]
    got = [t.item() for t, _, _ in _run_wrapper(fx, gpu, steps = 3, opt = opt_g)]
    want = []
    batch = synth.dropout_batch()
    for _ in range(3):
        total, _, _ = selfflow_loss(cpu, batch, fx['times'], selfflow_noise(fx, 0), selfflow_noise(fx, 1))
        want.append(total.item())
        opt_c.zero_grad()
        total.backward()
        opt_c.step()
        with torch.no_grad():
            for pe, p in zip(cpu.teacher.ema_model.parameters(), cpu.student.parameters()):
                pe.lerp_(p, 1. - cpu.teacher.beta)
    assert all(abs(a - b) / abs(b) < LOSS_REL for a, b in zip(got, want)), (got, want)
    assert got[0] != got[2]
    for (n, p), pc, q in zip(gpu.student_predict_head.named_parameters(), cpu.student_predict_head.parameters(), p0):
        upd_g, upd_c = p.detach().cpu() - q, pc.detach() - q                  # the head's Adam updates (sign-like where a gradient is tiny)
        assert (upd_g - upd_c).abs().mean().item() < 0.1 * upd_c.abs().mean().item(), n
