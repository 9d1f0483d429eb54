"""TEST INFRASTRUCTURE ONLY - fp32 restatement of the Self-Flow wrapper's loss (`SelfMaskedRepTraining.forward`, T.py:3511-3569) on
oracle/torch_reference.py: the student's and the teacher's forwards over the padded batch that `pack(pad_rows = True)` describes, the predictor
head (RMSNorm, GEGLU FeedForward) and 1 - mean cosine similarity over every row of the padded layout.  FFN dropout is not restated here (the
asymmetric-dropout case is pinned by its reference fixture).  Pinned by tests/golden/small_selfflow*.pt in tests/test_selfflow_cpu.py.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.torch_reference import TorchReference, _rms


def hidden_states(model, batch, times, noise):
    """(loss dict of the padded training forward, hidden states [tokens, layer 1 .. depth, final norm], each [b, n, d])"""
    rb, _ = model.pack(batch, times = times, prob_uncond = 0., return_loss = True, pad_rows = True)
    lat = [torch.cat([x.detach().float().cpu() for x in lst]) if lst else None for lst in rb.latents]
    eps = [n.reshape(-1, model.dim_latents[t]).float().cpu() if n is not None else None for t, n in enumerate(noise)]
    res = TorchReference(model).run(rb, lat, eps, text_loss_weight = model.text_loss_weight, flow_loss_weight = model.flow_loss_weight)
    return res, [*res['hiddens'], res['embed']]


def selfflow_loss(wrapper, batch, times, noise, teacher_noise):
    """(total, student loss, Self-Flow loss) of one wrapper forward with autograd through the student and the head"""
    student, teacher = wrapper.student, wrapper.teacher.ema_model
    assert not wrapper.use_asymmetric_dropout or (student.transformer.ff_dropout == 0. and wrapper.student_dropout_rate == 0.), 'FFN dropout is not restated'
    res, hs = hidden_states(student, batch, times, noise)
    with torch.no_grad():
        _, ht = hidden_states(teacher, batch, times, teacher_noise)
    x, y = hs[wrapper.student_layer], ht[wrapper.teacher_layer]
    head = wrapper.student_predict_head
    ff = head[1].net
    value, gate = F.linear(_rms(x, head[0].gamma), ff[0].weight, ff[0].bias).chunk(2, dim = -1)
    pred = F.linear(F.gelu(gate) * value, ff[3].weight, ff[3].bias)
    ssl = 1. - F.cosine_similarity(pred, y, dim = -1).mean()
    return res['total'] + ssl * wrapper.rep_loss_weight, res['total'], ssl
