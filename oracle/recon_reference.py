"""TEST INFRASTRUCTURE ONLY - plain-PyTorch fp32 restatement of the reference's reconstruction loss and of the value-only velocity term of
`forward_modality`, on top of oracle/torch_reference.py (which it leaves as it is).  Pinned by tests/test_recon_cpu.py against
tests/golden/small_recon*.pt (outputs of the reference itself, oracle/make_golden_recon.py).

The reconstruction loss is restated with the reference's own formula, not with the identity the kernel uses:
  interleaved (MP.py:177-194, T.py:3299-3308, 3420-3431):  recon_i = mse(noised_i, noise_i + pred_i (1 - t_i)) per instance, averaged per type,
      weighted by the type's token share and `reconstruction_loss_weight`;
  forward_modality (T.py:2836-2856):  mse(noise + pred (1 - t), the modality before the encoder).
`model_output_clean` is not restated here (TorchReference predicts the flow directly); its fixture is checked on the GPU only.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.torch_reference import OracleEngine


class ReconOracleEngine(OracleEngine):
    """OracleEngine that also takes the engine's reconstruction / velocity keywords (`recon_weight`, `recon_g`, `vel_targets`, `vel_weight`,
    `vel_grad`).  Injected by the tests: `model._engine = ReconOracleEngine(model)`."""

    def __init__(self, model):
        if getattr(model, 'model_output_clean', False):
            raise NotImplementedError('the CPU checker does not restate model_output_clean')
        super().__init__(model)

    def forward(self, rb, latents, eps, *, train, want_logits = False, vlimit = 0, text_loss_weight = 1., flow_loss_weight = 1., modality_only = False, cache = None,
                want_preds = None, recon_weight = 0., recon_g = None, vel_targets = None, vel_weight = 0., vel_grad = True, **_):
        with torch.set_grad_enabled(train):
            res = self.ref.run(rb, latents, eps, text_loss_weight = text_loss_weight, flow_loss_weight = flow_loss_weight, vlimit = vlimit,
                               modality_only = modality_only, want_loss = train, cache = cache)
            extra = {}
            if train:
                total = res['total']
                T = float(rb.total_tokens)
                rt = torch.as_tensor(rb.row_time)
                if vel_targets is not None:
                    assert not vel_grad, 'the checker restates the value-only velocity term of forward_modality'
                    vel = []
                    for t, (s0, s1) in enumerate(rb.type_rows):
                        if vel_targets[t] is None or s1 == s0:
                            vel.append(torch.zeros(())); continue
                        flow = latents[t].float().cpu() - eps[t].float().cpu()
                        vel.append(F.mse_loss(flow, vel_targets[t].float().cpu()))
                        total = total + vel[-1] * vel_weight
                    extra['vel'] = [v.detach() for v in vel]
                if recon_weight > 0.:
                    per_type = [[] for _ in range(rb.n_types)]
                    sums = torch.zeros(len(rb.instances), dtype = torch.float64)
                    for k, inst in enumerate(rb.instances):
                        t = inst.modality_type
                        r0 = rb.type_rows[t][0] + inst.row0
                        r1 = r0 + inst.length
                        x = latents[t].float().cpu()[inst.row0:inst.row0 + inst.length]
                        e = eps[t].float().cpu()[inst.row0:inst.row0 + inst.length]
                        p = res['preds'][t][inst.row0:inst.row0 + inst.length]
                        tt = rt[r0:r1, None]
                        recon = e + p * (1. - tt)
                        if modality_only:
                            orig = (recon_g[t].float().cpu()[inst.row0:inst.row0 + inst.length] + e) if recon_g is not None and recon_g[t] is not None else x
                            loss_i = F.mse_loss(recon, orig)
                        else:
                            loss_i = F.mse_loss(x * tt + e * (1. - tt), recon)
                        per_type[t].append(loss_i)
                        sums[k] = loss_i.detach().double() * inst.length * x.shape[1]
                    means = [torch.stack(v).mean() if v else torch.zeros(()) for v in per_type]
                    for t, m in enumerate(means):
                        total = total + m * (1. if modality_only else rb.n_type_tokens[t] / T) * recon_weight
                    extra.update(recon = [m.detach() for m in means], recon_inst = sums)
                res['total'] = total
        valid = res['valid']
        pack = lambda t: t[valid]
        out = dict(embed = pack(res['embed']).detach(), logits = pack(res['logits']).detach(), preds = [p.detach() if p is not None else None for p in res['preds']])
        if train:
            self.state = res
            out.update(total = res['total'].detach(), text = res['text'].detach(), flows = res['flows'].detach(), **extra)
        return out
