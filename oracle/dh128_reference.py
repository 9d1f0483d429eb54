"""TEST INFRASTRUCTURE ONLY - the CPU checker at any `dim_head` (64 or 128), on top of oracle/torch_reference.py and oracle/noqknorm_reference.py
(which it leaves as they are: their results at 64 are pinned by the existing fixtures).  Pinned by tests/test_dh128_cpu.py against
tests/golden/*dh128*.pt (outputs of the reference itself, oracle/make_golden_dh128.py).

TorchReference.stack and .cached_attention read the head width as the literal 64; here they are restated with the model's `dim_head`: the q / k
RMSNorm spans the whole head (scale sqrt(dim_head)), RoPE rotates dim_head / 2 frequency pairs, the logit scale is dim_head^-1/2.  Everything
else (`run`, the kv-cache decoder, the ODE solver, the `qk_rmsnorm = False` switch) is inherited.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

import oracle.torch_reference as _tr
from oracle.noqknorm_reference import NoQkNormReference
from oracle.torch_reference import OracleEngine, OracleKVCache, TorchReference


class _HeadDimStack(TorchReference):
    def stack(self, rb, x0, cond_tok, is_mod, kv_limit, rope_pos, valid, attend = None):
        tr, D, H, DH = self.tr, self.tr.dim, self.tr.heads, self.tr.dim_head
        sd = dict(self.m.named_parameters())
        B, n, _ = x0.shape
        cond = None
        if cond_tok is not None:
            w = self.tr.to_time_cond[0].weights
            fr = cond_tok[..., None] * w * 2 * math.pi
            feats = torch.cat((cond_tok[..., None], fr.sin(), fr.cos()), dim = -1)
            cond = F.silu(F.linear(feats, sd['transformer.to_time_cond.1.weight'], sd['transformer.to_time_cond.1.bias']))
        j = torch.arange(n)
        mask = (j[None, None, :] <= kv_limit[:, :, None]) & valid[:, None, :]
        freqs = self.m.rotary_emb.freqs
        x, hid, skips = x0, [x0], []
        isM = is_mod[..., None]

        def wrap_in(x, pre):
            xh = F.layer_norm(x, (D,))
            t = xh * (sd[f'{pre}.layernorm_gamma'] + 1.)
            if cond is None:
                return t
            g, b = F.linear(cond, sd[f'{pre}.to_film.weight'], sd[f'{pre}.to_film.bias']).chunk(2, dim = -1)
            return torch.where(isM, xh * (g + 1.) + b, t)

        def wrap_out(y, pre):
            t = y * (sd[f'{pre}.layerscale'] + 1.)
            if cond is None:
                return t
            z = F.linear(cond, sd[f'{pre}.to_ada_ln_zero.weight'], sd[f'{pre}.to_ada_ln_zero.bias']).sigmoid()
            return torch.where(isM, y * z, t)

        for i in range(tr.depth):
            pre = f'transformer.layers.{i}'
            layer = i + 1
            if layer <= tr.depth // 2:
                skips.append(x)
            elif f'{pre}.0.weight' in sd:
                x = F.linear(torch.cat((x, skips.pop()), dim = -1), sd[f'{pre}.0.weight']) + x
            u = wrap_in(x, f'{pre}.1')
            qk = F.linear(u, sd[f'{pre}.1.fn.to_qk.0.weight']).reshape(B, n, 2, H, DH)
            q, k = qk[:, :, 0].transpose(1, 2), qk[:, :, 1].transpose(1, 2)
            v = F.linear(u, sd[f'{pre}.1.fn.to_v.0.weight']).reshape(B, n, H, DH).transpose(1, 2)
            q, k = _tr._rms(q, sd[f'{pre}.1.fn.q_norm.gamma']), _tr._rms(k, sd[f'{pre}.1.fn.k_norm.gamma'])     # module lookup: see NoQkNormReference
            q, k = _tr._rope(q, rope_pos[:, None], freqs), _tr._rope(k, rope_pos[:, None], freqs)
            cap = tr.softcap_value
            if attend is not None:
                o = attend(i, q, k, v)
            else:
                sim = torch.einsum('bhid,bhjd->bhij', q * DH ** -0.5, k)
                sim = (sim / cap).tanh() * cap
                sim = sim.masked_fill(~mask[:, None], -torch.finfo(sim.dtype).max)
                o = torch.einsum('bhij,bhjd->bhid', sim.softmax(dim = -1), v)
            o = o * F.linear(u, sd[f'{pre}.1.fn.to_gates.0.weight']).transpose(1, 2)[..., None].sigmoid()
            a = F.linear(o.transpose(1, 2).reshape(B, n, H * DH), sd[f'{pre}.1.fn.to_out.1.weight'])
            x = x + wrap_out(a, f'{pre}.1')
            u = wrap_in(x, f'{pre}.2')
            hcat = F.linear(u, sd[f'{pre}.2.fn.net.0.weight'], sd[f'{pre}.2.fn.net.0.bias'])
            val, gate = hcat.chunk(2, dim = -1)
            f = F.linear(F.gelu(gate) * val, sd[f'{pre}.2.fn.net.3.weight'], sd[f'{pre}.2.fn.net.3.bias'])
            x = x + wrap_out(f, f'{pre}.2')
            hid.append(x)
            vals = torch.stack(hid)
            keys = _tr._rms(vals, sd[f'{pre}.3.norm_keys.gamma'])
            sim_l = torch.einsum('lbnd,d->bnl', keys, sd[f'{pre}.3.pseudo_queries']) * D ** -0.5
            x = torch.einsum('bnl,lbnd->bnd', sim_l.softmax(dim = -1), vals)
        out = _tr._rms(x, sd['transformer.norm.gamma'])
        return out, hid

    def cached_attention(self, rb, cache):
        cap_rows, softcap, DH = cache.cap, self.tr.softcap_value, self.tr.dim_head
        def attend(layer, q, k, v):
            o = torch.zeros_like(q)
            for b in range(rb.B):
                s0, n = int(rb.cu[b]), int(rb.seq_lens[b])
                if n == 0:
                    continue
                rows = torch.as_tensor(rb.kv_row[s0:s0 + n]).long()
                cache.k[layer][rows] = k[b, :, :n].transpose(0, 1)
                cache.v[layer][rows] = v[b, :, :n].transpose(0, 1)
                start = (int(rows[0]) // cap_rows) * cap_rows
                end = int(rb.kv_limit[s0:s0 + n].max()) + 1
                kk, vv = cache.k[layer][start:end].transpose(0, 1), cache.v[layer][start:end].transpose(0, 1)
                sim = torch.einsum('hid,hjd->hij', q[b, :, :n] * DH ** -0.5, kk)
                sim = (sim / softcap).tanh() * softcap
                j = torch.arange(start, end)
                vis = j[None, :] <= torch.as_tensor(rb.kv_limit[s0:s0 + n]).long()[:, None]
                sim = sim.masked_fill(~vis[None], -torch.finfo(sim.dtype).max)
                o[b, :, :n] = torch.einsum('hij,hjd->hid', sim.softmax(dim = -1), vv)
            return o
        return attend


class HeadDimReference(NoQkNormReference, _HeadDimStack):
    """NoQkNormReference.stack (the qk_rmsnorm switch) around the head-dim-generic stack"""


class HeadDimKVCache(OracleKVCache):
    def __init__(self, model, n_slabs, cap):
        tr = model.transformer
        self.n_slabs, self.cap, self.rows = n_slabs, cap, n_slabs * cap
        self.k = torch.zeros(tr.depth, self.rows, tr.heads, tr.dim_head)
        self.v = torch.zeros(tr.depth, self.rows, tr.heads, tr.dim_head)


class HeadDimOracleEngine(OracleEngine):
    """OracleEngine at the model's `dim_head` (with or without the qk-RMSNorm).  Injected by the tests: `model._engine = HeadDimOracleEngine(model)`."""

    def __init__(self, model):
        super().__init__(model)
        self.ref = HeadDimReference(model)

    def new_cache(self, n_slabs, cap):
        return HeadDimKVCache(self.model, n_slabs, cap)
