"""CUDA engine: drives the C-ABI kernels (libtfx_b200.so) for the Transfusion block stack - forward,
backward, loss heads and the fused optimizer - over the ragged descriptor built by
`modality_processing.pack_batch`.

PyTorch supplies device memory, the current stream and (for data parallel) `torch.distributed`; every
floating-point operation of the hot path is a kernel of this repository.  There is no CPU or eager
fallback: constructing the engine without the built extension, or on a non-CUDA device, raises.

Data flow of one layer (reference transfusion.py:1203-1246, math restated in SURVEY.md appendix A):

    x_in --(skip_proj GEMM, K = [x | skip])--> x_a --adaLN--> u_A --GEMM qkvg (+qk-norm, RoPE)--> q,k,v,g
         --flash attention (span mask, softcap, value gate)--> o --GEMM to_out (+gate, +residual)--> x_b
         --adaLN--> u_F --GEMM ffn_in (+GEGLU)--> h --GEMM ffn_out (+gate, +residual)--> x_c = H[l]
         --AttentionResidual over H[0..l]--> x_in of the next layer

The residual stream and all normalisation statistics are fp32; GEMM / attention operands are bf16 with
fp32 accumulation.
"""
from __future__ import annotations

import functools
import math
import ctypes
from dataclasses import dataclass

import numpy as np
import torch
from torch import Tensor

from . import _lib
from ._pinned import POOL
from .modality_processing import RaggedBatch
from .transfusion import MODEL_DIMS, MIN_HEADS, MAX_HEADS, DIM_HEADS, MAX_HEADS_D128

BF16, F32, I32, I64 = torch.bfloat16, torch.float32, torch.int32, torch.int64


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


_EMPTY_I32 = np.zeros(0, dtype = np.int32)


# ------------------------------------------------------------------ axial positional embedding (optional: `add_pos_emb`; T.py:1383-1403, 2792-2796; MP.py:1003-1046)
# One MLP Linear(1, h) -> SiLU -> Linear(h, D) per axis, evaluated on the integer coordinates 0 .. L-1 (L = batch maximum of that axis) and summed over
# the axes per latent row.  The tables have at most a few hundred rows: plain tensor algebra on the device (not kernels), off every benchmarked path.
def posemb_tables(params, lens, device):
    """params: per axis (w0 [h, 1], b0 [h], w2 [D, h], b2 [D]); returns per axis (seq [L, 1], pre [L, h], act [L, h], table [L, D])"""
    out = []
    for (w0, b0, w2, b2), L in zip(params, lens):
        seq = torch.arange(int(L), device = device, dtype = F32)[:, None]
        pre = seq * w0.reshape(1, -1) + b0
        act = pre * torch.sigmoid(pre)
        out.append((seq, pre, act, act @ w2.t() + b2))
    return out


def posemb_add(rows: Tensor, tables, coords):
    """rows[s] += sum over axes of table_axis[coord_axis[s]]"""
    for (_, _, _, e), c in zip(tables, coords):
        rows += e.index_select(0, c)


def posemb_backward(d_rows: Tensor, tables, coords, params, grads):
    """accumulates the parameter gradients (grads: per axis views (gw0, gb0, gw2, gb2)) of the rows' gradient d_rows [n, D] fp32"""
    for (seq, pre, act, e), c, (w0, b0, w2, b2), (gw0, gb0, gw2, gb2) in zip(tables, coords, params, grads):
        d_e = torch.zeros_like(e).index_add_(0, c, d_rows)
        gw2 += d_e.t() @ act
        gb2 += d_e.sum(0)
        sig = torch.sigmoid(pre)
        d_pre = (d_e @ w2) * (sig * (1. + pre * (1. - sig)))
        gw0 += (d_pre * seq).sum(0)[:, None]
        gb0 += d_pre.sum(0)


def pack_job_table(jobs, device):
    """device job table of `tfx_cast_pack_multi` for jobs (src, ld_src, c_src, row_src, dst, r_dst, c_dst, dst_is_f32):
    returns (table, block -> job, first block of each job, number of blocks)"""
    # struct TfxPackJob (include/tfx_b200.h): 56 bytes
    dt = np.dtype([('src', '<u8'), ('ld_src', '<i8'), ('row_src', '<u8'), ('dst', '<u8'), ('R_dst', '<i8'), ('C_src', '<i4'), ('C_dst', '<i4'),
                   ('dst_f32', '<i4'), ('pad', '<i4')])
    assert dt.itemsize == 56
    tab = np.zeros(len(jobs), dtype = dt)
    blk_job, blk_first = [], []
    for j, (src, ld_src, c_src, row_src, d, r_dst, c_dst, f32) in enumerate(jobs):
        tab[j] = (src.data_ptr(), ld_src, row_src.data_ptr() if row_src is not None else 0, d.data_ptr(), r_dst, c_src, c_dst, f32, 0)
        nb = (r_dst * c_dst + 2047) // 2048
        blk_first.append(len(blk_job))
        blk_job.extend([j] * nb)
    return (torch.from_numpy(tab.view(np.uint8).copy()).to(device), torch.tensor(blk_job, dtype = I32, device = device),
            torch.tensor(blk_first, dtype = I32, device = device), len(blk_job))


def w1_row_src(inner: int) -> np.ndarray:
    """packed FeedForward W1 (GEGLU epilogue layout): tile t = [value rows 64t.. | gate rows inner+64t..]; source row of every packed row, -1 past `inner`"""
    Ip = _round_up(inner, 64)
    src = np.full(2 * Ip, -1, dtype = np.int64)
    for t in range(Ip // 64):
        for j in range(64):
            c = 64 * t + j
            if c < inner:
                src[128 * t + j] = c
                src[128 * t + 64 + j] = inner + c
    return src


@functools.lru_cache(maxsize = None)
def wgrad_splits(n_out, n_in, K, sms):
    """split-K factor of a wgrad GEMM (dW[n_out, n_in] over K tokens, both operands MN-major).  For each candidate the library reports the launch
    geometry (`_lib.gemm_store_items`: the tile, and so the work items, depend on the k-blocks per item); the busiest SM then runs
    ceil(items / sms) items of (k-blocks x tile rows / 128) units.  The fewest splits within 5 % of the shortest such path win: every split
    adds one red.add pass over dW.  Work items keep at least 16 k-blocks.  E.g. over 131072 tokens on 132 SMs the [1664 x 512] QKVG gradient
    has 7 x 4 = 28 tiles of 256 x 128: 9 splits are 252 items (2 waves of 228 k-blocks), 14 splits 3 waves of 147 (3 % shorter) and 4 splits
    one 85 % wave of 512; 9 are taken."""
    cost = {}
    for s in range(1, 65):
        items, kb, tile_m, s_eff = _lib.gemm_store_items(n_out, n_in, K, 1, 1, s)
        if s_eff != s or (s > 1 and kb < 16):
            break
        cost[s] = -(-items // sms) * kb * tile_m // 128
    best = min(cost.values())
    return min(s for s, c in cost.items() if c <= 1.05 * best)


class KVCache:
    """Slab kv cache (decode path; reference layout `(layers, 2, batch, heads, seq, dim_head)`, T.py:976-977, 1264, 2260, re-padded and
    concatenated per step there).  Here: per layer one K (post-RoPE) and one V matrix, bf16 `[n_slabs * cap, heads * dim_head]`, token-major like
    every other activation; sample / branch `s` owns rows `[s * cap, (s + 1) * cap)`.  Appends happen in place from the QKVG GEMM epilogue;
    how much of a slab is valid is host / device bookkeeping of the sampler (`len`), never a mask tensor."""

    def __init__(self, engine, n_slabs: int, cap: int):
        self.n_slabs, self.cap, self.rows = int(n_slabs), int(cap), int(n_slabs) * int(cap)
        nbytes = 2 * engine.depth * self.rows * engine.HI * 2
        assert nbytes < 96 << 30, f'kv cache of {nbytes / 2**30:.1f} GiB requested ({n_slabs} slabs x {cap} rows): lower max_length / batch the prompts'
        # zero-filled: rows past a slab's filled length are read by whole-tile loads (and multiplied by p = 0): they must be finite
        self.k = torch.zeros(engine.depth, self.rows, engine.HI, device = engine.device, dtype = BF16)
        self.v = torch.zeros(engine.depth, self.rows, engine.HI, device = engine.device, dtype = BF16)
        # LASER (T.py:981-983): the cache keeps the raw values, attention reads exp(softclamp(v)) from a second slab written in place
        self.vl = torch.zeros_like(self.v) if engine.laser else None

    def slab_start(self, s):
        return np.asarray(s, dtype = np.int64) * self.cap


class Engine:
    def __init__(self, model):
        self.ops = _lib.Ops()                       # raises loudly if the extension is missing
        self.model = model
        tr = model.transformer
        self.D, self.H, self.depth = tr.dim, tr.heads, tr.depth
        self.DH = tr.dim_head
        self.HI = self.H * self.DH
        self.inner = tr.ff_inner
        self.Ip = _round_up(self.inner, 64)
        self.laser, self.laser_clamp, self.vres = tr.attn_laser, tr.laser_softclamp_value, tr.use_value_residual
        # `attn_kwargs = dict(gate_values = False)` (T.py:901-904, 1026-1027): no to_gates, attention output without the sigmoid(gate) factor;
        # every attention-side call of such a model gets gates = None
        self.gated = bool(getattr(tr, 'gate_values', True))
        # packed rows [to_qk | to_v | gate tile]: the 128-row gate tile (to_gates at rows [0, H), the value-residual mix Linear at
        # [round_even(H), + H), zero pad) exists iff the model is gated or has the value residual; otherwise the QKVG GEMM computes no tile
        self.gate_tile = self.gated or self.vres
        self.NQ = 3 * self.HI + (128 if self.gate_tile else 0)
        # first packed row of the mix Linear: behind the gates, at an even row so that the bf16 pairs of its gradient columns stay 4-byte aligned
        # (an odd head count exists at dim_head 128 only)
        self.MIX = 3 * self.HI + _round_up(self.H, 2)
        self.V = model.text_embed.weight.shape[0]
        self.Vp = _round_up(self.V, 8)
        self.Kt = _round_up(self.D + 1, 64)         # padded K of the time-cond Linear
        self.W = 2 * self.depth                     # AdaptiveWrappers
        self.softcap = tr.softcap_value
        # qk_rmsnorm = False (T.py:949-951 skipped): q, k are RoPE(u W^T) only, so no bound on the logits follows from the gammas and every layer runs
        # the general (running-maximum) attention kernels; the q / k norm gammas stay out of the flat buffers (their .grad stays None, as in the reference)
        self.qk_norm = bool(getattr(tr, 'qk_rmsnorm', True))
        # the bounded-logit (wgmma) attention kernels exist for 64-wide normed heads only; every other model runs the general kernels alone
        self.fast = self.qk_norm and self.DH == 64
        self.fastp = None                           # per layer: bounded-logit attention parameters (tfx_attn_fast_params), `fast` models only
        # dim_head = 128 takes the `_d128` twin of every per-head kernel (same arguments, 128-wide heads); the elementwise LASER value
        # kernels see a 128-wide head as two 64-wide ones
        self.d128 = self.DH == 128
        self.sfx = '_d128' if self.d128 else ''
        self.vheads = self.HI // 64
        self.clean, self.clean_eps = bool(getattr(model, 'model_output_clean', False)), float(getattr(model, 'eps', 1e-2))
        self.posemb = tuple(bool(a) for a in getattr(model, 'add_pos_emb', ()))      # per modality type: axial positional embedding on the latent tokens
        self.scale = self.DH ** -0.5
        self.dls = list(model.dim_latents)
        self.dlp = [_round_up(d, 8) for d in self.dls]
        assert self.D in MODEL_DIMS, f'model dim must be one of {MODEL_DIMS} for the row kernels'
        if self.d128:
            assert 1 <= self.H <= MAX_HEADS_D128, f'heads must be in [1, {MAX_HEADS_D128}] at dim_head 128'
        else:
            assert self.DH == 64, f'dim_head must be one of {DIM_HEADS}'
            assert self.H % 2 == 0 and MIN_HEADS <= self.H <= MAX_HEADS, 'heads must be even (two 64-wide heads per 128-column GEMM tile) and at most 32'
        self.device = None
        self.flat = None
        self.ws = {}
        self._dirty = True
        self._ptr_arrays = []
        self.launches = 0
        self.graph_pins = None                      # list of retired workspace tensors once any CUDA graph has been captured
        self.frozen = False                         # True inside a sampling session: parameters cannot change, skip the re-pack check

    # ------------------------------------------------------------------ parameters
    def _trainable(self):
        m = self.model
        skip = set()
        for mod in list(m.modality_encoder) + list(m.modality_decoder):
            if mod is not None:
                skip |= {id(p) for p in mod.parameters()}
        if not self.qk_norm:                        # built but unused without the qk-RMSNorm (T.py:886-888, 949-951): no gradient, no optimizer state
            skip |= {id(p) for n, p in m.named_parameters() if n.endswith(('.fn.q_norm.gamma', '.fn.k_norm.gamma'))}
        return [(n, p) for n, p in m.named_parameters() if p.requires_grad and id(p) not in skip]

    def attach(self):
        """Move all trainable parameters into one flat fp32 buffer (views keep the state_dict layout) with a
        matching flat gradient buffer: one fused Adam launch, one all-reduce, wgrad GEMMs write straight in."""
        named = self._trainable()
        # Flat-buffer order = bucket order of the data-parallel all-reduce.  Gradients of the conditioning path (to_time_cond, every
        # to_film / to_ada_ln_zero) are produced AFTER the layer loop of backward() from tables accumulated over all layers, so those
        # parameters live in a "late" region behind the per-layer parameters: a layer bucket handed to NCCL is then really final.
        late = lambda n: ('.to_film.' in n) or ('.to_ada_ln_zero.' in n) or n.startswith('transformer.to_time_cond.')
        named = [(n, p) for n, p in named if not late(n)] + [(n, p) for n, p in named if late(n)]
        dev = named[0][1].device
        if dev.type != 'cuda':
            raise _lib.TfxError(f'the CUDA engine needs the model on a CUDA device (got {dev}); there is no CPU path')
        rc = self.ops.lib.tfx_init(dev.index if dev.index is not None else torch.cuda.current_device())
        _lib.check(rc, 'tfx_init')
        self.device = dev
        offs, total = {}, 0
        for n, p in named:
            offs[n] = total
            total += _round_up(p.numel(), 4)
        flat = torch.zeros(total, device = dev, dtype = F32)
        gflat = torch.zeros(total, device = dev, dtype = F32)
        for n, p in named:
            o, k = offs[n], p.numel()
            flat[o:o + k].copy_(p.data.reshape(-1).float())
            p.data = flat[o:o + k].view(p.shape)
            p.grad = gflat[o:o + k].view(p.shape)
        self.flat, self.gflat, self.offs, self.named = flat, gflat, offs, dict(named)
        self.named_first = named[0][1]
        self.exp_avg = self.exp_avg_sq = None
        self.opt_step = 0
        self._first_ptr = named[0][1].data_ptr()
        self.late_start = min((offs[n] for n, _ in named if late(n)), default = total)
        self._build_maps()
        self._dirty = True
        if not getattr(self, '_hooked', False):          # checkpoints loaded after the first forward must reach the bf16 operand copies
            self.model.register_load_state_dict_post_hook(lambda *a, **k: self.mark_dirty())
            self._hooked = True

    def mark_dirty(self):
        """Tell the engine that parameter VALUES changed outside its own optimizer (manual `p.add_`, custom optimizers stepping in
        eval mode ...): the next forward re-packs the bf16 GEMM operand copies.  Training forwards always re-pack."""
        self._dirty = True

    def ensure_attached(self):
        if self.flat is None or self.named_first.data_ptr() != self._first_ptr:
            self.attach()

    def P(self, name):            # parameter tensor by state-dict name
        return self.named[name]

    def _posemb_params(self, t, nax, grads = False):
        get = self.G if grads else self.P
        return [tuple(get(f'pos_emb_mlp.{t}.mlps.{a}.{k}') for k in ('0.weight', '0.bias', '2.weight', '2.bias')) for a in range(nax)]

    def G(self, name):            # gradient view inside the flat buffer
        o, p = self.offs[name], self.named[name]
        return self.gflat[o:o + p.numel()].view(p.shape)

    def _build_maps(self):
        """Row maps between packed bf16 operand layouts and the state-dict parameter layouts."""
        dev, D, HI, H, inner, Ip = self.device, self.D, self.HI, self.H, self.inner, self.Ip
        src = w1_row_src(inner)
        self.w1_row_src = torch.from_numpy(src.astype(np.int32)).to(dev)
        self.w1_row_src64 = torch.from_numpy(src).to(dev)
        self.layer_maps = []
        for i in range(self.depth):
            pre = f'transformer.layers.{i}'
            w1_off = self.offs[f'{pre}.2.fn.net.0.weight']
            b1_off = self.offs[f'{pre}.2.fn.net.0.bias']
            w1_rows = torch.where(self.w1_row_src64 >= 0, w1_off + self.w1_row_src64 * D, torch.full_like(self.w1_row_src64, -1))
            b1_cols = torch.where(self.w1_row_src64 >= 0, b1_off + self.w1_row_src64, torch.full_like(self.w1_row_src64, -1)).to(I32)
            q_off, v_off = self.offs[f'{pre}.1.fn.to_qk.0.weight'], self.offs[f'{pre}.1.fn.to_v.0.weight']
            r = np.full(self.NQ, -1, dtype = np.int64)              # -1: a packed row without a parameter (pad, or the gates of an ungated model)
            r[:2 * HI] = q_off + np.arange(2 * HI) * D
            r[2 * HI:3 * HI] = v_off + np.arange(HI) * D
            if self.gated:
                r[3 * HI:3 * HI + H] = self.offs[f'{pre}.1.fn.to_gates.0.weight'] + np.arange(H) * D
            if f'{pre}.1.fn.to_learned_value_residual.0.weight' in self.offs:        # value-residual mix Linear: pad rows [MIX, MIX + H) of the packed weight
                r[self.MIX:self.MIX + H] = self.offs[f'{pre}.1.fn.to_learned_value_residual.0.weight'] + np.arange(H) * D
            w2_off = self.offs[f'{pre}.2.fn.net.3.weight']
            w2_rows = torch.from_numpy(w2_off + np.arange(D, dtype = np.int64) * inner).to(dev)
            self.layer_maps.append(dict(w1_rows = w1_rows.contiguous(), b1_cols = b1_cols.contiguous(), qkvg_rows = torch.from_numpy(r).to(dev), w2_rows = w2_rows))
        # conditioning tables: wrapper w occupies columns [w*3D, (w+1)*3D): gamma | beta | z
        rows = np.full(self.W * 3 * D, -1, dtype = np.int64)
        bias_idx = np.zeros(self.W * 3 * D, dtype = np.int64)
        for w in range(self.W):
            i, j = divmod(w, 2)
            pre = f'transformer.layers.{i}.{j + 1}'
            fo, zo = self.offs[f'{pre}.to_film.weight'], self.offs[f'{pre}.to_ada_ln_zero.weight']
            rows[w * 3 * D: w * 3 * D + 2 * D] = fo + np.arange(2 * D) * 4 * D
            rows[w * 3 * D + 2 * D: (w + 1) * 3 * D] = zo + np.arange(D) * 4 * D
            bias_idx[w * 3 * D: w * 3 * D + 2 * D] = self.offs[f'{pre}.to_film.bias'] + np.arange(2 * D)
            bias_idx[w * 3 * D + 2 * D: (w + 1) * 3 * D] = self.offs[f'{pre}.to_ada_ln_zero.bias'] + np.arange(D)
        self.fz_rows = torch.from_numpy(rows).to(dev)
        self.fz_bias_idx = torch.from_numpy(bias_idx).to(dev)
        tw = self.offs['transformer.to_time_cond.1.weight']
        self.wt_rows = torch.from_numpy(tw + np.arange(4 * D, dtype = np.int64) * (D + 1)).to(dev)

    def buf(self, name, shape, dtype, zero = False):
        t = self.ws.get(name)
        n = int(np.prod(shape)) if len(shape) else 1
        if t is None or t.dtype != dtype or t.numel() < n:
            if t is not None and self.graph_pins is not None:
                self.graph_pins.append(t)       # a captured graph may hold this address: never hand the block back to the allocator
            t = torch.empty(max(n, 1), device = self.device, dtype = dtype)
            self.ws[name] = t
            if zero:
                t.zero_()
        return t[:n].view(shape)

    def pin_workspaces(self):
        """Called before a CUDA-graph capture: from now on a workspace buffer that has to grow is retired, not freed (captured graphs
        bake raw device pointers; see data_parallel._StepGraph and sampling.DecodeSession)."""
        if self.graph_pins is None:
            self.graph_pins = []

    def _build_pack_jobs(self):
        """Destination buffers + the device-resident job table of `tfx_cast_pack_multi` (built once per attach)."""
        D, HI, H, Ip, inner = self.D, self.HI, self.H, self.Ip, self.inner
        pk = self.packed = {}
        jobs = []
        def dst(name, rows, cols, dtype = BF16):
            t = pk[name] = torch.zeros(rows, cols, device = self.device, dtype = dtype) if cols else torch.zeros(rows, device = self.device, dtype = dtype)
            return t
        def job(src, ld_src, c_src, row_src, d, r_dst, c_dst):
            jobs.append((src, ld_src, c_src, row_src, d, r_dst, c_dst, 1 if d.dtype == F32 else 0))
        for i in range(self.depth):
            pre = f'transformer.layers.{i}'
            wq = dst(f'qkvg{i}', self.NQ, D)
            job(self.P(f'{pre}.1.fn.to_qk.0.weight'), D, D, None, wq, 2 * HI, D)
            job(self.P(f'{pre}.1.fn.to_v.0.weight'), D, D, None, wq[2 * HI:], HI, D)
            if self.gated:
                job(self.P(f'{pre}.1.fn.to_gates.0.weight'), D, D, None, wq[3 * HI:], H, D)
            if f'{pre}.1.fn.to_learned_value_residual.0.weight' in self.named:
                job(self.P(f'{pre}.1.fn.to_learned_value_residual.0.weight'), D, D, None, wq[self.MIX:], H, D)
            job(self.P(f'{pre}.1.fn.to_out.1.weight'), HI, HI, None, dst(f'wo{i}', D, HI), D, HI)
            job(self.P(f'{pre}.2.fn.net.0.weight'), D, D, self.w1_row_src, dst(f'w1{i}', 2 * Ip, D), 2 * Ip, D)
            job(self.P(f'{pre}.2.fn.net.3.weight'), inner, inner, None, dst(f'w2{i}', D, Ip), D, Ip)
            job(self.P(f'{pre}.2.fn.net.0.bias'), 1, 1, self.w1_row_src, dst(f'b1{i}', 2 * Ip, 0, F32), 2 * Ip, 1)
            if f'{pre}.0.weight' in self.named:
                job(self.P(f'{pre}.0.weight'), 2 * D, 2 * D, None, dst(f'wskip{i}', D, 2 * D), D, 2 * D)
        job(self.P('to_text_logits.weight'), D, D, None, dst('wvocab', self.V, D), self.V, D)
        for t, (dl, dlp) in enumerate(zip(self.dls, self.dlp)):
            job(self.P(f'model_to_latent_projs.{t}.weight'), D, D, None, dst(f'wm2l{t}', dl, D), dl, D)
            if f'latent_to_model_projs.{t}.weight' in self.named:
                job(self.P(f'latent_to_model_projs.{t}.weight'), dl, dl, None, dst(f'wl2m{t}', D, dlp), D, dlp)
        job(self.P('transformer.to_time_cond.1.weight'), D + 1, D + 1, None, dst('wt', 4 * D, self.Kt), 4 * D, self.Kt)
        wfz = dst('wfz', self.W * 3 * D, 4 * D)
        bfz = dst('bfz', self.W * 3 * D, 0, F32)
        for w in range(self.W):
            i, j = divmod(w, 2)
            pre = f'transformer.layers.{i}.{j + 1}'
            job(self.P(f'{pre}.to_film.weight'), 4 * D, 4 * D, None, wfz[w * 3 * D:], 2 * D, 4 * D)
            job(self.P(f'{pre}.to_ada_ln_zero.weight'), 4 * D, 4 * D, None, wfz[w * 3 * D + 2 * D:], D, 4 * D)
            job(self.P(f'{pre}.to_film.bias'), 2 * D, 2 * D, None, bfz[w * 3 * D:], 1, 2 * D)
            job(self.P(f'{pre}.to_ada_ln_zero.bias'), D, D, None, bfz[w * 3 * D + 2 * D:], 1, D)
        self._pack_tab, self._pack_blk_job, self._pack_blk_first, self._pack_nblocks = pack_job_table(jobs, self.device)
        self._pack_ptr = self._first_ptr

    def pack_weights(self, force = False):
        """fp32 master parameters -> bf16 GEMM operands in kernel layouts: ONE launch.  Parameters are views of the flat buffer with their
        own version counters, so in-place updates by torch.optim / load_state_dict / user code are invisible here: training forwards
        therefore ALWAYS re-pack (force = True, ~0.1 ms); inference forwards re-pack when the engine knows of a change (its own optimizer,
        backward(), load_state_dict hook, `mark_dirty()`)."""
        have = getattr(self, 'packed', None) is not None and getattr(self, '_pack_ptr', None) == self._first_ptr
        if have and not self._dirty and (self.frozen or not force):
            return
        if getattr(self, '_pack_ptr', None) != self._first_ptr:
            self._build_pack_jobs()
        self.ops.cast_pack_multi(self._pack_tab, self._pack_blk_job, self._pack_blk_first, self._pack_nblocks)
        # per layer: is the bounded-logit (wgmma) attention path valid for the current q/k norm gammas?  (device-side decision)
        if self.fast:
            if self.fastp is None or self.fastp.device != self.device:
                self.fastp = torch.zeros(self.depth, 8, device = self.device, dtype = F32)
            for i in range(self.depth):
                pre = f'transformer.layers.{i}.1.fn'
                self.ops.attn_fast_params(self.P(f'{pre}.q_norm.gamma'), self.P(f'{pre}.k_norm.gamma'), 64, self.scale, self.softcap, self.fastp[i])
        self._dirty = False

    # ------------------------------------------------------------------ descriptor upload
    META_NAMES = ['text_id', 'label', 'kv_limit', 'rope_pos', 'cond_row', 'slot', 'tile_q0', 'tile_qend', 'tile_kv0', 'tile_kvend',
                  'kt_kv0', 'kt_kvend', 'kt_q0', 'kt_qend', 'row_token', 't2_q0', 't2_qend', 't2_kv0', 't2_kvend', 'k2_kv0', 'k2_kvend', 'k2_q0', 'k2_qend', 'k2_order', 'kv_row', 'pos_c0', 'pos_c1', 'pos_c2',
                  'row_inst']

    def stage_meta(self, rb: RaggedBatch):
        """All per-token / per-tile int32 metadata and the float metadata of a batch in ONE pooled pinned buffer.
        Returns (raw pinned buffer, int32 view, layout) - layout = (sizes per array, n_int, n_float)."""
        ints = [getattr(rb, n) if getattr(rb, n) is not None else _EMPTY_I32 for n in self.META_NAMES]
        sizes = [_round_up(a.shape[0], 4) for a in ints]
        fl = np.concatenate([rb.cond_times, rb.row_time] + ([rb.inst_w] if rb.inst_w is not None else [])).astype(np.float32)
        n_int, n_fl = sum(sizes), _round_up(fl.shape[0], 4)
        raw = POOL.take((n_int + n_fl) * 4)                       # pooled pinned staging: no per-step cudaHostAlloc
        host = raw[:(n_int + n_fl) * 4].view(I32)
        hv = host.numpy()
        off = 0
        for a, s in zip(ints, sizes):
            hv[off:off + a.shape[0]] = a; off += s
        hv[n_int:n_int + fl.shape[0]] = fl.view(np.int32)
        return raw, host, (tuple(a.shape[0] for a in ints), tuple(sizes), n_int, fl.shape[0])

    def meta_views(self, rb: RaggedBatch, devbuf: Tensor, layout):
        lens, sizes, n_int, n_fl = layout
        d, off = {}, 0
        for n, ln, s in zip(self.META_NAMES, lens, sizes):
            d[n] = devbuf[off:off + ln]; off += s
        fdev = devbuf[n_int:n_int + n_fl].view(F32)
        d['cond_times'], d['row_time'] = fdev[:rb.n_cond], fdev[rb.n_cond:rb.n_cond + rb.S]
        if rb.inst_w is not None:                                  # reconstruction loss: per-instance weights behind the row times
            d['inst_w'] = fdev[rb.n_cond + rb.S:]
        d['h2d_bytes'] = devbuf.numel() * 4
        d['_keep'] = devbuf
        d['_layout'] = layout
        return d

    def upload(self, rb: RaggedBatch):
        """One pinned staging buffer, one H2D copy for all integer + float metadata."""
        if rb.dev:
            return rb.dev
        raw, host, layout = self.stage_meta(rb)
        devbuf = host.to(self.device, non_blocking = True)
        POOL.give(raw)
        rb.dev = self.meta_views(rb, devbuf, layout)
        return rb.dev

    def rope_table(self, max_pos: int):
        """cos/sin tables: [pos][dim_head / 2] (row kernels) and its transpose [dim_head / 2][pos] (thread-per-row QKVG epilogue)"""
        n = _round_up(max_pos + 1, 1024)
        t = self.ws.get('rope_cs')
        if t is None or t.shape[0] < n:
            if t is not None and self.graph_pins is not None:
                self.graph_pins += [t, self.ws['rope_cs_t']]
            nf = self.DH // 2
            t = torch.empty(n, nf, 2, device = self.device, dtype = F32)
            tt = torch.empty(nf, n, 2, device = self.device, dtype = F32)
            self.ops.rope_table(self.model.rotary_emb.freqs.detach().float().contiguous(), t, tt, n, nf)
            self.ws['rope_cs'], self.ws['rope_cs_t'] = t, tt
        return t

    def _ptr_array(self, tensors):
        arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
        self._ptr_arrays.append(arr)            # keep alive until the launch has consumed it (host-side copy at launch)
        if len(self._ptr_arrays) > 256:
            self._ptr_arrays = self._ptr_arrays[-64:]
        return ctypes.cast(arr, ctypes.c_void_p)

    # ------------------------------------------------------------------ forward
    def forward(self, rb: RaggedBatch, latents: list | None, eps: list | None, *, train: bool, want_logits = False, vlimit = 0,
                text_loss_weight = 1., flow_loss_weight = 1., modality_only = False, cache: KVCache | None = None, want_preds = None,
                vel_targets = None, vel_weight = 0., dropout = False, dropout_key = None, vel_grad = True, recon_weight = 0., recon_g = None, rep_layer = None):
        """Runs the block stack over a ragged batch.  `latents[t]`: fp32 [S_t, dl_t] device tensors (clean latents when
        `eps` is given, already-noised / decode-time latents otherwise).  With train=True activations are kept for
        `backward()` and the fused loss heads produce the loss scalars and the head gradients in the same pass.
        `dropout`: the owning module is in training mode; FFN dropout then applies to a train forward (`Transformer.ff_dropout_p`), with the
        masks of `dropout_key` (see `dropout_key()`).
        `vel_grad = False`: the velocity term only adds its value, mse(flow, vel_target) (forward_modality, T.py:2823-2834).
        `recon_weight > 0` (train forwards): the reconstruction loss (MP.py:177-194, T.py:3420-3431) is folded into the flow head's gradient
        pass (tfx_mse_recon_fwd_bwd); its residual per row is (1 - t) pred - t flow, or with `recon_g` (per type, forward_modality T.py:2840-2856)
        (1 - t) pred - g.  Needs the batch's reconstruction metadata (`modality_processing.build_recon_meta`).
        `rep_layer` (Self-Flow, `SelfMaskedRepTraining`): index into the hidden states [tokens, layer 1 .. depth, final norm]; `res['rep']` is that
        state in packed rows.  A train forward hands it out in fp32 and `backward(g_rep = ...)` takes its gradient; an inference forward (the
        teacher) returns the kept buffer itself and applies FFN dropout like a train forward (its module follows the wrapper's `.train()`)."""
        self.ensure_attached()
        self.pack_weights(force = train)
        o, D, HI, H, Ip, M = self.ops, self.D, self.HI, self.H, self.Ip, rb.M
        dv = self.upload(rb)
        nc, S = rb.n_cond, rb.S
        p_ff = self.model.transformer.ff_dropout_p(train or rep_layer is not None, dropout)
        st = self.state = dict(rb = rb, train = train, layers = [], p_ff = p_ff, drop_key = self.dropout_key(dropout_key) if p_ff > 0. else None)
        pk = self.packed
        rope = self.rope_table(rb.max_rope_pos)
        cond_row = dv['cond_row'] if nc > 0 else None
        tag = 'T' if train else 'I'
        # kv-cache (incremental) forward: the M tokens of `rb` are NEW tokens; their keys / values are appended in place at rows
        # dv['kv_row'] of the cache slabs and kv_limit / the attention tile tables are expressed in cache-row coordinates
        assert cache is None or not train, 'the kv cache is an inference-time structure'
        kv_rows = dv['kv_row'] if cache is not None else None
        M_kv = cache.rows if cache is not None else 0
        want_preds = want_logits if want_preds is None else want_preds

        # ---- conditioning tables, one row per distinct time (reference evaluates them per token: T.py:1132,749,767)
        if nc > 0:
            feats = self.buf('feats', (nc, self.Kt), BF16)
            o.time_features(dv['cond_times'], self.model.transformer.to_time_cond[0].weights, feats, nc, D // 2, self.Kt)
            cpre = self.buf('cpre', (nc, 4 * D), F32)
            o.gemm_store(feats, self.Kt, 0, pk['wt'], self.Kt, 0, nc, 4 * D, self.Kt, cpre, 4 * D, None, 0, self.P('transformer.to_time_cond.1.bias'), None, 1.0, 0, 1)
            cond = self.buf('cond', (nc, 4 * D), BF16)
            o.table_op(cpre, 4 * D, None, 0, None, 0, cond, 4 * D, nc, 4 * D, 1)
            tab = self.buf('tab', (nc, self.W * 3 * D), F32)
            o.gemm_store(cond, 4 * D, 0, pk['wfz'], 4 * D, 0, nc, self.W * 3 * D, 4 * D, tab, self.W * 3 * D, None, 0, pk['bfz'], None, 1.0, 0, 1)
            zg = self.buf('zg', (nc, self.W * D), F32)
            for w in range(self.W):
                o.table_op(tab[:, w * 3 * D + 2 * D:], self.W * 3 * D, None, 0, zg[:, w * D:], self.W * D, None, 0, nc, D, 0)
            st.update(feats = feats, cpre = cpre, cond = cond, tab = tab, zg = zg)
        tab_ld, zg_ld = self.W * 3 * D, self.W * D

        # ---- flow noise inject + latent_to_model (MP.py:645-667), token assemble (T.py:3173-3184)
        modtok = None
        if S > 0:
            modtok = self.buf('modtok', (S, D), F32)
            st['noised'], st['flow'] = [], []
            for t, (s0, s1) in enumerate(rb.type_rows):
                n = s1 - s0
                if n == 0:
                    st['noised'].append(None); st['flow'].append(None); continue
                dl, dlp = self.dls[t], self.dlp[t]
                x = latents[t]
                assert x.shape == (n, dl) and x.dtype == F32 and x.is_cuda, f'latents[{t}] must be a cuda fp32 [{n}, {dl}] tensor'
                noised = self.buf(f'noised{t}', (n, dlp), BF16)
                if dlp != dl:
                    noised[:, dl:].zero_()
                has_proj = f'latent_to_model_projs.{t}.weight' in self.named
                nf32 = None if has_proj else modtok[s0:s1]
                if eps is not None and eps[t] is not None:
                    flow = self.buf(f'flow{t}', (n, dl), F32)
                    o.flow_noise(x, eps[t], dv['row_time'][s0:s1], noised, dlp, nf32, flow, n, dl)
                else:
                    flow = None
                    o.flow_noise(x, None, None, noised, dlp, None, None, n, dl)
                    if not has_proj:
                        modtok[s0:s1].copy_(x)
                if has_proj:
                    o.gemm_store(noised, dlp, 0, pk[f'wl2m{t}'], dlp, 0, n, D, dl, modtok[s0:s1], D, None, 0, self.P(f'latent_to_model_projs.{t}.bias'), None, 1.0, 0, 1)
                if self.posemb and self.posemb[t]:          # + axial positional embedding (T.py:2792-2796)
                    nax = int(self.model.modality_num_dim[t])
                    coords = [dv[f'pos_c{a}'][s0:s1] for a in range(nax)]
                    tabs = posemb_tables(self._posemb_params(t, nax), rb.pos_max[t][:nax], self.device)
                    posemb_add(modtok[s0:s1], tabs, coords)
                    st.setdefault('posemb', {})[t] = (tabs, coords)
                st['noised'].append(noised); st['flow'].append(flow)
        x0 = self.buf(f'{tag}x0', (M, D), F32)
        x0b = self.buf(f'{tag}x0b', (M, D), BF16)
        o.embed_assemble(dv['text_id'], self.P('text_embed.weight'), modtok, dv['slot'] if S > 0 else None, x0, x0b, M, D)

        # ---- block stack
        hid = [x0b]
        skips = []
        x_in, x_in_b = x0, x0b
        n_tiles = int(rb.tile_q0.shape[0])
        for i in range(self.depth):
            L = {}
            pre = f'transformer.layers.{i}'
            lt = f'{tag}{i}' if train else 'I'           # inference reuses one set of buffers
            layer = i + 1
            first_half = layer <= self.depth // 2
            if first_half:
                skips.append((i, x_in_b))
            has_skip = (not first_half) and f'{pre}.0.weight' in self.named
            if has_skip:
                src_i, skip_b = skips.pop()
                x_a = self.buf(f'{lt}xa', (M, D), F32)
                o.gemm_resid(x_in_b, D, skip_b, D, D, pk[f'wskip{i}'], 2 * D, M, D, 2 * D, None, x_in, x_a, None, None, None, None, 0, None)
                L.update(skip_src = src_i, skip_b = skip_b)
            else:
                x_a = x_in
            wA, wF = 2 * i, 2 * i + 1
            filmA = tab[:, wA * 3 * D:] if nc > 0 else None
            filmF = tab[:, wF * 3 * D:] if nc > 0 else None
            zgA = zg[:, wA * D:] if nc > 0 else None
            zgF = zg[:, wF * D:] if nc > 0 else None
            uA = self.buf(f'{lt}uA', (M, D), BF16); statsA = self.buf(f'{lt}sA', (M, 2), F32)
            o.adaln_fwd(x_a, cond_row, filmA, tab_ld, self.P(f'{pre}.1.layernorm_gamma'), uA, statsA, M, D)
            q = self.buf(f'{lt}q', (M, HI), BF16)
            if cache is not None:
                k, v = cache.k[i], cache.v[i]
            else:
                # inference shares one buffer set across layers, but the value residual reads the FIRST layer's values in every later layer
                k = self.buf(f'{lt}k', (M, HI), BF16); v = self.buf(f'{lt}v0' if (self.vres and i == 0) else f'{lt}v', (M, HI), BF16)
            gates = self.buf(f'{lt}g', (M, H), F32) if self.gated else None
            has_mix = self.vres and i > 0
            mixpre = self.buf(f'{lt}mix', (M, H), F32) if has_mix else None
            if self.qk_norm:
                qk_inv = self.buf(f'{lt}qi', (M, 2 * H), F32)
                getattr(o, 'gemm_qkvg' + self.sfx)(uA, D, pk[f'qkvg{i}'], D, M, H, D, q, k, v, gates, qk_inv, self.P(f'{pre}.1.fn.q_norm.gamma'), self.P(f'{pre}.1.fn.k_norm.gamma'),
                            dv['rope_pos'], self.ws['rope_cs_t'], int(self.ws['rope_cs_t'].shape[1]), kv_rows, mixpre)
            else:
                qk_inv = None
                getattr(o, 'gemm_qkvg_rope' + self.sfx)(uA, D, pk[f'qkvg{i}'], D, M, H, D, q, k, v, gates, dv['rope_pos'], self.ws['rope_cs_t'],
                                                       int(self.ws['rope_cs_t'].shape[1]), kv_rows, mixpre)
            if has_mix:                                  # learned value residual (T.py:956-960): v = v mix + v_first_layer (1 - mix), in place (also on the cache rows)
                v_first = cache.v[0] if cache is not None else st['layers'][0]['v']
                getattr(o, 'vmix_fwd' + self.sfx)(v, HI, kv_rows, v_first, HI, mixpre, self.P(f'{pre}.1.fn.to_learned_value_residual.0.bias'), M, H)
            v_att, att_gates = v, gates
            if self.laser:                               # LASER (T.py:981-983): attention runs on exp(softclamp(v)); log + gate follow it
                v_att = cache.vl[i] if cache is not None else self.buf(f'{lt}vl', (M, HI), BF16)
                o.laser_v_fwd(v, HI, kv_rows, v_att, HI, M, self.vheads, self.laser_clamp)
                att_gates = None
            att = self.buf(f'{lt}o', (M, HI), BF16); lse = self.buf(f'{lt}lse', (H, M), F32)
            o_l = self.buf(f'{lt}ol', (M, HI), BF16) if self.laser else att
            fp = self.fastp[i] if self.fast else None
            if getattr(rb, 'single_row_tiles', False):
                # text decode: one query row per sample against its cache slab (split-KV decode kernel)
                getattr(o, 'attn_decode' + self.sfx)(q, k, v_att, HI, HI, HI, att_gates, H, dv['kv_limit'], dv['tile_q0'], dv['tile_kv0'], dv['tile_kvend'], n_tiles, o_l, HI, self.scale, self.softcap)
            else:
                # both kernels are enqueued; the one whose precondition (read from `fp` on the device) fails returns immediately.  Without the
                # qk-RMSNorm, or at dim_head 128, only the general kernel runs (fp = None)
                if self.fast:
                    o.attn_fwd_tc(q, k, v_att, HI, HI, HI, att_gates, H, dv['kv_limit'], dv['t2_q0'], dv['t2_qend'], dv['t2_kv0'], dv['t2_kvend'], int(rb.t2_q0.shape[0]),
                                  o_l, HI, lse, M, M_kv, self.scale, self.softcap, fp)
                if self.d128:
                    o.attn_fwd_d128(q, k, v_att, HI, HI, HI, att_gates, H, dv['kv_limit'], dv['tile_q0'], dv['tile_qend'], dv['tile_kv0'], dv['tile_kvend'],
                                    n_tiles, o_l, HI, lse, M, self.scale, self.softcap)
                else:
                    o.attn_fwd(q, k, v_att, HI, HI, HI, att_gates, H, dv['kv_limit'], dv['tile_q0'], dv['tile_qend'], dv['tile_kv0'], dv['tile_kvend'], n_tiles,
                               o_l, HI, lse, M, self.scale, self.softcap, fp)
            if self.laser:
                getattr(o, 'laser_out_fwd' + self.sfx)(o_l, gates, att, M, H)
            x_b = self.buf(f'{lt}xb', (M, D), F32); yA = self.buf(f'{lt}yA', (M, D), BF16) if train else None
            o.gemm_resid(att, HI, None, 0, 0, pk[f'wo{i}'], HI, M, D, HI, None, x_a, x_b, None, yA, cond_row, zgA, zg_ld, self.P(f'{pre}.1.layerscale'))
            uF = self.buf(f'{lt}uF', (M, D), BF16); statsF = self.buf(f'{lt}sF', (M, 2), F32)
            o.adaln_fwd(x_b, cond_row, filmF, tab_ld, self.P(f'{pre}.2.layernorm_gamma'), uF, statsF, M, D)
            vg = self.buf(f'{lt}vg', (M, 2 * Ip), BF16); h = self.buf(f'{lt}h', (M, Ip), BF16)
            if p_ff > 0.:
                o.gemm_geglu_drop(uF, D, pk[f'w1{i}'], D, pk[f'b1{i}'], M, 2 * Ip, D, vg, h, st['drop_key'], p_ff, i)
            else:
                o.gemm_geglu(uF, D, pk[f'w1{i}'], D, pk[f'b1{i}'], M, 2 * Ip, D, vg, h)
            yF = self.buf(f'{lt}yF', (M, D), BF16) if train else None
            # x_c feeds nothing but the AttentionResiduals (the residual stream continues from their fp32 output): it is kept in bf16 only, which
            # halves the largest HBM term of the step
            x_c = self.buf(f'{tag}Hb{i + 1}', (M, D), BF16)
            o.gemm_resid(h, Ip, None, 0, 0, pk[f'w2{i}'], Ip, M, D, Ip, self.P(f'{pre}.2.fn.net.3.bias'), x_b, None, x_c, yF, cond_row, zgF, zg_ld,
                         self.P(f'{pre}.2.layerscale'))
            hid.append(x_c)
            xr = self.buf(f'{tag}xr{i}', (M, D), F32); xrb = self.buf(f'{tag}xrb{i}', (M, D), BF16)
            rlse = self.buf(f'{tag}rlse{i}', (M,), F32) if train else None
            o.attn_residual_fwd_h16(self._ptr_array(hid), len(hid), self.P(f'{pre}.3.norm_keys.gamma'), self.P(f'{pre}.3.pseudo_queries'), xr, xrb, rlse, M, D)
            L.update(xr = xr, rlse = rlse, mixpre = mixpre, o_l = o_l, v_att = v_att)
            L.update(x_a = x_a, uA = uA, statsA = statsA, q = q, k = k, v = v, gates = gates, qk_inv = qk_inv, att = att, lse = lse, yA = yA, x_b = x_b,
                     uF = uF, statsF = statsF, vg = vg, h = h, yF = yF, x_in = x_in, x_in_b = x_in_b, has_skip = has_skip, first_half = first_half)
            st['layers'].append(L)
            x_in, x_in_b = xr, xrb
        st['hid'] = hid
        st['x_last'] = x_in

        # ---- final RMSNorm (T.py:1250) + compaction of modality rows
        out = self.buf(f'{tag}out', (M, D), F32)
        outb = self.buf(f'{tag}outb', (M, D), BF16)
        omod = self.buf(f'{tag}omod', (max(S, 1), D), BF16)
        o.rmsnorm_fwd(x_in, self.P('transformer.norm.gamma'), out, outb, dv['slot'] if S > 0 else None, omod if S > 0 else None, M, D)
        if self.clean and S > 0:                        # model predicts the clean modality in model space (MP.py:100-126): flow = (embed - noised tokens) / max(1 - t, eps)
            o.clean_flow_fwd(out, dv['row_token'], modtok, dv['cond_times'], dv['cond_row'], self.clean_eps, omod, S, D)
        st.update(out = out, outb = outb, omod = omod)
        res = dict(embed = out)
        if rep_layer is not None:
            h = (*hid, out)[rep_layer]
            if train and h.dtype != F32:                 # the predictor head's RMSNorm reads fp32 rows
                h = self.buf('rep_f32', (M, D), F32).copy_(h)
            st['rep_layer'] = rep_layer
            res['rep'] = h

        # ---- heads
        if want_logits or train:
            logits = self.buf(f'{tag}logits', (M, self.Vp), F32)
            o.gemm_store(outb, D, 0, pk['wvocab'], D, 0, M, self.V, D, logits, self.Vp, None, 0, None, None, 1.0, 0, 1)
            res['logits'] = logits
            st['logits'] = logits
        preds = []
        if S > 0 and (train or want_preds):
            for t, (s0, s1) in enumerate(rb.type_rows):
                n = s1 - s0
                if n == 0:
                    preds.append(None); continue
                dl = self.dls[t]
                pred = self.buf(f'{tag}pred{t}', (n, dl), F32)
                o.gemm_store(omod[s0:s1], D, 0, pk[f'wm2l{t}'], D, 0, n, dl, D, pred, dl, None, 0, None, None, 1.0, 0, 1)
                preds.append(pred)
            res['preds'] = preds
        if train:
            T = float(rb.total_tokens)
            acc = self.buf('lossacc', (2 + len(self.dls),), torch.float64)
            acc.zero_()
            nvalid = self.buf('nvalid', (1,), I32); nvalid.zero_()
            dlog = self.buf('dlogits', (M, self.Vp), BF16)
            if modality_only:
                dlog.zero_()
            else:
                gs = (text_loss_weight / T) if vlimit == 0 else 1.0 / max(rb.n_valid, 1)
                o.ce_fwd_bwd(logits, self.Vp, dv['label'], self.V, vlimit, gs, dlog, self.Vp, acc[0:1], nvalid, M)
            st['dlogits'] = dlog
            st['dpred'] = []
            flow_terms = []
            vel_terms = {}
            recon_on = recon_weight > 0.
            recon_terms = {}
            if recon_on:
                assert 'inst_w' in dv, 'the reconstruction loss needs the batch packed for a model with reconstruction_loss_weight > 0'
                rsum = self.buf('reconacc', (len(self.dls),), torch.float64); rsum.zero_()
                rinst = self.buf('reconinst', (S,), torch.float64); rinst.zero_()       # per-instance sums of squares, sized by S (graph signature)
            def flow_grad(t, target, G, sumsq, dpred, n, dl, dlp):
                s0 = rb.type_rows[t][0]
                if not recon_on:
                    o.mse_fwd_bwd(preds[t], dl, target, dpred, dlp, G, sumsq, n, dl)
                    return
                g = recon_g[t] if recon_g is not None and recon_g[t] is not None else st['flow'][t]
                rs = 2.0 * recon_weight * wt / dl
                o.mse_recon_fwd_bwd(preds[t], dl, target, g, dv['row_time'][s0:s0 + n], 0 if modality_only else 1, dv['row_inst'][s0:s0 + n], dv['inst_w'],
                                    dpred, dlp, G, rs, sumsq, rinst, rsum[t:t + 1], n, dl)
                recon_terms[t] = (rsum[t] / dl).float()
            for t, (s0, s1) in enumerate(rb.type_rows):
                n = s1 - s0
                if n == 0 or st['flow'][t] is None:
                    st['dpred'].append(None); flow_terms.append(None); continue
                dl, dlp = self.dls[t], self.dlp[t]
                wt = 1.0 if modality_only else rb.n_type_tokens[t] / T
                dpred = self.buf(f'dpred{t}', (n, dlp), BF16)
                if dlp != dl:
                    dpred[:, dl:].zero_()
                ga = 2.0 * flow_loss_weight * wt / (n * dl)
                if vel_targets is not None and vel_targets[t] is not None and not vel_grad:
                    # value only: mse(flow, target) (forward_modality's velocity term carries no gradient, T.py:2834)
                    vacc = self.buf('velacc', (len(self.dls),), torch.float64)
                    if not vel_terms:
                        vacc.zero_()
                    o.mse_fwd_bwd(vel_targets[t], dl, st['flow'][t], None, dlp, 0., vacc[t: t + 1], n, dl)
                    vel_terms[t] = (vacc[t] / (n * dl)).float()
                    flow_grad(t, st['flow'][t], ga, acc[1 + t: 2 + t], dpred, n, dl, dlp)
                elif vel_targets is not None and vel_targets[t] is not None and vel_weight != 0.:
                    # velocity consistency (T.py:3383-3418): + w_v * wt * mse(pred, ema_pred).  d/dpred of a |p - f|^2 + b |p - e|^2 is
                    # (a + b) (p - (a f + b e) / (a + b)): ONE gradient pass against the blended target; the two loss values come from two
                    # loss-only passes (their dpred output is overwritten by the blended pass)
                    e = vel_targets[t]
                    assert e.shape == (n, dl) and e.dtype == F32
                    gb = 2.0 * vel_weight * wt / (n * dl)
                    vacc = self.buf('velacc', (len(self.dls),), torch.float64)
                    if t == 0 or not vel_terms:
                        vacc.zero_()
                    o.mse_fwd_bwd(preds[t], dl, e, None, dlp, gb, vacc[t: t + 1], n, dl)
                    o.mse_fwd_bwd(preds[t], dl, st['flow'][t], None, dlp, ga, acc[1 + t: 2 + t], n, dl)
                    blend = self.buf(f'velblend{t}', (n, dl), F32)
                    blend.zero_()
                    o.axpy_f32(blend, st['flow'][t], ga / (ga + gb), n * dl)
                    o.axpy_f32(blend, e, gb / (ga + gb), n * dl)
                    scratch = self.buf('velscratch', (1,), torch.float64)
                    flow_grad(t, blend, ga + gb, scratch, dpred, n, dl, dlp)
                    vel_terms[t] = (vacc[t] / (n * dl)).float()
                else:
                    flow_grad(t, st['flow'][t], ga, acc[1 + t: 2 + t], dpred, n, dl, dlp)
                st['dpred'].append(dpred)
                flow_terms.append((acc[1 + t] / (n * dl)).float() )
            # loss assembly on a handful of device scalars (no host sync): transfusion.py:3331-3376
            # mean CE over the valid labels: the count comes from the device (ce_fwd_bwd counts them), so the launch sequence does not
            # depend on how many labels classifier-free-guidance dropout nulled in this batch (CUDA-graph replay across batches)
            text = (acc[0] / nvalid[0].clamp(min = 1)).float()
            flows = torch.stack([f if f is not None else torch.zeros((), device = self.device) for f in flow_terms]) if flow_terms else torch.zeros(0, device = self.device)
            if vlimit:
                total = text.clone()         # distinct tensor: autograd.Function outputs must not alias each other
            elif modality_only:
                total = flows.sum()
                for t, f in vel_terms.items():
                    total = total + f * vel_weight
                for t, r in recon_terms.items():
                    total = total + r * recon_weight
            else:
                total = (acc[0] / T).float() * text_loss_weight          # = text * (n_valid / T) * w  (T.py:3331, 3371)
                for t, f in enumerate(flow_terms):
                    if f is not None:
                        total = total + f * (rb.n_type_tokens[t] / T) * flow_loss_weight
                for t, f in vel_terms.items():
                    total = total + f * (rb.n_type_tokens[t] / T) * vel_weight
                for t, r in recon_terms.items():
                    total = total + r * (rb.n_type_tokens[t] / T) * recon_weight
            vel = [vel_terms.get(t, torch.zeros((), device = self.device)) for t in range(len(self.dls))] if vel_terms else None
            res.update(loss_acc = acc, n_valid = nvalid, total = total, text = text, flows = flows, vel = vel)
            if recon_on:
                res.update(recon = [recon_terms.get(t, torch.zeros((), device = self.device)) for t in range(len(self.dls))], recon_inst = rinst)
        return res

    def dropout_key(self, src = None, out: Tensor | None = None) -> Tensor:
        """Device key (int32 [2] holding the two u32 words) of a forward's dropout masks (csrc/dropout.cuh).  `src` None: drawn from torch's
        CUDA generator, so `torch.manual_seed` reproduces a run; (k0, k1): those words (deterministic runs); a device int32 [2] tensor: used
        as is.  `out`: the int32 [2] device tensor to fill instead of the engine's own (a captured step graph's static input)."""
        if torch.is_tensor(src):
            assert src.dtype == I32 and src.numel() == 2 and src.device == self.device, 'a dropout key tensor is int32 [2] on the engine device'
            return src
        key = out if out is not None else self.buf('drop_key', (2,), I32)
        if src is None:
            key.random_(-2 ** 31, 2 ** 31)
        else:
            key.copy_(torch.from_numpy(np.array(src, dtype = np.uint32).view(np.int32)))
        return key

    def _prepare_grads(self):
        """`.grad` of every trainable parameter must be its view of the flat gradient buffer (kernels accumulate there)."""
        missing = [(n, p) for n, p in self.named.items() if p.grad is None or p.grad.data_ptr() != self.gflat.data_ptr() + 4 * self.offs[n]]
        if not missing:
            return
        if len(missing) == len(self.named):
            self.gflat.zero_()
        for n, p in missing:
            gv = self.G(n)
            if len(missing) != len(self.named):
                gv.zero_()
            if p.grad is not None:
                gv.copy_(p.grad)
            p.grad = gv

    # ------------------------------------------------------------------ backward
    def backward(self, gscale = None, bucket_cb = None, g_rep = None):
        """Backward of the last train forward: gradients are ACCUMULATED into the flat gradient buffer
        (`param.grad` views).  All weight gradients are split-K wgmma GEMMs over the token dimension.
        `gscale`: device scalar d(loss) handed in by autograd (folded into the head gradients, no host sync).
        `bucket_cb(layer)`: called after the kernels of a layer have been enqueued (gradient bucket ready).
        `g_rep`: fp32 [M, D] gradient of the hidden state the forward handed out (`rep_layer`), added where that state's gradient is complete."""
        st = self.state
        assert st['train'], 'backward() needs a train forward'
        rep_at = None
        if g_rep is not None:
            rep_at = st.get('rep_layer')
            assert rep_at is not None and g_rep.dtype == F32 and g_rep.is_contiguous() and g_rep.shape == (st['rb'].M, self.D), 'g_rep: fp32 [M, D] of a rep_layer forward'
        self._prepare_grads()
        self._grads_clean = False
        self._dirty = True                      # an optimizer step (ours or torch.optim's) normally follows
        if gscale is not None:
            gs = gscale.detach().float().reshape(1)
            self.ops.scale_bf16(st['dlogits'], gs, st['dlogits'].numel())
            for dp in st['dpred']:
                if dp is not None:
                    self.ops.scale_bf16(dp, gs, dp.numel())
        rb, dv = st['rb'], st['rb'].dev
        o, D, HI, H, Ip, M, inner = self.ops, self.D, self.HI, self.H, self.Ip, st['rb'].M, self.inner
        pk, nc, S = self.packed, rb.n_cond, rb.S
        cond_row = dv['cond_row'] if nc > 0 else None
        tab_ld, zg_ld = self.W * 3 * D, self.W * D
        ks = max(1, min(64, M // 2048))           # split-K cap of the latent_to_model wgrads (K = that modality's tokens)
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        def ksplit(n_out, n_in, K = M):
            return wgrad_splits(n_out, n_in, K, sms)
        def wgrad(dy, ld_dy, n_out, act, ld_act, n_in, gname, K = M):
            # dW[n_out, n_in] += dy^T act : both operands MN-major over the token (K) dimension, split-K atomics
            o.gemm_store(dy, ld_dy, 1, act, ld_act, 1, n_out, n_in, K, self.G(gname), n_in, None, 0, None, None, 1.0, 1, ksplit(n_out, n_in, K))

        # ---- heads
        dlog = st['dlogits']
        d_out = self.buf('d_out', (M, D), F32)
        o.gemm_store(dlog, self.Vp, 0, pk['wvocab'], D, 1, M, D, self.V, d_out, D, None, 0, None, None, 1.0, 0, 1)
        wgrad(dlog, self.Vp, self.V, st['outb'], D, D, 'to_text_logits.weight')
        if S > 0:
            dmod = self.buf('dmod', (S, D), F32)
            any_flow = False
            for t, (s0, s1) in enumerate(rb.type_rows):
                n = s1 - s0
                dp = st['dpred'][t] if n else None
                if dp is None:
                    if n:
                        dmod[s0:s1].zero_()
                    continue
                any_flow = True
                dl, dlp = self.dls[t], self.dlp[t]
                o.gemm_store(dp, dlp, 0, pk[f'wm2l{t}'], D, 1, n, D, dl, dmod[s0:s1], D, None, 0, None, None, 1.0, 0, 1)
                wgrad(dp, dlp, dl, st['omod'][s0:s1], D, D, f'model_to_latent_projs.{t}.weight', K = n)
            dneg = None
            if any_flow and self.clean:
                dneg = self.buf('dmod_neg', (S, D), F32)
                o.clean_flow_bwd(dmod, dneg, dv['row_token'], dv['cond_times'], dv['cond_row'], self.clean_eps, S, D)
            if any_flow:
                o.scatter_add_rows(d_out, dmod, dv['row_token'], S, D)
        if rep_at == self.depth + 1:
            o.axpy_f32(d_out, g_rep, 1.0, M * D)
        g = self.buf('gx', (M, D), F32)
        o.rmsnorm_bwd(d_out, st['x_last'], self.P('transformer.norm.gamma'), g, self.G('transformer.norm.gamma'), M, D)

        # ---- block stack, reverse
        hid = st['hid']
        dH = [self.buf(f'dH{l}', (M, D), F32) for l in range(self.depth + 1)]     # each written once, by the attn_residual_bwd2 that assembles it
        dskip = {}
        if nc > 0:
            dtab = self.buf('dtab', (nc, self.W * 3 * D), F32); dtab.zero_()
            dzg = self.buf('dzg', (nc, self.W * D), F32); dzg.zero_()
        dy = self.buf('dy', (M, D), BF16)
        du = self.buf('du', (M, D), F32)
        arws = self.buf('attn_res_ws', (int(o.lib.tfx_attn_residual_bwd_workspace_floats(M, D)),), F32)
        sc_stride = (self.depth + 2) * 3
        arsc = self.buf('attn_res_sc', (self.depth, M, self.depth + 2, 3), F32)
        dxs = {}
        for i in reversed(range(self.depth)):
            L = st['layers'][i]
            pre = f'transformer.layers.{i}'
            lm = self.layer_maps[i]
            wA, wF = 2 * i, 2 * i + 1
            # complete gradient of x_c of THIS layer (hidden i + 1), assembled once from this layer's term and the stored scalars / incoming gradients of the
            # later AttentionResiduals; the scalars for the earlier hiddens are stored for their own assembly further down the stack
            dxs[i] = g
            later = list(range(i + 1, self.depth))
            gam = [self.P(f'transformer.layers.{j}.3.norm_keys.gamma') for j in [i] + later]
            pqs = [self.P(f'transformer.layers.{j}.3.pseudo_queries') for j in [i] + later]
            o.attn_residual_bwd2(self._ptr_array(hid[:i + 2]), i + 2, 1, self._ptr_array(gam), self._ptr_array(pqs), self._ptr_array([dxs[j] for j in later] or [g]),
                                 self._ptr_array([arsc[j][0, i + 1] for j in later] or [g]), len(later), g, L['xr'], L['rlse'], dH[i + 1], arsc[i], sc_stride,
                                 self.G(f'{pre}.3.norm_keys.gamma'), self.G(f'{pre}.3.pseudo_queries'), arws, M, D)
            gx = dH[i + 1]                       # complete gradient w.r.t. x_c of this layer; updated in place below
            if rep_at == i + 1:
                o.axpy_f32(gx, g_rep, 1.0, M * D)
            # -- feed-forward branch
            o.resid_bwd(gx, L['yF'], cond_row, st['zg'][:, wF * D:] if nc > 0 else None, zg_ld, self.P(f'{pre}.2.layerscale'), dy,
                        dzg[:, wF * D:] if nc > 0 else None, zg_ld, self.G(f'{pre}.2.layerscale'), self.G(f'{pre}.2.fn.net.3.bias'), M, D)
            dh = self.buf('dh', (M, Ip), BF16)
            o.gemm_store(dy, D, 0, pk[f'w2{i}'], Ip, 1, M, Ip, D, None, 0, dh, Ip, None, None, 1.0, 0, 1)
            o.gemm_store(dy, D, 1, L['h'], Ip, 1, D, inner, M, self.gflat, 0, None, 0, None, lm['w2_rows'], 1.0, 1, ksplit(D, inner))
            dvg = self.buf('dvg', (M, 2 * Ip), BF16)
            rpb = self.ops.lib.tfx_geglu_bwd_rows_per_block()
            nblk = (M + rpb - 1) // rpb
            part = self.buf('geglu_part', (nblk, 2 * Ip), F32)
            if st['p_ff'] > 0.:
                o.geglu_bwd_drop(dh, L['vg'], dvg, M, Ip, None, None, part, st['drop_key'], st['p_ff'], i)
            else:
                o.geglu_bwd(dh, L['vg'], dvg, M, Ip, None, None, part)
            o.colsum_f32(part, 2 * Ip, nblk, 2 * Ip, lm['b1_cols'], self.gflat)
            o.gemm_store(dvg, 2 * Ip, 0, pk[f'w1{i}'], D, 1, M, D, 2 * Ip, du, D, None, 0, None, None, 1.0, 0, 1)
            o.gemm_store(dvg, 2 * Ip, 1, L['uF'], D, 1, 2 * Ip, D, M, self.gflat, 0, None, 0, None, lm['w1_rows'], 1.0, 1, ksplit(2 * Ip, D))
            o.adaln_bwd(du, L['x_b'], L['statsF'], cond_row, st['tab'][:, wF * 3 * D:] if nc > 0 else None, tab_ld, self.P(f'{pre}.2.layernorm_gamma'), gx,
                        dtab[:, wF * 3 * D:] if nc > 0 else None, tab_ld, self.G(f'{pre}.2.layernorm_gamma'), M, D)
            # -- attention branch
            o.resid_bwd(gx, L['yA'], cond_row, st['zg'][:, wA * D:] if nc > 0 else None, zg_ld, self.P(f'{pre}.1.layerscale'), dy,
                        dzg[:, wA * D:] if nc > 0 else None, zg_ld, self.G(f'{pre}.1.layerscale'), None, M, D)
            dog = self.buf('dog', (M, HI), BF16)
            o.gemm_store(dy, D, 0, pk[f'wo{i}'], HI, 1, M, HI, D, None, 0, dog, HI, None, None, 1.0, 0, 1)
            wgrad(dy, D, D, L['att'], HI, HI, f'{pre}.1.fn.to_out.1.weight')
            dop = self.buf('dop', (M, HI), BF16); dsum_hm = self.buf('dsum_hm', (H, M), F32); dsum_mh = self.buf('dsum_mh', (M, H), F32) if self.gated else None
            dq = self.buf('dq', (M, HI), F32); dk = self.buf('dk', (M, HI), F32)
            if self.laser:
                getattr(o, 'laser_bwd_prep' + self.sfx)(dog, L['o_l'], L['gates'], dop, dsum_hm, dsum_mh, dq, M, H)
            else:
                getattr(o, 'attn_bwd_prep' + self.sfx)(dog, L['att'], L['gates'], dop, dsum_hm, dsum_mh, dq, M, H)
            dqkvg = self.buf('dqkvg', (M, self.NQ), BF16)
            if i == self.depth - 1 and self.gate_tile:
                # pad columns (and the gate columns of an ungated model) are never written by the kernels; cleared once per backward (inside
                # captured graphs too)
                dqkvg[:, 3 * HI + (H if self.gated else 0):].zero_()
            fp = self.fastp[i] if self.fast else None
            if self.fast:
                o.attn_bwd_tc(L['q'], L['k'], L['v_att'], dop, HI, HI, HI, HI, L['lse'], dsum_hm, dv['kv_limit'], dv['k2_kv0'], dv['k2_kvend'], dv['k2_q0'], dv['k2_qend'],
                              dv['k2_order'], int(rb.k2_kv0.shape[0]), dq, dk, dqkvg[:, 2 * HI:], self.NQ, M, H, self.scale, self.softcap, fp)
            if self.d128:
                o.attn_bwd_d128(L['q'], L['k'], L['v_att'], dop, HI, HI, HI, HI, L['lse'], dsum_hm, dv['kv_limit'], dv['kt_kv0'], dv['kt_kvend'], dv['kt_q0'],
                                dv['kt_qend'], int(rb.kt_kv0.shape[0]), dq, dk, dqkvg[:, 2 * HI:], self.NQ, M, H, self.scale, self.softcap)
            else:
                o.attn_bwd(L['q'], L['k'], L['v_att'], dop, HI, HI, HI, HI, L['lse'], dsum_hm, dv['kv_limit'], dv['kt_kv0'], dv['kt_kvend'], dv['kt_q0'], dv['kt_qend'],
                           int(rb.kt_kv0.shape[0]), dq, dk, dqkvg[:, 2 * HI:], self.NQ, M, H, self.scale, self.softcap, fp)
            dv_cols = dqkvg[:, 2 * HI:]
            if self.laser:                               # d v' -> d v (v' = exp(softclamp(v)))
                o.laser_v_bwd(dv_cols, self.NQ, L['v'], HI, M, self.vheads, self.laser_clamp)
            if self.vres:
                dv0 = self.buf('dv_first', (M, HI), F32)
                if i == self.depth - 1:
                    dv0.zero_()
                if i > 0:                                # d v_mixed -> d v_raw; the first layer's share accumulates in dv0, d mix_pre goes to the packed column block
                    getattr(o, 'vmix_bwd' + self.sfx)(dv_cols, self.NQ, L['v'], HI, st['layers'][0]['v'], HI, L['mixpre'], self.P(f'{pre}.1.fn.to_learned_value_residual.0.bias'), dv0,
                               dqkvg[:, self.MIX:], self.NQ, M, H)
                    o.colsum_bf16(dqkvg[:, self.MIX:], self.NQ, M, H, None, self.G(f'{pre}.1.fn.to_learned_value_residual.0.bias'))
                else:
                    dqkvg[:, self.MIX:self.MIX + H].zero_()      # the first layer has no mix Linear: its column block must not carry layer 1's values
                    o.add_f32_into_bf16(dv_cols, self.NQ, dv0, HI, M, HI)
            if self.qk_norm:
                getattr(o, 'qk_bwd_pack' + self.sfx)(dq, dk, L['q'], L['k'], L['qk_inv'], self.P(f'{pre}.1.fn.q_norm.gamma'), self.P(f'{pre}.1.fn.k_norm.gamma'), dv['rope_pos'],
                              self.ws['rope_cs'], L['gates'], dsum_mh, dqkvg, self.NQ, self.G(f'{pre}.1.fn.q_norm.gamma'), self.G(f'{pre}.1.fn.k_norm.gamma'), M, H)
            else:
                getattr(o, 'qk_bwd_pack_rope' + self.sfx)(dq, dk, dv['rope_pos'], self.ws['rope_cs'], L['gates'], dsum_mh, dqkvg, self.NQ, M, H)
            o.gemm_store(dqkvg, self.NQ, 0, pk[f'qkvg{i}'], D, 1, M, D, self.NQ, du, D, None, 0, None, None, 1.0, 0, 1)
            o.gemm_store(dqkvg, self.NQ, 1, L['uA'], D, 1, self.NQ, D, M, self.gflat, 0, None, 0, None, lm['qkvg_rows'], 1.0, 1, ksplit(self.NQ, D))
            o.adaln_bwd(du, L['x_a'], L['statsA'], cond_row, st['tab'][:, wA * 3 * D:] if nc > 0 else None, tab_ld, self.P(f'{pre}.1.layernorm_gamma'), gx,
                        dtab[:, wA * 3 * D:] if nc > 0 else None, tab_ld, self.G(f'{pre}.1.layernorm_gamma'), M, D)
            # -- U-Net skip projection: x_a = x_in + W_skip [x_in | skip]
            if L['has_skip']:
                o.resid_bwd(gx, None, None, None, 0, None, dy, None, 0, None, None, M, D)
                wsk = pk[f'wskip{i}']
                gw = self.G(f'{pre}.0.weight')
                o.gemm_store(dy, D, 1, L['x_in_b'], D, 1, D, D, M, gw, 2 * D, None, 0, None, None, 1.0, 1, ksplit(D, D))
                o.gemm_store(dy, D, 1, L['skip_b'], D, 1, D, D, M, gw.view(-1)[D:], 2 * D, None, 0, None, None, 1.0, 1, ksplit(D, D))
                src = L['skip_src']
                assert src not in dskip                   # every skip source feeds exactly one skip projection: plain store, no zero fill
                dskip[src] = self.buf(f'dskip{src}', (M, D), F32)
                o.gemm_store(dy, D, 0, wsk[:, D:], 2 * D, 1, M, D, D, dskip[src], D, None, 0, None, None, 1.0, 0, 1)
                o.gemm_store(dy, D, 0, wsk, 2 * D, 1, M, D, D, gx, D, None, 0, None, None, 1.0, 1, 1)
            if i in dskip:
                o.axpy_f32(gx, dskip[i], 1.0, M * D)
            g = gx
            if bucket_cb is not None:
                bucket_cb(i)
        # ---- input side: gradient w.r.t. x0 = path gradient + AttentionResidual contributions to H[0]
        allj = list(range(self.depth))                   # gradient of the input embedding x0 through all AttentionResiduals: assembly only
        gam = [self.P(f'transformer.layers.{j}.3.norm_keys.gamma') for j in [0] + allj]
        pqs = [self.P(f'transformer.layers.{j}.3.pseudo_queries') for j in [0] + allj]
        o.attn_residual_bwd2(self._ptr_array(hid[:1]), 1, 0, self._ptr_array(gam), self._ptr_array(pqs), self._ptr_array([dxs[j] for j in allj]),
                             self._ptr_array([arsc[j][0, 0] for j in allj]), len(allj), None, None, None, dH[0], None, sc_stride, None, None, None, M, D)
        o.axpy_f32(g, dH[0], 1.0, M * D)
        if rep_at == 0:
            o.axpy_f32(g, g_rep, 1.0, M * D)
        dmodtok = self.buf('dmodtok', (max(S, 1), D), BF16)
        o.embed_bwd(g, dv['text_id'], dv['slot'] if S > 0 else None, self.G('text_embed.weight'), dmodtok if S > 0 else None, M, D)
        if S > 0:
            if self.clean and dneg is not None:           # the clean-prediction flow also depends on the (projected) noised tokens
                o.add_f32_into_bf16(dmodtok, D, dneg, D, S, D)
            for t, (tabs, coords) in st.get('posemb', {}).items():      # axial positional embedding: the rows' gradient is the table gradient, scattered by coordinate
                s0, s1 = rb.type_rows[t]
                nax = len(tabs)
                posemb_backward(dmodtok[s0:s1].float(), tabs, coords, self._posemb_params(t, nax), self._posemb_params(t, nax, grads = True))
            for t, (s0, s1) in enumerate(rb.type_rows):
                n = s1 - s0
                if n == 0 or f'latent_to_model_projs.{t}.weight' not in self.named:
                    continue
                dl, dlp = self.dls[t], self.dlp[t]
                o.gemm_store(dmodtok[s0:s1], D, 1, st['noised'][t], dlp, 1, D, dl, n, self.G(f'latent_to_model_projs.{t}.weight'), dl, None, 0, None, None, 1.0, 1,
                             max(1, min(ks, n // 128)))
                o.colsum_bf16(dmodtok[s0:s1], D, n, D, None, self.G(f'latent_to_model_projs.{t}.bias'))
        # ---- conditioning path
        if nc > 0:
            W3 = self.W * 3 * D
            for w in range(self.W):
                o.table_op(dzg[:, w * D:], zg_ld, st['zg'][:, w * D:], zg_ld, dtab[:, w * 3 * D + 2 * D:], W3, None, 0, nc, D, 2)
            dtabb = self.buf('dtabb', (nc, W3), BF16)
            o.cast_bf16(dtab, dtabb, nc * W3)
            dcond = self.buf('dcond', (nc, 4 * D), F32)
            o.gemm_store(dtabb, W3, 0, pk['wfz'], 4 * D, 1, nc, 4 * D, W3, dcond, 4 * D, None, 0, None, None, 1.0, 0, 1)
            o.gemm_store(dtabb, W3, 1, st['cond'], 4 * D, 1, W3, 4 * D, nc, self.gflat, 0, None, 0, None, self.fz_rows, 1.0, 1, 1)
            bsum = self.buf('bsum', (W3,), F32); bsum.zero_()
            o.colsum_f32(dtab, W3, nc, W3, None, bsum)
            self.gflat.index_add_(0, self.fz_bias_idx, bsum)
            dcpre = self.buf('dcpre', (nc, 4 * D), BF16)
            o.table_op(dcond, 4 * D, st['cpre'], 4 * D, None, 0, dcpre, 4 * D, nc, 4 * D, 3)
            o.gemm_store(dcpre, 4 * D, 1, st['feats'], self.Kt, 1, 4 * D, D + 1, nc, self.gflat, 0, None, 0, None, self.wt_rows, 1.0, 1, 1)
            o.colsum_bf16(dcpre, 4 * D, nc, 4 * D, None, self.G('transformer.to_time_cond.1.bias'))

    # ------------------------------------------------------------------ kv-cache decode (sampling.py drives these)
    def new_cache(self, n_slabs: int, cap: int) -> KVCache:
        self.ensure_attached()
        return KVCache(self, n_slabs, cap)

    def text_decoder(self, cache, S, **kw):
        from .decode import TextDecoder
        return TextDecoder(self, cache, S, **kw)

    def ode_solve(self, cache, rb, y, **kw):
        from .decode import ode_solve
        return ode_solve(self, cache, rb, y, **kw)

    # ------------------------------------------------------------------ optimizer
    def zero_grad(self):
        if not getattr(self, '_grads_clean', False):
            self.gflat.zero_()
        self._grads_clean = False       # whoever asked for clean gradients is about to write them

    def clip_grad_norm_(self, max_norm: float, pre_scale: float = 1.0):
        """torch.nn.utils.clip_grad_norm_ over the flat gradient buffer, entirely on the device (no host sync).  `pre_scale` = 1/world when
        the buffer holds the all-reduced sum.  Returns the (unclipped) total norm as a device tensor."""
        ss = self.buf('gnorm_ss', (1,), torch.float64)
        ss.zero_()
        n = self.gflat.numel()
        self.ops.grad_sumsq(self.gflat, n, ss)
        self.ops.clip_by_norm(self.gflat, n, ss, float(max_norm), float(pre_scale))
        return ss.sqrt() * pre_scale

    def ema_update(self, decay: float):
        """EMA copy of all trainable parameters (one flat buffer, same layout as the master parameters)."""
        if getattr(self, 'ema_flat', None) is None or self.ema_flat.numel() != self.flat.numel():
            self.ema_flat = self.flat.clone()
            return
        self.ops.ema_update(self.ema_flat, self.flat, self.flat.numel(), float(decay))

    def ema_state_dict(self):
        assert getattr(self, 'ema_flat', None) is not None, 'no EMA update has run yet'
        return {n: self.ema_flat[o:o + self.named[n].numel()].view(self.named[n].shape) for n, o in self.offs.items()}

    def adam_step(self, lr = 1e-3, betas = (0.9, 0.999), eps = 1e-8, weight_decay = 0., decoupled = False, grad_scale = 1.0, zero_grads = False, device_step = False):
        """zero_grads: clear the flat gradient buffer in the same pass (saves a separate fill); the next `zero_grad()` is then free."""
        if self.exp_avg is None:
            self.exp_avg = torch.zeros_like(self.flat); self.exp_avg_sq = torch.zeros_like(self.flat)
        self.opt_step += 1
        step_dev = None
        if device_step:                         # CUDA-graph replays: the step counter lives on the device (the caller keeps it equal to opt_step - 1)
            assert getattr(self, 'opt_step_dev', None) is not None, 'device_step needs engine.opt_step_dev (int32 [1] on the device)'
            step_dev = self.opt_step_dev
        self.ops.adam_step(self.flat, self.gflat, self.exp_avg, self.exp_avg_sq, self.flat.numel(), lr, betas[0], betas[1], eps, weight_decay, int(decoupled),
                           self.opt_step, grad_scale, int(zero_grads), step_dev)
        self._grads_clean = bool(zero_grads)
        self._dirty = True


class RepHead:
    """Self-Flow predictor head and representation loss (`SelfMaskedRepTraining`, T.py:3490-3493, 3455-3460, 3556-3559) on the kernels of the
    block stack, in the student engine's workspaces:  u = RMSNorm(x) (final-norm row kernel) -> GEGLU GEMM epilogue -> a = W2 h + b2 ->
    loss = 1 - mean cos(a, teacher rows) with da in the same pass (tfx_rep_cos_fwd_bwd).  `head` is `Sequential(RMSNorm, FeedForward)` with the
    reference's parameter names (`0.gamma`, `1.net.0.*`, `1.net.3.*`); its gradients accumulate into the parameters' `.grad`."""

    def __init__(self, engine: Engine, head):
        self.eng, self.head = engine, head
        self._ptrs = None

    def _prepare(self):
        head, dev = self.head, self.eng.device
        gamma, w1, b1, w2, b2 = head[0].gamma, head[1].net[0].weight, head[1].net[0].bias, head[1].net[3].weight, head[1].net[3].bias
        ptrs = tuple(p.data_ptr() for p in (gamma, w1, b1, w2, b2))
        if ptrs != self._ptrs:
            D, inner = w1.shape[1], w2.shape[1]
            Ip = _round_up(inner, 64)
            assert w1.is_cuda and all(p.dtype == F32 and p.is_contiguous() for p in (gamma, w1, b1, w2, b2)), 'the predictor head must hold contiguous fp32 cuda parameters'
            src = w1_row_src(inner)
            src32 = torch.from_numpy(src.astype(np.int32)).to(dev)
            self.w1p = torch.zeros(2 * Ip, D, device = dev, dtype = BF16)
            self.w2p = torch.zeros(D, Ip, device = dev, dtype = BF16)
            self.b1p = torch.zeros(2 * Ip, device = dev, dtype = F32)
            jobs = [(w1, D, D, src32, self.w1p, 2 * Ip, D, 0), (w2, inner, inner, None, self.w2p, D, Ip, 0), (b1, 1, 1, src32, self.b1p, 2 * Ip, 1, 1)]
            self.pack = pack_job_table(jobs, dev)
            self.b1_cols = src32
            self.w1_rows = torch.from_numpy(np.where(src >= 0, src * D, -1)).to(dev)
            self.w2_rows = torch.from_numpy(np.arange(D, dtype = np.int64) * inner).to(dev)
            self.D, self.inner, self.Ip, self._ptrs = D, inner, Ip, ptrs
        return gamma, b2

    def forward(self, x: Tensor, teacher: Tensor, g: Tensor) -> Tensor:
        """x: fp32 [M, D] student rows; teacher: bf16 / fp32 [M, D] rows; g: fp32 [1] device scalar d(total)/d(loss) the gradient is computed
        for.  Returns the loss (fp32 device scalar, mean over the M rows)."""
        eng, o = self.eng, self.eng.ops
        gamma, b2 = self._prepare()
        M, D, Ip = x.shape[0], self.D, self.Ip
        assert x.dtype == F32 and x.shape == teacher.shape == (M, D) and teacher.dtype in (F32, BF16) and x.is_contiguous() and teacher.is_contiguous()
        o.cast_pack_multi(*self.pack)
        u = eng.buf('rh_u', (M, D), BF16)
        o.rmsnorm_fwd(x, gamma, None, u, None, None, M, D)
        vg = eng.buf('rh_vg', (M, 2 * Ip), BF16); h = eng.buf('rh_h', (M, Ip), BF16)
        o.gemm_geglu(u, D, self.w1p, D, self.b1p, M, 2 * Ip, D, vg, h)
        a = eng.buf('rh_a', (M, D), F32)
        o.gemm_store(h, Ip, 0, self.w2p, Ip, 0, M, D, Ip, a, D, None, 0, b2, None, 1.0, 0, 1)
        da = eng.buf('rh_da', (M, D), BF16)
        part = eng.buf('rh_part', (int(o.lib.tfx_rep_cos_blocks(M)),), torch.float64)
        ticket = eng.buf('rh_ticket', (1,), I32, zero = True)
        loss = eng.buf('rh_loss', (1,), F32)
        o.rep_cos_fwd_bwd(a, teacher, 1 if teacher.dtype == BF16 else 0, g, M, da, part, ticket, loss, M, D)
        self.state = dict(x = x, u = u, vg = vg, h = h, da = da, g = g, M = M)
        return loss[0].clone()

    def backward(self, g_loss: Tensor | None = None) -> Tensor:
        """Accumulates the head's parameter gradients; returns d(total)/dx (fp32 [M, D], an engine workspace).  `g_loss`: autograd's
        d(total)/d(loss) when it differs from the forward's `g` (da is rescaled by g_loss / g)."""
        eng, o, st = self.eng, self.eng.ops, self.state
        M, D, inner, Ip = st['M'], self.D, self.inner, self.Ip
        head = self.head
        params = [head[0].gamma, head[1].net[0].weight, head[1].net[0].bias, head[1].net[3].weight, head[1].net[3].bias]
        for p in params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        ggamma, gw1, gb1, gw2, gb2 = (p.grad for p in params)
        da = st['da']
        if g_loss is not None:
            o.scale_bf16(da, (g_loss.detach().float().reshape(1) / st['g']), da.numel())
        sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
        dh = eng.buf('rh_dh', (M, Ip), BF16)
        o.gemm_store(da, D, 0, self.w2p, Ip, 1, M, Ip, D, None, 0, dh, Ip, None, None, 1.0, 0, 1)
        o.gemm_store(da, D, 1, st['h'], Ip, 1, D, inner, M, gw2, 0, None, 0, None, self.w2_rows, 1.0, 1, wgrad_splits(D, inner, M, sms))
        o.colsum_bf16(da, D, M, D, None, gb2)
        dvg = eng.buf('rh_dvg', (M, 2 * Ip), BF16)
        rpb = o.lib.tfx_geglu_bwd_rows_per_block()
        nblk = (M + rpb - 1) // rpb
        part = eng.buf('rh_geglu_part', (nblk, 2 * Ip), F32)
        o.geglu_bwd(dh, st['vg'], dvg, M, Ip, None, None, part)
        o.colsum_f32(part, 2 * Ip, nblk, 2 * Ip, self.b1_cols, gb1)
        du = eng.buf('rh_du', (M, D), F32)
        o.gemm_store(dvg, 2 * Ip, 0, self.w1p, D, 1, M, D, 2 * Ip, du, D, None, 0, None, None, 1.0, 0, 1)
        o.gemm_store(dvg, 2 * Ip, 1, st['u'], D, 1, 2 * Ip, D, M, gw1, 0, None, 0, None, self.w1_rows, 1.0, 1, wgrad_splits(2 * Ip, D, M, sms))
        gx = eng.buf('rh_gx', (M, D), F32)
        o.rmsnorm_bwd(du, st['x'], head[0].gamma, gx, ggamma, M, D)
        return gx
