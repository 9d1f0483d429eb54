"""Host-side mirror of the reference's public API (`Transfusion`, `Transformer`) over the CUDA engine.

Same constructor keywords, method names, return conventions, special-token layout and - crucially -
the same `state_dict()` keys and shapes as lucidrains/transfusion-pytorch v0.19.4
(transfusion_pytorch/transfusion.py:1041-1097, 1290-1540), so reference checkpoints load here and vice
versa.  What differs is everything underneath: the modules below only OWN parameters; all arithmetic of
the block stack, attention, loss heads and optimizer runs in the sm_90a kernels of `libtfx_b200.so`
driven by `engine.Engine` over the ragged descriptor of `modality_processing.pack_batch`.

Out of scope here (raise loudly): U-Net pre/post encoders (`pre_post_transformer_enc_dec`), attention dropout, dim_head other than 64 or 128, a custom
`loss_fn` of `SelfMaskedRepTraining`.  `qk_rmsnorm = False` is supported: the q / k norm gammas are still built (same state-dict keys) and get
no gradient, as in the reference.
"""
from __future__ import annotations

import math
from functools import partial
from itertools import chain
from typing import Callable, NamedTuple

import numpy as np
import torch
from torch import nn, Tensor, tensor, is_tensor, cat
from torch.nn import Module, ModuleList

from .sampling import SamplingMixin
from ._pinned import POOL
from .modality_processing import (
    ModalitySample, RaggedBatch, pack_batch, pack_text_only, pack_incremental, get_processing_strategy, DEFAULT_PROCESSING_STRATEGY, is_int_tensor)

# Deepest model the AttentionResidual kernels take (TFX_MAX_DEPTH in include/tfx_b200.h): their hidden-state lists hold x0 and 64 layer outputs
MAX_DEPTH = 64
# Model widths the row kernels are built for: the cases of TFX_DISPATCH_NCH (csrc/common.cuh), D = 128 * NCH
MODEL_DIMS = (128, 256, 384, 512, 768, 1024, 1536, 2048)
# Heads the attention kernels take at dim_head 64: two heads per 128-column GEMM tile, at most 32 (an inner width of 2048, the widest the
# q / k backward pack and the row attention kernels are built for)
MIN_HEADS, MAX_HEADS = 2, 32
DIM_HEADS = (64, 128)                # attention head widths the kernels implement
MAX_HEADS_D128 = 16                  # heads at dim_head = 128 (inner width <= 2048, as at 64)


class TextKVCache:
    """Handle returned as the first element of the reference's `(kv_cache, tokens_seen)` tuple (T.py:2613, 2636): B cache slabs that grow in place."""

    def __init__(self, engine, B, cap):
        self.engine, self.B, self.length = engine, B, 0
        self.cache = engine.new_cache(B, cap)

    def reserve(self, n_new):
        need = self.length + n_new
        if need <= self.cache.cap:
            return
        old, cap = self.cache, max(2 * self.cache.cap, need + 64)
        new = self.engine.new_cache(self.B, cap)
        for name in ('k', 'v'):
            src, dst = getattr(old, name), getattr(new, name)
            dst.view(dst.shape[0], self.B, cap, *dst.shape[2:])[:, :, :old.cap].copy_(src.view(src.shape[0], self.B, old.cap, *src.shape[2:]))
        self.cache = new


class LossBreakdown(NamedTuple):
    total: Tensor
    text: Tensor
    flow: list
    velocity: list | None = None
    recon: list | None = None


def exists(v):
    return v is not None


def default(v, d):
    return v if exists(v) else d


def cast_tuple(t, length = 1):
    return t if isinstance(t, tuple) else ((t,) * length)


def default_to_modality_shape_fn(maybe_shape_str) -> tuple:
    return tuple(int(s) for s in maybe_shape_str.split(','))


def print_modality_sample(modality_sample):
    out = []
    for part in modality_sample:
        if isinstance(part, tuple):
            out.append((f'modality:{part[0]}', tuple(part[1].shape)))
        elif is_int_tensor(part):
            out.append(('text', tuple(part.shape)))
        else:
            out.append(('modality', tuple(part.shape)))
    print(out)


def _collate(data):
    return [list(d) for d in data]


def create_dataloader(dataset, **kwargs):
    from torch.utils.data import DataLoader
    return DataLoader(dataset, collate_fn = _collate, **kwargs)


# ------------------------------------------------------------------------------------------- text sampling helpers
def min_p_filter(logits, min_p = 0.1):
    probs = logits.softmax(dim = -1)
    limit = min_p * probs.amax(dim = -1, keepdim = True)
    return torch.where(probs < limit, float('-inf'), logits)


def sample_text_token(logits, temperature = 1.0, min_p = 0.1):
    if temperature == 0.:
        return logits.argmax(dim = -1, keepdim = True)
    logits = min_p_filter(logits / temperature, min_p = min_p)
    return torch.multinomial(logits.softmax(dim = -1), 1)


def default_modality_length_to_time_fn(num_modalities: Tensor) -> Tensor:
    """Past ("already decoded") modalities get t = 0.5, the rest share one uniform time per sample
    (transfusion.py:186-200)."""
    nm = num_modalities.float().cpu()
    total = int(nm.amax().item()) if nm.numel() else 0
    if total == 0:
        return torch.empty((nm.shape[0], 0))
    rand_num = torch.floor(torch.rand_like(nm) * nm)
    seq = torch.arange(total)
    prev = seq[None, :] < rand_num[:, None]
    cur = torch.rand_like(nm)
    return torch.where(prev, torch.tensor(0.5), cur[:, None].expand(-1, total))


# ------------------------------------------------------------------------------------------- parameter holders
class _Gamma(Module):
    """owns `gamma` of an RMSNorm (transfusion.py:779-786)"""
    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.zeros(dim))


class _Fourier(Module):
    def __init__(self, dim):
        super().__init__()
        assert dim % 2 == 0
        self.register_buffer('weights', torch.randn(dim // 2))       # persistent, as in transfusion.py:622


class _AttentionParams(Module):
    def __init__(self, dim, dim_head, heads, learned_value_residual_mix = False, gate_values = True):
        super().__init__()
        inner = dim_head * heads
        if learned_value_residual_mix:           # T.py:894-898 (layers after the first, `use_value_residual`)
            self.to_learned_value_residual = nn.Sequential(nn.Linear(dim, heads), nn.Sigmoid())
        self.to_qk = nn.Sequential(nn.Linear(dim, inner * 2, bias = False))
        self.q_norm, self.k_norm = _Gamma(dim_head), _Gamma(dim_head)
        self.to_v = nn.Sequential(nn.Linear(dim, inner, bias = False))
        if gate_values:                          # T.py:901-904: `gate_values = False` builds no to_gates
            self.to_gates = nn.Sequential(nn.Linear(dim, heads, bias = False))
        self.to_out = nn.Sequential(nn.Identity(), nn.Linear(inner, dim, bias = False))


class _FeedForwardParams(Module):
    def __init__(self, dim, inner):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(dim, inner * 2), nn.Identity(), nn.Identity(), nn.Linear(inner, dim))


class _AdaptiveParams(Module):
    """parameters of one AdaptiveWrapper (transfusion.py:640-669)"""
    def __init__(self, fn, dim, dim_cond, ada_ln_zero_init_bias = -2.):
        super().__init__()
        self.fn = fn
        self.layernorm_gamma = nn.Parameter(torch.zeros(dim))
        self.layerscale = nn.Parameter(torch.zeros(dim))
        self.to_film = nn.Linear(dim_cond, dim * 2)
        self.to_ada_ln_zero = nn.Linear(dim_cond, dim)
        nn.init.zeros_(self.to_film.weight)
        nn.init.zeros_(self.to_ada_ln_zero.weight)
        nn.init.constant_(self.to_ada_ln_zero.bias, ada_ln_zero_init_bias)


class _AttnResidualParams(Module):
    def __init__(self, dim):
        super().__init__()
        self.norm_keys = _Gamma(dim)
        self.pseudo_queries = nn.Parameter(torch.zeros(dim))
        nn.init.normal_(self.pseudo_queries, std = 0.02)


class _AxialPosEmb(Module):
    """parameters of `axial_positional_embedding.ContinuousAxialPositionalEmbedding(dim, num_axial_dims)` (T.py:1398-1401): one MLP
    `Linear(1, 2 dim) -> SiLU -> Linear(2 dim, dim)` per axis, evaluated on the integer coordinate and summed over the axes.  Holds the
    parameters only (state-dict layout `mlps.{axis}.{0,2}.{weight,bias}`); the engine evaluates the factorised tables."""
    def __init__(self, dim, num_axial_dims, mlp_expansion = 2.):
        super().__init__()
        self.num_axial_dims = num_axial_dims
        hidden = int(dim * mlp_expansion)
        self.mlps = ModuleList([nn.Sequential(nn.Linear(1, hidden), nn.SiLU(), nn.Linear(hidden, dim)) for _ in range(num_axial_dims)])


class _Rotary(Module):
    def __init__(self, dim, theta = 10000):
        super().__init__()
        freqs = 1. / (theta ** (torch.arange(0, dim, 2)[:(dim // 2)].float() / dim))
        self.freqs = nn.Parameter(freqs, requires_grad = False)


class Transformer(Module):
    """Parameter container with the reference's constructor (transfusion.py:1043-1097).  The forward pass
    lives in the engine; this class validates that the requested variant is one the kernels implement."""

    def __init__(self, dim, *, depth, dim_head = 64, heads = 8, dropout = 0., ff_expansion_factor = 4, attn_kwargs: dict = dict(),
                 ff_kwargs: dict = dict(), attn_laser = False, unet_skips = True, use_flex_attn = False, qk_rmsnorm = True,
                 use_value_residual = False):
        super().__init__()
        unsupported = []
        if dim_head not in DIM_HEADS: unsupported.append(f'dim_head {dim_head} (the attention kernels take {" or ".join(map(str, DIM_HEADS))})')
        if depth > MAX_DEPTH: unsupported.append(f'depth {depth} > {MAX_DEPTH}')
        if dim not in MODEL_DIMS: unsupported.append(f'dim {dim} (the row kernels take {", ".join(map(str, MODEL_DIMS))})')
        if dim_head == 128:                          # one head fills a 128-column QKVG tile: any count up to the 2048-wide inner limit
            if not 1 <= heads <= MAX_HEADS_D128: unsupported.append(f'heads {heads} at dim_head 128 (must be in [1, {MAX_HEADS_D128}])')
        elif heads % 2 or not MIN_HEADS <= heads <= MAX_HEADS: unsupported.append(f'heads {heads} (must be even and in [{MIN_HEADS}, {MAX_HEADS}])')
        ff_dropout = float(ff_kwargs.get('dropout', 0.))
        for name, p in (('dropout', dropout), ("ff_kwargs['dropout']", ff_dropout)):
            if not 0. <= p <= 1.:
                raise ValueError(f'{name} probability has to be between 0 and 1, but got {p}')      # nn.Dropout's check
        # attention dropout (T.py:1017) is not implemented by the attention kernels.  With use_flex_attn the reference takes the flex_attention
        # branch on CUDA (T.py:987-995), which applies no attention dropout, so there `dropout` is accepted and has no effect.
        if dropout != 0. and not use_flex_attn: unsupported.append('dropout > 0 (attention dropout) without use_flex_attn')
        extra = set(attn_kwargs) - {'softcap_value', 'laser_softclamp_value', 'gate_values'}
        if extra: unsupported.append(f'attn_kwargs {sorted(extra)}')
        extra = set(ff_kwargs) - {'dropout'}         # FeedForward(dim, mult, dropout) (T.py:837-850): dropout is its only option besides the two above
        if extra: unsupported.append(f'ff_kwargs {sorted(extra)}')
        if unsupported:
            raise NotImplementedError('not implemented by the CUDA kernels: ' + ', '.join(unsupported))
        self.dim, self.depth, self.dim_head, self.heads = dim, depth, dim_head, heads
        self.use_flex_attn = use_flex_attn           # accepted: the fused kernel IS the span-aware attention
        self.use_value_residual = bool(use_value_residual)
        self.attn_laser = bool(attn_laser)
        self.qk_rmsnorm = bool(qk_rmsnorm)           # False: q, k = RoPE(to_qk(x)) without the norms (T.py:949-951); their gammas stay built (T.py:886-888)
        self.laser_softclamp_value = float(attn_kwargs.get('laser_softclamp_value', 15.))
        self.softcap_value = float(attn_kwargs.get('softcap_value', 50.))
        self.gate_values = bool(attn_kwargs.get('gate_values', True))      # False: out = to_out(attn v), no sigmoid(gate) factor (T.py:1026-1027)
        self.ff_inner = int(dim * ff_expansion_factor * 2 / 3)
        self.ff_dropout = ff_dropout                 # nn.Dropout after GEGLU (T.py:848): fused into the GEGLU GEMM epilogue, training forwards only

        self.to_time_cond = nn.Sequential(_Fourier(dim), nn.Linear(dim + 1, dim * 4), nn.SiLU())
        layers = ModuleList([])
        for ind in range(depth):
            skip_proj = nn.Linear(dim * 2, dim, bias = False) if (ind >= depth / 2 and unet_skips) else None
            attn = _AdaptiveParams(_AttentionParams(dim, dim_head, heads, learned_value_residual_mix = ind > 0 and use_value_residual,
                                                    gate_values = self.gate_values), dim, dim * 4)
            ff = _AdaptiveParams(_FeedForwardParams(dim, self.ff_inner), dim, dim * 4)
            layers.append(ModuleList([skip_proj, attn, ff, _AttnResidualParams(dim)]))
        self.layers = layers
        self.norm = _Gamma(dim)

    def ff_dropout_p(self, train: bool, training: bool) -> float:
        """FFN dropout probability of one forward: nn.Dropout drops only in training mode (`training`, of the owning Transfusion), and only a
        forward that keeps its activations for a backward (`train`) is a training forward; sampling, eval and the velocity-consistency EMA model
        never drop.  The Self-Flow teacher's inference forward (`SelfMaskedRepTraining`) passes train = True here: in training mode it drops."""
        return self.ff_dropout if (train and training) else 0.

    def forward(self, *args, **kwargs):
        raise RuntimeError('Transformer.forward is executed by the CUDA engine through Transfusion; call the Transfusion methods')


# ------------------------------------------------------------------------------------------- autograd seam
class _TrainStep(torch.autograd.Function):
    """One node for the whole training forward: the engine keeps its own activations and writes parameter
    gradients straight into the flat `.grad` buffer, so autograd only has to hand us d(total loss)."""

    @staticmethod
    def forward(ctx, engine, rb, latents, eps, kw, anchor):
        res = engine.forward(rb, latents, eps, train = True, **kw)
        ctx.engine = engine
        engine._last_vel = res.get('vel')
        engine._last_res = res
        if 'rep' in res:            # a hidden state handed out in packed rows (`rep_layer`): its gradient comes back to backward()
            return res['total'], res['text'], res['flows'], res['rep']
        return res['total'], res['text'], res['flows']

    @staticmethod
    def backward(ctx, g_total, g_text, g_flows, *g_rep):
        kw = dict(g_rep = g_rep[0]) if g_rep else {}
        ctx.engine.backward(gscale = g_total, bucket_cb = getattr(ctx.engine, '_bucket_cb', None), **kw)
        return None, None, None, None, None, None


class Transfusion(SamplingMixin, Module):
    def __init__(
        self,
        *,
        num_text_tokens,
        transformer: dict | Transformer,
        model_output_clean = False,
        dim_latent: int | tuple | None = None,
        channel_first_latent: bool | tuple = False,
        add_pos_emb: bool | tuple = False,
        modality_encoder: Module | tuple | None = None,
        modality_decoder: Module | tuple | None = None,
        pre_post_transformer_enc_dec = None,
        modality_default_shape: tuple | None = None,
        fallback_to_default_shape_if_invalid = False,
        modality_num_dim: int | tuple | None = None,
        to_modality_shape_fn: Callable | tuple = default_to_modality_shape_fn,
        ignore_index = -1,
        flow_loss_weight = 1.,
        text_loss_weight = 1.,
        velocity_consistency_loss_weight = 0.1,
        reconstruction_loss_weight = 0.,
        modality_encoder_decoder_requires_batch_dim = True,
        odeint_kwargs: dict = dict(atol = 1e-5, rtol = 1e-5, method = 'midpoint'),
        eps = 1e-2,
        prob_uncond = 0.1,
        modality_processing: str = DEFAULT_PROCESSING_STRATEGY,
    ):
        super().__init__()
        self.modality_processing = modality_processing
        get_processing_strategy(modality_processing)
        if isinstance(transformer, dict):
            transformer = Transformer(**transformer)
        self.transformer = transformer
        dim = self.dim = transformer.dim

        self.model_output_clean = bool(model_output_clean)
        if exists(pre_post_transformer_enc_dec): raise NotImplementedError('pre_post_transformer_enc_dec (U-Net) is outside the CUDA hot path')
        assert ignore_index == -1, 'the fused loss kernel uses -1 as the ignore index'

        self.dim_latents = cast_tuple(default(dim_latent, dim))
        self.num_modalities = len(self.dim_latents)
        self.channel_first_latent = cast_tuple(channel_first_latent, self.num_modalities)
        assert len(self.channel_first_latent) == self.num_modalities
        self.to_modality_shape_fn = cast_tuple(to_modality_shape_fn, self.num_modalities)

        is_flat_shape = modality_default_shape is None or (isinstance(modality_default_shape, tuple) and all(isinstance(v, int) for v in modality_default_shape))
        if is_flat_shape:
            modality_default_shape = (modality_default_shape,) * self.num_modalities
        self.modality_default_shape = modality_default_shape
        assert len(self.modality_default_shape) == self.num_modalities
        self.fallback_to_default_shape_if_invalid = fallback_to_default_shape_if_invalid
        modality_num_dim = default(modality_num_dim, tuple(len(s) if exists(s) else None for s in self.modality_default_shape))
        self.modality_num_dim = cast_tuple(modality_num_dim, self.num_modalities)
        assert len(self.modality_num_dim) == self.num_modalities
        assert all(not exists(nd) or not exists(s) or len(s) == nd for nd, s in zip(self.modality_num_dim, self.modality_default_shape))

        self.add_pos_emb = cast_tuple(add_pos_emb, self.num_modalities)
        assert len(self.add_pos_emb) == self.num_modalities
        self.pos_emb_mlp = ModuleList([])                # T.py:1383-1403
        for add, nd in zip(self.add_pos_emb, self.modality_num_dim):
            if not add:
                self.pos_emb_mlp.append(None)
                continue
            assert exists(nd), '`modality_num_dim` must be set if you wish to automatically inject axial positional embeddings'
            assert nd <= 3, 'axial positional embeddings are implemented for up to 3 axes'
            self.pos_emb_mlp.append(_AxialPosEmb(dim, nd))

        modality_encoder = cast_tuple(modality_encoder, 1 if exists(modality_encoder) else self.num_modalities)
        modality_decoder = cast_tuple(modality_decoder, 1 if exists(modality_decoder) else self.num_modalities)
        self.modality_encoder, self.modality_decoder = ModuleList(modality_encoder), ModuleList(modality_decoder)
        assert len(self.modality_encoder) == self.num_modalities and len(self.modality_decoder) == self.num_modalities
        self.encdec_needs_batch_dim = modality_encoder_decoder_requires_batch_dim

        # special token layout (transfusion.py:1422-1449)
        self.num_text_tokens = num_text_tokens
        self.sos_id, self.eos_id, self.null_text_id = num_text_tokens, num_text_tokens + 1, num_text_tokens + 2
        first = num_text_tokens + 3
        self.som_ids = [first + m for m in range(self.num_modalities)]
        self.eom_ids = [first + self.num_modalities + m for m in range(self.num_modalities)]
        self.meta_id = first + 2 * self.num_modalities
        self._char_offset = self.meta_id + 1

        self.latent_to_model_projs = ModuleList([nn.Linear(dl, dim) if dl != dim else nn.Identity() for dl in self.dim_latents])
        self.model_to_latent_projs = ModuleList([nn.Linear(dim, dl, bias = False) for dl in self.dim_latents])
        self.rotary_emb = _Rotary(transformer.dim_head)

        vocab = num_text_tokens + 3 + 2 * self.num_modalities + 129
        self.text_embed = nn.Embedding(vocab, dim)
        self.to_text_logits = nn.Linear(dim, vocab, bias = False)
        self.register_buffer('text_only_logits_mask', torch.arange(vocab) < num_text_tokens, persistent = False)
        self.register_buffer('zero', tensor(0.), persistent = False)

        self.ignore_index = ignore_index
        self.flow_loss_weight, self.text_loss_weight = flow_loss_weight, text_loss_weight
        self.velocity_consistency_loss_weight = velocity_consistency_loss_weight
        # reconstruction loss (MP.py:177-194, T.py:3420-3431, 2836-2856): folded into the flow head's gradient pass (tfx_mse_recon_fwd_bwd)
        self.has_recon_loss, self.reconstruction_loss_weight = reconstruction_loss_weight > 0., reconstruction_loss_weight
        self.model_output_clean, self.eps = model_output_clean, eps
        self.odeint_kwargs = dict(odeint_kwargs)
        assert self.odeint_kwargs.get('method', 'midpoint') == 'midpoint', 'only the fixed-grid midpoint solver is implemented'
        self.prob_uncond = prob_uncond
        self._engine = None

    # ------------------------------------------------------------------ small API surface
    @property
    def device(self):
        return next(self.parameters()).device

    def char_tokenizer(self, text: str, device = None):
        return (tensor([ord(c) for c in text], device = device, dtype = torch.long) + self._char_offset).long()

    def decode_chars(self, t: Tensor) -> str:
        return ''.join(chr(v) for v in (t - self._char_offset).clamp(min = 0, max = 127).tolist())

    def get_modality_info(self, modality_type = None):
        t = default(modality_type, 0)
        return dict(encoder = self.modality_encoder[t], decoder = self.modality_decoder[t], latent_to_model = self.latent_to_model_projs[t],
                    model_to_latent = self.model_to_latent_projs[t], add_pos_emb = self.add_pos_emb[t], pos_emb_mlp = self.pos_emb_mlp[t], num_dim = self.modality_num_dim[t],
                    dim_latent = self.dim_latents[t], default_shape = self.modality_default_shape[t], som_id = self.som_ids[t], eom_id = self.eom_ids[t],
                    to_shape_fn = self.to_modality_shape_fn[t], channel_first_latent = self.channel_first_latent[t], modality_type = t)

    def parameters_without_encoder_decoder(self):
        return set(self.parameters()) - set(self.modality_encoder.parameters()) - set(self.modality_decoder.parameters())

    def muon_parameters(self):
        params = []
        for layer in self.transformer.layers:
            a, f = layer[1].fn, layer[2].fn
            params += [*a.to_v.parameters(), *a.to_out.parameters(), f.net[0].weight, f.net[-1].weight]
        return params

    def create_dataloader(self, *args, **kwargs):
        return create_dataloader(*args, **kwargs)

    def create_ema(self, beta = 0.99, *ema_kwargs):
        """T.py:1681-1699.  The copy's parameters live in a second flat buffer; `ema.update()` is one `tfx_ema_update` launch."""
        from .ema import EMA
        return EMA(self, beta = beta, forward_method_names = ('sample', 'sample_one', 'sample_many', 'generate_text_only', 'generate_modality_only'))

    @property
    def engine(self):
        if self._engine is None:
            from .engine import Engine
            self._engine = Engine(self)
        return self._engine

    # ------------------------------------------------------------------ engine glue
    def _latents_to_device(self, rb: RaggedBatch):
        """Per modality type: the instances' latents concatenated into one fp32 [S_t, dim_latent] device matrix.
        Host tensors that are already pinned are DMA'd straight into their slice (no host-side copy); pageable ones go
        through a persistent pinned staging buffer (one memcpy, no per-step cudaHostAlloc)."""
        dev = self.device
        out, nbytes = [], 0
        for t, lst in enumerate(rb.latents):
            if not lst:
                out.append(None); continue
            if dev.type != 'cuda':
                out.append(cat([x.detach().float() for x in lst]).contiguous()); continue
            dl = lst[0].shape[-1]
            rows = [x.shape[0] for x in lst]
            dst = torch.empty(sum(rows), dl, device = dev, dtype = torch.float32)
            stage, stage_raw, off, soff = None, None, 0, 0
            for x, n in zip(lst, rows):
                x = x.detach()
                if x.is_cuda:
                    dst[off:off + n].copy_(x)
                elif x.dtype == torch.float32 and x.is_contiguous() and x.is_pinned():
                    dst[off:off + n].copy_(x, non_blocking = True); nbytes += x.numel() * 4
                else:
                    if stage is None:
                        need = sum(r for r, y in zip(rows, lst) if not y.is_cuda) * dl
                        stage_raw = POOL.take(need * 4)
                        stage = stage_raw[:need * 4].view(torch.float32)
                    view = stage[soff:soff + n * dl].view(n, dl)
                    view.copy_(x)
                    dst[off:off + n].copy_(view, non_blocking = True)
                    soff += n * dl; nbytes += n * dl * 4
                off += n
            if stage is not None:
                POOL.give(stage_raw)
            out.append(dst)
        rb.latent_h2d_bytes = nbytes
        return out

    def _latents_into(self, rb: RaggedBatch, dst_list: list) -> int:
        """Same as `_latents_to_device` but into existing per-type device matrices (CUDA-graph static inputs); returns the H2D byte count."""
        nbytes = 0
        for t, lst in enumerate(rb.latents):
            if not lst:
                continue
            dst, dl = dst_list[t], lst[0].shape[-1]
            rows = [x.shape[0] for x in lst]
            stage, stage_raw, off, soff = None, None, 0, 0
            for x, n in zip(lst, rows):
                x = x.detach()
                if x.is_cuda:
                    dst[off:off + n].copy_(x)
                elif x.dtype == torch.float32 and x.is_contiguous() and x.is_pinned():
                    dst[off:off + n].copy_(x, non_blocking = True); nbytes += x.numel() * 4
                else:
                    if stage is None:
                        need = sum(r for r, y in zip(rows, lst) if not y.is_cuda) * dl
                        stage_raw = POOL.take(need * 4)
                        stage = stage_raw[:need * 4].view(torch.float32)
                    view = stage[soff:soff + n * dl].view(n, dl)
                    view.copy_(x)
                    dst[off:off + n].copy_(view, non_blocking = True)
                    soff += n * dl; nbytes += n * dl * 4
                off += n
            if stage is not None:
                POOL.give(stage_raw)
        return nbytes

    def _run(self, rb, latents, eps, *, train, dropout_key = None, **kw):
        eng = self.engine
        if self.transformer.ff_dropout_p(train, self.training) > 0.:
            kw.update(dropout = True, dropout_key = dropout_key)
        if train and self.has_recon_loss and rb.inst_w is not None:
            kw.setdefault('recon_weight', self.reconstruction_loss_weight)
        if train and torch.is_grad_enabled():
            anchor = self.text_embed.weight
            total, text, flows, *rep = _TrainStep.apply(eng, rb, latents, eps, kw, anchor)
            last = eng._last_res
            out = dict(total = total, text = text, flows = flows, vel = eng._last_vel, recon = last.get('recon'), recon_inst = last.get('recon_inst'), preds = last.get('preds'))
            if rep:
                out['rep'] = rep[0]
            return out
        return eng.forward(rb, latents, eps, train = train, **kw)

    def _recon_breakdown(self, rb, res):
        """`LossBreakdown.recon` (T.py:3288-3311, 3441): per modality type (all of them, absent ones included) the list of per-instance reconstruction
        MSEs in scan order; device scalars, no host synchronisation"""
        out = [[] for _ in range(self.num_modalities)]
        inst = res.get('recon_inst')
        if inst is None or not rb.instances:
            return out
        ni = len(rb.instances)
        denom = np.fromiter((i.length * self.dim_latents[i.modality_type] for i in rb.instances), dtype = np.float64, count = ni)
        vals = (inst[:ni] / torch.from_numpy(denom).to(inst.device, non_blocking = True)).float()
        for k, i in enumerate(rb.instances):
            out[i.modality_type].append(vals[k])
        return out

    def forward_packed(self, rb: RaggedBatch, latents: list, noise: list | None = None, return_breakdown = False, dropout_key = None):
        """Training step from an already packed (and possibly already uploaded) ragged batch: the part of `forward`
        after pack/route.  Used by bench.py to time the device-resident path.  `dropout_key`: see `forward`."""
        eps = noise if exists(noise) else [torch.randn_like(l) if exists(l) else None for l in latents]
        res = self._run(rb, latents, eps, train = True, text_loss_weight = self.text_loss_weight, flow_loss_weight = self.flow_loss_weight, dropout_key = dropout_key)
        self._last_batch = rb
        if return_breakdown:
            recon = self._recon_breakdown(rb, res) if self.has_recon_loss else None
            return res['total'], LossBreakdown(res['total'], res['text'], list(res['flows']), None, recon)
        return res['total']

    # ------------------------------------------------------------------ text only (transfusion.py:2585-2707)
    def forward_text(self, text: Tensor, return_loss = True, return_embed = False, cache = None, return_hiddens = False, return_kv_cache = False, dropout_key = None):
        """`cache` / `return_kv_cache` follow the reference's tuple convention `(kv, tokens_seen)` (T.py:2613, 2636); `kv` is a `TextKVCache`
        handle onto in-place cache slabs instead of a `(layers, 2, b, h, n, d)` tensor that is concatenated per call (T.py:969-977)."""
        raw_cache, tokens_seen = default(cache, (None, 0))
        if return_loss:
            assert not exists(raw_cache) and not return_kv_cache, 'the kv cache is a decode-time structure'
            rb = pack_text_only(text, return_loss = True)
            res = self._run(rb, None, None, train = True, vlimit = self.num_text_tokens, dropout_key = dropout_key)
            if return_hiddens:
                return res['total'], self._hiddens_padded(rb)
            return res['total']
        use_cache = exists(raw_cache) or return_kv_cache
        B, n = text.shape
        V = self.to_text_logits.weight.shape[0]
        if not use_cache:
            rb = pack_text_only(text, return_loss = False)
            res = self.engine.forward(rb, None, None, train = False, want_logits = True)
            kv = None
        else:
            eng = self.engine
            kv = raw_cache if exists(raw_cache) else TextKVCache(eng, B, max(256, 2 * n))
            assert kv.B == B, 'cache was built for a different batch size'
            kv.reserve(n)
            rb = pack_incremental([[row] for row in text.detach().cpu().long()], None, self, slab = np.arange(B), base_len = np.full(B, kv.length), rope_base = np.full(B, tokens_seen),
                                  cap = kv.cache.cap)
            res = eng.forward(rb, None, None, train = False, want_logits = True, cache = kv.cache)
            kv.length += n
        # fresh tensors: the engine's result buffers are workspaces that the next call overwrites (callers keep logits across decode steps)
        out = res['embed'].reshape(B, n, -1).clone() if return_embed else res['logits'][:, :V].reshape(B, n, -1).clone()
        ret = (out,)
        if return_kv_cache:
            ret = (*ret, (kv, tokens_seen + n))
        if return_hiddens:
            ret = (*ret, self._hiddens_padded(rb))
        return ret[0] if len(ret) == 1 else ret

    def _hiddens_padded(self, rb):
        """hidden states of the last forward in the reference's layout (T.py:1199, 1244, 1252-1254): [tokens, layer 1 .. depth, final norm], each [b, n, d]"""
        st = self.engine.state
        n_max = int(rb.seq_lens.max()) if rb.B else 0
        def unpack(t):
            out = t.new_zeros((rb.B, n_max, t.shape[-1]))
            for b in range(rb.B):
                out[b, :rb.seq_lens[b]] = t[rb.cu[b]:rb.cu[b + 1]]
            return out
        return [unpack(h.float().clone()) for h in (*st['hid'], st['out'])]      # (the engine keeps the layer hiddens in bf16)

    @torch.no_grad()
    def generate_text_only(self, prompt: Tensor, seq_len: int, temperature = 1.0, min_p = 0.1, cache_kv = True, seed = None, use_cuda_graph = True) -> Tensor:
        """T.py:2669-2707.  Always decodes against the kv cache (`cache_kv = False` only re-computes the same values in the reference):
        one prefill of the prompt, then one captured CUDA graph per token - embed, block stack with in-place cache append and the decode
        attention kernel, logits, on-device argmax / min-p + Gumbel sampling - with no host synchronisation until the tokens are read back."""
        was = self.training
        self.eval()
        eng = self.engine
        frozen_before = getattr(eng, 'frozen', False)
        try:
            B, n = prompt.shape
            steps = max(0, seq_len - n)
            if steps == 0:
                return prompt[..., n:].clone()
            cache = eng.new_cache(B, seq_len + 1)
            eng.pack_weights()
            eng.frozen = True
            rb = pack_incremental([[row] for row in prompt.detach().cpu().long()], None, self, slab = np.arange(B), base_len = np.zeros(B), rope_base = np.zeros(B), cap = cache.cap)
            res = eng.forward(rb, None, None, train = False, want_logits = True, cache = cache)
            if seed is None:
                seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())
            # greedy: argmax over ALL logits (T.py:2692-2693); otherwise min-p over all logits, then restricted to text ids (T.py:2695-2698)
            dec = eng.text_decoder(cache, B, slab0 = 0, hist_cap = steps + 1, eos_id = -1, som_ids = [], max_length = 2 ** 30, temperature = temperature, min_p = min_p,
                                   vlimit = 0 if temperature == 0. else self.num_text_tokens, seed = seed, use_graph = use_cuda_graph)
            dec.set_state(np.full(B, n), np.full(B, n), np.zeros(B), np.zeros(B), np.zeros(B))
            dec.sample_first(res['logits'], rb.cu[1:] - 1)
            for _ in range(steps - 1):
                dec.step()
            _, hist = dec.get_state()
            return torch.stack([torch.from_numpy(h) for h in hist]).to(prompt.device)
        finally:
            eng.frozen = frozen_before
            self.train(was)

    # ------------------------------------------------------------------ modality only (transfusion.py:2709-2866)
    def forward_modality(self, modalities: Tensor, times = None, modality_type = None, encode_modality = True, velocity_consistency_ema_model = None,
                         velocity_consistency_delta_time = 1e-5, return_loss = True, return_loss_breakdown = False, noise = None):
        """T.py:2709-2866.  Training returns flow + w_v velocity + w_r recon, and with `return_loss_breakdown` (flow, velocity, recon).
        Velocity consistency: the student runs at t (1 - delta), the EMA model predicts at t + delta on the clean encoded tokens, and the term
        mse(flow, ema prediction) adds its value only.  Reconstruction: noise + pred (1 - t) against the input before the encoder; through a
        `modality_decoder` (user module, run under no_grad) it adds its value only, otherwise it is fused into the flow head's gradient pass."""
        if self.num_modalities > 1:
            assert exists(modality_type), '`modality_type` must be explicitly passed in on forward when training on greater than 1 modality'
        mt = default(modality_type, 0)
        enc, dec = self.modality_encoder[mt], self.modality_decoder[mt]
        orig = modalities
        x = modalities
        if encode_modality and exists(enc):
            with torch.no_grad():
                enc.eval(); x = enc(x.to(self.device)).detach()
        B = x.shape[0]
        if times is None:
            times = torch.rand((B,))
        ema = velocity_consistency_ema_model if return_loss else None
        vel_target = None
        if exists(ema):
            if hasattr(ema, 'ema_model'):
                assert isinstance(ema.ema_model, Transfusion)
                if hasattr(ema, '_engines'):
                    ema._engines()
                ema = ema.ema_model
            orig_times = times.clone()
            times = times * (1. - velocity_consistency_delta_time)        # T.py:2753-2755
            with torch.no_grad():
                ema.eval()
                vel_target = ema.forward_modality(x, modality_type = mt, times = orig_times + velocity_consistency_delta_time, encode_modality = False, return_loss = False)
            vel_target = self._modality_rows(vel_target, mt)
        samples = [[(mt, x[b])] for b in range(B)]
        rb = pack_batch(samples, times.reshape(B, 1), self, return_loss = False, return_embed = True)
        rb.kv_limit[:] = np.repeat(rb.cu[1:] - 1, rb.seq_lens).astype(np.int32)      # no mask at all (transfusion.py:2800-2804)
        rb.rope_pos[:] = 0                                                            # no rotary embedding in this path
        from .modality_processing import build_tiles
        build_tiles(rb, np.repeat(rb.cu[:-1], rb.seq_lens).astype(np.int32))
        lat = self._latents_to_device(rb)
        if return_loss:
            eps = [None] * self.num_modalities
            eps[mt] = noise.reshape(-1, self.dim_latents[mt]).float().to(self.device) if exists(noise) else torch.randn_like(lat[mt])
            rb.has_labels = True
            kw = {}
            if exists(vel_target):
                kw.update(vel_targets = [vel_target if t == mt else None for t in range(self.num_modalities)], vel_weight = self.velocity_consistency_loss_weight, vel_grad = False)
            fused_recon = self.has_recon_loss and not exists(dec)
            if self.has_recon_loss:
                assert encode_modality, 'the reconstruction loss compares with the modality before the encoder (T.py:2841)'
                if fused_recon and exists(enc):      # residual (1 - t) pred - (orig - noise)
                    o = self._modality_rows(orig.to(self.device), mt)
                    if o.shape != eps[mt].shape:
                        raise ValueError(f'reconstruction loss without a decoder: the modality before the encoder {tuple(orig.shape)} must have the shape of the encoded one {tuple(x.shape)}')
                    g = [None] * self.num_modalities
                    g[mt] = o - eps[mt]
                    kw['recon_g'] = g
                kw['recon_weight'] = self.reconstruction_loss_weight if fused_recon else 0.
            res = self._run(rb, lat, eps, train = True, modality_only = True, flow_loss_weight = 1., **kw)
            flow_loss = res['flows'][mt]
            total = res['total']
            velocity_loss = res['vel'][mt] if exists(vel_target) else self.zero
            recon_loss = res['recon'][mt] if fused_recon else self.zero
            if self.has_recon_loss and exists(dec):
                # decoder(noise + pred (1 - t)) under no_grad (T.py:2843-2848): adds to the value, carries no gradient
                with torch.no_grad():
                    s0, s1 = rb.type_rows[mt]
                    tr = rb.dev['row_time'][s0:s1, None] if rb.dev else torch.as_tensor(rb.row_time[s0:s1])[:, None]
                    rec = eps[mt] + res['preds'][mt] * (1. - tr)
                    dec.eval()
                    out = dec(self._rows_to_modality(rec, x, mt))
                    recon_loss = torch.nn.functional.mse_loss(out.float(), orig.to(out.device).float())
                total = total + recon_loss * self.reconstruction_loss_weight
            if return_loss_breakdown:
                return total, (flow_loss, velocity_loss, recon_loss)
            return total
        res = self.engine.forward(rb, lat, None, train = False, want_logits = True)
        return self._rows_to_modality(res['preds'][mt], x, mt)

    def _rows_to_modality(self, rows, like, mt):
        """[B * n, dim_latent] compact rows -> the layout of `like` ([B, *axial, d] or channel first [B, d, *axial])"""
        B, cf = like.shape[0], self.channel_first_latent[mt]
        inst_shape = like.shape[2:] if cf else like.shape[1:-1]
        out = rows.reshape(B, *inst_shape, self.dim_latents[mt])
        return out.movedim(-1, 1) if cf else out

    def _modality_rows(self, t, mt):
        """inverse of `_rows_to_modality`: a fresh fp32 [B * n, dim_latent] matrix on the model's device"""
        if self.channel_first_latent[mt]:
            t = t.movedim(1, -1)
        return t.reshape(-1, self.dim_latents[mt]).float().to(self.device).clone()

    # ------------------------------------------------------------------ host side of forward(): CFG dropout, encoders, times, pack / route
    def pack(self, modalities, times = None, num_modalities_to_times_fn = None, prob_uncond = None, return_loss = True, return_embed = False, is_decoding = False,
             pad_rows = False):
        """Everything `forward` does on the host before the first kernel (transfusion.py:3011-3082 + modality_processing): returns the ragged
        batch descriptor and the times that were used.  Exposed so that a training loop can pack step i+1 while step i runs on the device
        (`DataParallelTrainer` does, and replays a captured CUDA graph when the descriptor has the same shape signature).
        `pad_rows`: feed every sample at the longest sample's length (`modality_processing.pack_batch`), as `SelfMaskedRepTraining` does."""
        batch = len(modalities)
        samples = [list(s) if isinstance(s, list) else s for s in modalities]
        if return_loss:
            se = self.__dict__.get('_sos_eos')
            if se is None:
                se = self.__dict__['_sos_eos'] = (tensor([self.sos_id]), tensor([self.eos_id]))      # immutable, shared by every sample
            samples = [[se[0], *s, se[1]] for s in samples]
        # classifier free guidance dropout (transfusion.py:3027-3043): all int tensors of a dropped sample -> null id
        prob_uncond = default(prob_uncond, self.prob_uncond)
        if self.training and prob_uncond > 0:
            drop = (torch.rand(batch) < prob_uncond).tolist()
            samples = [[torch.full_like(p, self.null_text_id) if is_int_tensor(p) else p for p in s] if d else s for s, d in zip(samples, drop)]
        # modality encoders (user modules, outside the hot path)
        n_mods = []
        encoders = list(self.modality_encoder)          # plain list: ModuleList indexing costs ~2.5 us per part
        for s in samples:
            cnt = 0
            for j, part in enumerate(s):
                if not isinstance(part, tuple) and part.is_floating_point():
                    part = s[j] = (0, part)
                if isinstance(part, tuple):
                    cnt += 1
                    enc = encoders[part[0]]
                    if exists(enc) and not is_decoding:
                        with torch.no_grad():
                            enc.eval()
                            v = part[1].to(self.device)
                            v = enc(v[None])[0] if self.encdec_needs_batch_dim else enc(v)
                            s[j] = (part[0], v.detach())
            n_mods.append(cnt)
        if times is None and max(n_mods, default = 0) > 0:
            fn = default(num_modalities_to_times_fn, default_modality_length_to_time_fn)
            times = fn(tensor(n_mods))
        process = get_processing_strategy(self.modality_processing)
        rb = process(samples, times, self, need_axial_pos_emb = any(self.add_pos_emb), return_loss = return_loss, return_embed = return_embed, pad_rows = pad_rows)
        return rb, times

    # ------------------------------------------------------------------ main forward (transfusion.py:2925-3450)
    def forward(
        self,
        modalities,
        times = None,
        num_modalities_to_times_fn: Callable | None = None,
        modality_type = None,
        cache = None,
        decode_length = None,
        decoding_text_or_modality = None,
        velocity_consistency_ema_model = None,
        velocity_consistency_delta_time = 1e-3,
        return_only_pred_flows = False,
        return_loss = True,
        return_breakdown = False,
        return_embed = False,
        return_hiddens = False,
        return_kv_cache = False,
        return_times = False,
        prob_uncond = None,
        noise = None,            # extension: list (per type) of [S_t, dim_latent] noise for deterministic parity runs
        velocity_consistency_noise = None,      # extension: same, for the EMA teacher's own draw (T.py:3388-3392 draws it with randn_like)
        dropout_key = None,      # extension: (k0, k1) u32 key of the dropout masks (csrc/dropout.cuh) for deterministic runs; None draws one per forward
    ):
        is_decoding = exists(decoding_text_or_modality)
        if is_int_tensor(modalities):
            return self.forward_text(modalities, return_loss = return_loss and not return_embed, return_embed = return_embed, cache = cache,
                                     return_kv_cache = return_kv_cache, return_hiddens = return_hiddens, dropout_key = dropout_key)
        if is_tensor(modalities) and modalities.is_floating_point():
            assert return_loss
            return self.forward_modality(modalities, modality_type = modality_type)
        return_loss = return_loss and not (return_embed or is_decoding)
        assert not exists(cache) and not return_kv_cache, 'interleaved decoding against the kv cache is driven by sample() / sample_many() (engine.KVCache); `forward_text` takes / returns a cache'

        # ---- velocity consistency (T.py:2965-2971, 3003-3008, 3084-3088, 3383-3418): the EMA model predicts the flow at t + delta from its own
        # noise draw; the student is trained at t (1 - delta) and pulled towards that prediction
        ema = velocity_consistency_ema_model
        if exists(ema) and hasattr(ema, 'ema_model'):
            assert isinstance(ema.ema_model, Transfusion)
            if hasattr(ema, '_engines'):
                ema._engines()
            ema = ema.ema_model
        need_velocity = not is_decoding and exists(ema)
        vel_targets = None
        if need_velocity:
            assert return_loss, 'velocity consistency is a training loss'
            velocity_modalities = [list(m) if isinstance(m, list) else m for m in modalities]
            if times is None:
                n_mods = tensor([sum(1 for part in m if isinstance(part, tuple) or (is_tensor(part) and part.is_floating_point())) for m in modalities])
                times = default(num_modalities_to_times_fn, default_modality_length_to_time_fn)(n_mods)
            orig_times = times.clone()
            times = times * (1. - velocity_consistency_delta_time)
            with torch.no_grad():
                ema.eval()
                vel_targets = ema(velocity_modalities, times = orig_times + velocity_consistency_delta_time, return_only_pred_flows = '_compact', noise = velocity_consistency_noise)

        rb, times = self.pack(modalities, times = times, num_modalities_to_times_fn = num_modalities_to_times_fn, prob_uncond = prob_uncond,
                              return_loss = return_loss, return_embed = return_embed, is_decoding = is_decoding)
        lat = self._latents_to_device(rb)
        if return_loss:
            if exists(noise):
                eps = [n.reshape(-1, self.dim_latents[t]).float().to(self.device) if exists(n) else None for t, n in enumerate(noise)]
            else:
                eps = [torch.randn_like(l) if exists(l) else None for l in lat]
            if return_only_pred_flows:
                # early return used by the velocity-consistency teacher (T.py:3313-3316): noise inject + block stack + flow head, no loss
                res = self.engine.forward(rb, lat, eps, train = False, want_logits = False, want_preds = True)
                self._last_batch = rb
                compact = [p.clone() if exists(p) else None for p in res.get('preds', [None] * self.num_modalities)]
                if return_only_pred_flows == '_compact':
                    return compact
                out = [[] for _ in range(self.num_modalities)]
                for inst in rb.instances:                 # per type, per instance, in scan order (the reference's `pred_flows` layout)
                    t = inst.modality_type
                    out[t].append(compact[t][inst.row0: inst.row0 + inst.length])
                return out
            kw = dict(vel_targets = vel_targets, vel_weight = self.velocity_consistency_loss_weight) if need_velocity else {}
            res = self._run(rb, lat, eps, train = True, text_loss_weight = self.text_loss_weight, flow_loss_weight = self.flow_loss_weight, dropout_key = dropout_key, **kw)
            total = res['total']
            self._last_batch = rb
            if not return_breakdown and not return_hiddens and not return_times:
                return total
            ret = (total,)
            if return_breakdown:
                flows = [res['flows'][t] for t in range(self.num_modalities) if rb.type_rows[t][1] > rb.type_rows[t][0]]
                vel = [res['vel'][t] for t in range(self.num_modalities) if rb.type_rows[t][1] > rb.type_rows[t][0]] if need_velocity else None
                ret = (*ret, LossBreakdown(total, res['text'], flows, vel, self._recon_breakdown(rb, res)))
            if return_hiddens:
                ret = (*ret, self._hiddens_padded(rb))
            if return_times:
                ret = (*ret, times)
            return ret
        res = self.engine.forward(rb, lat, None, train = False, want_logits = not return_embed)
        self._last_batch = rb
        n_max = int(rb.seq_lens.max()) if rb.B else 0
        def unpack(t, width):
            out = t.new_zeros((rb.B, n_max, width))
            for b in range(rb.B):
                out[b, :rb.seq_lens[b]] = t[rb.cu[b]:rb.cu[b + 1], :width]
            return out
        out = (unpack(res['embed'], self.dim), rb) if return_embed else unpack(res['logits'], self.to_text_logits.weight.shape[0])
        ret = (out,)                                   # aux packing order of the reference (T.py:3256-3271); the descriptor stands in for `get_pred_flows`
        if return_hiddens:
            ret = (*ret, self._hiddens_padded(rb))
        if return_times:
            ret = (*ret, times)
        return ret[0] if len(ret) == 1 else ret


# ------------------------------------------------------------------------------------------- Self-Flow (T.py:3452-3569)
def default_rep_loss_fn(pred, target):
    """1 - mean cosine similarity over the last dim (T.py:3458-3460); `SelfMaskedRepTraining` runs it as the fused tfx_rep_cos_fwd_bwd kernel"""
    return 1. - torch.nn.functional.cosine_similarity(pred, target, dim = -1).mean()


class _RepLoss(torch.autograd.Function):
    """The predictor head and the representation loss as one node: its backward runs before the student's (`rep` is a `_TrainStep` output), so
    the engine's backward receives the gradient of the student's hidden state."""

    @staticmethod
    def forward(ctx, head, rep, teacher_rep, g, anchor):
        ctx.head = head
        return head.forward(rep, teacher_rep, g)

    @staticmethod
    def backward(ctx, g_loss):
        return None, ctx.head.backward(g_loss), None, None, None


class SelfMaskedRepTraining(Module):
    """Self-Flow training (T.py:3452-3569): the student's hidden state at `student_layer`, through a predictor head (RMSNorm + GEGLU FeedForward),
    is pulled towards the EMA teacher's hidden state at `teacher_layer` by 1 - mean cosine similarity, averaged over the padded [b, n] layout as
    in the reference (pad rows: `modality_processing.pack_batch`).  Asymmetric dropout sets the student's and the teacher's FFN dropout (the
    `nn.Dropout` modules `set_dropout_` reaches); attention dropout exists only as the no-op of `use_flex_attn`.  The teacher is an inference
    forward of the EMA engine that keeps its hidden states; the head runs on the block stack's kernels (`engine.RepHead`)."""

    def __init__(self, net: Transfusion, ema_beta = 0.999, rep_loss_weight = 0.1, student_layer = -3, teacher_layer = -1, loss_fn = default_rep_loss_fn,
                 use_asymmetric_dropout = True, student_dropout_rate = 0.1, teacher_dropout_rate = 0.):
        super().__init__()
        assert not use_asymmetric_dropout or student_dropout_rate > teacher_dropout_rate, 'student must have greater dropout rate than teacher to ensure teacher has a better view'
        if loss_fn is not default_rep_loss_fn:
            raise NotImplementedError('loss_fn: only the default (1 - mean cosine similarity) is implemented, as the fused kernel tfx_rep_cos_fwd_bwd')
        if use_asymmetric_dropout and (student_dropout_rate or teacher_dropout_rate) and not net.transformer.use_flex_attn:
            raise NotImplementedError('asymmetric dropout sets attention dropout, which the attention kernels do not implement; '
                                      'only use_flex_attn = True (no attention dropout in the reference either) is supported')
        n_hid = net.transformer.depth + 2
        for name, layer in (('student_layer', student_layer), ('teacher_layer', teacher_layer)):
            if not -n_hid <= layer < n_hid:
                raise IndexError(f'{name} = {layer}: the hidden states are [tokens, layer 1 .. {n_hid - 2}, final norm] ({n_hid} entries)')
        self.student = net
        self.teacher = net.create_ema(beta = ema_beta)
        self.rep_loss_weight = rep_loss_weight
        self.has_ssl_loss = rep_loss_weight > 0
        self.use_asymmetric_dropout = use_asymmetric_dropout
        self.student_dropout_rate, self.teacher_dropout_rate = student_dropout_rate, teacher_dropout_rate
        self.student_layer, self.teacher_layer = student_layer, teacher_layer
        self.loss_fn = loss_fn
        dim = net.dim
        self.student_predict_head = nn.Sequential(_Gamma(dim), _FeedForwardParams(dim, int(dim * 4 * 2 / 3)))      # RMSNorm(dim), FeedForward(dim)
        self.register_buffer('zero', tensor(0.))
        self.teacher.ema_model.train(self.training)        # a registered sub-module: the teacher follows the wrapper's .train() / .eval()
        self._head = None

    def parameters(self):
        return chain(self.student.parameters(), self.student_predict_head.parameters())

    def update_teacher(self):
        self.teacher.update()

    def forward(self, modalities, times = None, num_modalities_to_times_fn = None, prob_uncond = None, noise = None, teacher_noise = None, dropout_key = None):
        """Returns total, (student loss, Self-Flow loss).  `modalities`: interleaved samples (the only input the reference wrapper takes: its tensor
        forwards return no times).  `noise` / `teacher_noise`: per type [S_t, dim_latent] flow noise of the student's / the teacher's forward, as
        `Transfusion.forward(noise = ...)`; `dropout_key`: the student's FFN dropout masks (the teacher draws its own)."""
        if is_tensor(modalities):
            raise TypeError('SelfMaskedRepTraining takes interleaved sample lists (the reference wrapper needs the times of that forward)')
        student, ema = self.student, self.teacher
        if self.use_asymmetric_dropout:                    # set_dropout_ (T.py:156-159), persisting on the student
            student.transformer.ff_dropout = float(self.student_dropout_rate)
        if not self.has_ssl_loss:
            loss = student(modalities, times = times, num_modalities_to_times_fn = num_modalities_to_times_fn, prob_uncond = prob_uncond, noise = noise,
                           dropout_key = dropout_key)
            return loss, (loss, self.zero)
        n_hid = student.transformer.depth + 2

        def run(model, times_, noise_):
            rb, used_times = model.pack(modalities, times = times_, num_modalities_to_times_fn = num_modalities_to_times_fn, prob_uncond = prob_uncond,
                                        return_loss = True, pad_rows = True)
            lat = model._latents_to_device(rb)
            if exists(noise_):
                eps = [n.reshape(-1, model.dim_latents[t]).float().to(model.device) if exists(n) else None for t, n in enumerate(noise_)]
            else:
                eps = [torch.randn_like(l) if exists(l) else None for l in lat]
            return rb, used_times, lat, eps

        rb, times_used, lat, eps = run(student, times, noise)
        res = student._run(rb, lat, eps, train = True, text_loss_weight = student.text_loss_weight, flow_loss_weight = student.flow_loss_weight,
                           dropout_key = dropout_key, rep_layer = self.student_layer % n_hid)
        student._last_batch = rb
        student_loss = res['total']

        teacher = ema.ema_model
        ema._engines()
        if self.use_asymmetric_dropout:
            teacher.transformer.ff_dropout = float(self.teacher_dropout_rate)
        with torch.no_grad():
            rb_t, _, lat_t, eps_t = run(teacher, times_used, teacher_noise)          # the student's times (T.py:3539)
            assert rb_t.M == rb.M
            dropout = teacher.transformer.ff_dropout_p(True, teacher.training) > 0.
            tres = teacher.engine.forward(rb_t, lat_t, eps_t, train = False, want_logits = False, want_preds = False, rep_layer = self.teacher_layer % n_hid,
                                          dropout = dropout)
        if self._head is None or self._head.eng is not student.engine:
            from .engine import RepHead
            self._head = RepHead(student.engine, self.student_predict_head)
        g = torch.full((1,), float(self.rep_loss_weight), device = student.engine.device)        # d total / d loss of a plain total.backward()
        ssl = _RepLoss.apply(self._head, res['rep'], tres['rep'], g, self.student_predict_head[0].gamma)
        return student_loss + ssl * self.rep_loss_weight, (student_loss, ssl)
