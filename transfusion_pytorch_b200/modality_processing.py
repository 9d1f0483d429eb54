"""Pack / route of interleaved text + modality samples (host side, Python + NumPy).

Role of the reference's `modality_processing.py` (strategies naive/grouped/flat/hybrid/auto,
modality_processing.py:379-1256) - BASELINE.json keeps this step in Python.  The design differs in
what it emits: instead of padded `[b, n]` text / `[b, n, d]` modality buffers, a dense `Bool[b,n,n]` mask
and per-instance closures, it produces ONE ragged descriptor for the kernels:

  * sequences packed back to back (`cu_seqlens`), no padding positions;
  * per token int32 metadata: text id, next-token label, `kv_limit` (last visible key - the whole hybrid
    causal / in-span-bidirectional mask of transfusion.py:452-470 as one int), RoPE position
    (transfusion.py:398-415), condition row (which distinct time value), compact modality row (`slot`);
  * 64-row tile tables for the attention kernels;
  * modality latents of one type concatenated into one `[S_t, dim_latent]` matrix (the idea of the `flat`
    strategy, modality_processing.py:617-689) so noise-inject + `latent_to_model` are one launch per type.

All strategies of the reference produce identical token layouts (modality_processing.py:1258-1305), so the
registry below maps every strategy name onto this single ragged implementation.
`modality_positions` (type, offset, length) is kept bit-exact with the reference
(tests/golden + reference tests/test_modality_processing.py:482-493).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable

import numpy as np
import torch
from torch import Tensor, is_tensor

ModalitySample = list   # list[Int[''] | Int['_'] | Float['...'] | tuple[int, Float['...']]]

ATT_TILE = 64


def is_int_tensor(t) -> bool:
    return is_tensor(t) and t.dtype in (torch.int, torch.long)


@dataclass
class ModalityInstance:
    batch_index: int
    modality_type: int
    offset: int                 # offset inside the sample (reference convention, before the shift)
    length: int
    axial_shape: tuple
    row0: int                   # first row in the per-type compact latent matrix
    cond_row: int               # row of the condition table (distinct time)
    token0: int = -1            # packed token index of the first latent token (-1 if dropped)


@dataclass
class RaggedBatch:
    B: int
    M: int                                  # packed tokens fed to the transformer
    seq_lens: np.ndarray                    # [B] tokens per sample as fed (after the training shift)
    cu: np.ndarray                          # [B+1]
    full_lens: np.ndarray                   # [B] tokens per sample before the shift (reference `total_lens`)
    text_id: np.ndarray
    label: np.ndarray
    kv_limit: np.ndarray
    rope_pos: np.ndarray
    cond_row: np.ndarray
    slot: np.ndarray
    n_cond: int
    cond_times: np.ndarray                  # [n_cond] float32
    n_types: int
    type_rows: list                         # per type (s0, s1) row range in the global compact matrix
    row_token: np.ndarray                   # [S] packed token index of each compact row (-1: not fed)
    row_time: np.ndarray                    # [S] float32
    latents: list                           # per type: list of [len, dim_latent] tensors in scan order
    instances: list                         # list[ModalityInstance] in scan order
    modality_positions: list                # list[list[(type, offset, length)]]
    total_tokens: int
    n_type_tokens: list
    tile_q0: np.ndarray = None
    tile_qend: np.ndarray = None
    tile_kv0: np.ndarray = None
    tile_kvend: np.ndarray = None
    kt_kv0: np.ndarray = None
    kt_kvend: np.ndarray = None
    kt_q0: np.ndarray = None
    kt_qend: np.ndarray = None
    # same tables with 128-row tiles (bounded-logit wgmma attention: two 64-row warpgroups)
    t2_q0: np.ndarray = None
    t2_qend: np.ndarray = None
    t2_kv0: np.ndarray = None
    t2_kvend: np.ndarray = None
    k2_kv0: np.ndarray = None
    k2_kvend: np.ndarray = None
    k2_q0: np.ndarray = None
    k2_qend: np.ndarray = None
    k2_order: np.ndarray = None             # 128-key tiles sorted by the number of query tiles that see them (persistent attention backward)
    pos_c0: np.ndarray = None               # axial positional embedding (add_pos_emb): coordinate of every compact row along axis 0 / 1 / 2 of its instance (-1: none)
    pos_c1: np.ndarray = None
    pos_c2: np.ndarray = None
    pos_max: tuple = None                   # per type: per-axis table lengths (batch maximum, rounded up to a multiple of 8) or None
    row_inst: np.ndarray = None             # reconstruction loss only: [S] index into `instances` of every compact row
    inst_w: np.ndarray = None               # reconstruction loss only: [S] float32, entry i = 1 / (instances of i's type x rows of i); zero past the instances
    kv_row: np.ndarray = None               # kv-cache forward only: cache row each (new) token's key / value is appended at
    single_row_tiles: bool = False          # every attention tile holds exactly one query row (text decode): use the decode kernel
    max_rope_pos: int = 0
    has_labels: bool = False
    n_valid: int = 0
    dev: dict = field(default_factory = dict)   # device copies (filled by the engine)

    @property
    def S(self) -> int:
        return int(self.row_token.shape[0])


def _meta_ids(model, axial: tuple, modality_type: int):
    """[meta] <shape chars> [som] ... [eom] ids (transfusion.py:1426-1447, modality_processing.py:265-287); returns (prefix ids, [eom] as a 1-element array)."""
    cache = model.__dict__.setdefault('_meta_id_cache', {})
    key = (axial, modality_type)
    hit = cache.get(key)
    if hit is None:
        chars = [ord(c) + model.meta_id + 1 for c in ','.join(map(str, axial))]
        hit = cache[key] = (np.asarray([model.meta_id] + chars + [model.som_ids[modality_type]], dtype = np.int64), np.asarray([model.eom_ids[modality_type]], dtype = np.int64))
    return hit


_NEG = np.full(4096, -1, dtype = np.int64)


def _neg_ids(n: int):
    """n ids of -1 (modality positions carry no text id): a view of a shared array, no allocation per instance"""
    global _NEG
    if n > _NEG.shape[0]:
        _NEG = np.full(max(n, 2 * _NEG.shape[0]), -1, dtype = np.int64)
    return _NEG[:n]


ATT_GROUP_TOKENS = 8192          # L2-locality group of the attention work list (8 k tokens x (q, k, v, dO) bf16 x 512 = 32 MB of the 50 MB H100 L2)


def build_tiles(rb: RaggedBatch, qfirst: np.ndarray) -> None:
    """Attention tile tables; tiles never straddle a sequence.  Forward: per query tile the key range [kv0, kv_end) it can see;
    backward: per key tile the query range [q0, q_end) that can see it.  Built for 64-row tiles (general mma.sync kernels) and
    128-row tiles (bounded-logit kernels).  Vectorised: no per-tile Python work."""
    cu, lens = rb.cu.astype(np.int64), rb.seq_lens.astype(np.int64)
    kv_limit = np.asarray(rb.kv_limit)
    qfirst = np.asarray(qfirst)
    for T, pre_q, pre_k in ((ATT_TILE, 'tile', 'kt'), (2 * ATT_TILE, 't2', 'k2')):
        ntiles = (lens + T - 1) // T                                     # tiles per sequence
        total = int(ntiles.sum())
        if total == 0:
            z = np.zeros(0, dtype = np.int32)
            for name in (f'{pre_q}_q0', f'{pre_q}_qend', f'{pre_q}_kv0', f'{pre_q}_kvend', f'{pre_k}_kv0', f'{pre_k}_kvend', f'{pre_k}_q0', f'{pre_k}_qend'):
                setattr(rb, name, z)
            rb.k2_order = z
            continue
        seq = np.repeat(np.arange(rb.B), ntiles)                         # sequence of every tile
        first = np.cumsum(ntiles) - ntiles                               # index of the first tile of each sequence
        tin = np.arange(total) - first[seq]                              # tile index inside its sequence
        s = cu[:-1][seq]
        q0 = s + tin * T
        qe = np.minimum(q0 + T, s + lens[seq])
        kve = np.maximum.reduceat(kv_limit, q0) + 1                      # tiles are contiguous and cover every token
        kq0 = s + ((qfirst[q0] - s) // T) * T
        as32 = lambda a: np.ascontiguousarray(a, dtype = np.int32)
        for name, arr in ((f'{pre_q}_q0', q0), (f'{pre_q}_qend', qe), (f'{pre_q}_kv0', s), (f'{pre_q}_kvend', kve),
                          (f'{pre_k}_kv0', q0), (f'{pre_k}_kvend', qe), (f'{pre_k}_q0', kq0), (f'{pre_k}_qend', s + lens[seq])):
            setattr(rb, name, as32(arr))
        if pre_k == 'k2':
            # launch order of the bounded-logit backward (key tiles): heaviest first INSIDE groups of ~8 k consecutive tokens, group after group, so
            # that the Q / dO tiles of a sequence are read by CTAs that run at about the same time and stay in L2.  Small batches (fewer than ~12
            # groups) keep the global cost sort: most of their working set fits the L2 anyway.
            group = s // ATT_GROUP_TOKENS if rb.M >= 12 * ATT_GROUP_TOKENS else np.zeros_like(s)
            rb.k2_order = as32(np.lexsort((-(s + lens[seq] - kq0), group)))


def pack_batch(
    modalities: list,
    times,                       # Float[b, m] (CPU tensor / ndarray) or None
    model,
    *,
    return_loss: bool,
    return_embed: bool,
    need_axial_pos_emb: bool = False,
    pad_rows: bool = False,
) -> RaggedBatch:
    """`pad_rows` (training batches): every sample is fed at the length of the longest, as in the reference's padded `[b, n]` layout
    (MP.py:573 pads with -1, T.py:3136-3144 shifts, T.py:3173 embeds -1 as token 0).  A shorter sample's pad positions are its last token,
    which the shift no longer cuts, then token 0: text rows with label -1, causal attention (they see their sample, no real row sees them) and
    continuing rotary positions.  They change no loss term (`total_tokens` and `n_valid` count the real tokens only); the Self-Flow
    representation loss averages over them as the reference does."""
    B = len(modalities)
    n_types = model.num_modalities
    times_np = None
    if times is not None:
        times_np = times.detach().float().cpu().numpy() if is_tensor(times) else np.asarray(times, dtype = np.float32)

    pieces, piece_inst, sample_piece0, full_lens = [], [], [], []     # id pieces of the WHOLE batch in order (run-length description of the token stream)
    instances: list[ModalityInstance] = []
    latents = [[] for _ in range(n_types)]
    type_counts = [0] * n_types
    modality_positions = []
    cond_times = []
    dim_latents, channel_first, num_dim = model.dim_latents, model.channel_first_latent, model.modality_num_dim
    n_time_cols = times_np.shape[1] if times_np is not None else 0
    for b, sample in enumerate(modalities):
        offset, mi, positions = 0, 0, []
        sample_piece0.append(len(pieces))
        for item in sample:
            if isinstance(item, tuple):
                mtype, mt = item[0], item[1]
            elif item.is_floating_point():
                mtype, mt = 0, item
            else:
                assert item.dtype in (torch.int, torch.long) and item.ndim <= 1, 'text must be a 0-d or 1-d int tensor'
                arr = item.numpy() if (item.device.type == 'cpu' and not item.requires_grad) else item.detach().cpu().numpy()
                if arr.ndim != 1:
                    arr = arr.reshape(-1)
                pieces.append(arr); piece_inst.append(-1); offset += arr.shape[0]
                continue
            assert 0 <= mtype < n_types, f'received a modality index that is out of range. only {n_types} modalities specified'
            dl = dim_latents[mtype]
            cf = channel_first[mtype]
            assert mt.shape[0 if cf else -1] == dl, f'mismatch for modality latent dimension - expected {dl} but received {mt.shape[0 if cf else -1]} - modality shape is {tuple(mt.shape)}, perhaps you need to set `channel_first_latent` to the correct value'
            nd = num_dim[mtype]
            assert nd is None or nd == mt.ndim - 1, f'mismatch for modality number of dimensions - expected {nd} but received {mt.ndim - 1} {tuple(mt.shape)}'
            axial = tuple(mt.shape[1:]) if cf else tuple(mt.shape[:-1])
            length = axial[0] if len(axial) == 1 else math.prod(axial)
            flat = (mt.reshape(dl, length).t() if cf else (mt if mt.ndim == 2 else mt.reshape(length, dl)))
            pre = 0
            if not return_embed:
                meta, eom = _meta_ids(model, axial, mtype)
                pieces.append(meta); piece_inst.append(-1); pre = meta.shape[0]
            pieces.append(_neg_ids(length)); piece_inst.append(len(instances))
            if not return_embed:
                pieces.append(eom); piece_inst.append(-1)
            t_val = float(times_np[b, mi]) if n_time_cols > mi else 0.
            inst = ModalityInstance(b, mtype, offset + pre, length, axial, type_counts[mtype], len(cond_times))
            cond_times.append(t_val)
            type_counts[mtype] += length
            latents[mtype].append(flat)
            instances.append(inst); positions.append((mtype, offset + pre, length))
            offset += pre + length + (0 if return_embed else 1)
            mi += 1
        full_lens.append(offset); modality_positions.append(positions)
    sample_piece0.append(len(pieces))

    total_tokens = sum(full_lens)
    if pad_rows and return_loss and B and min(full_lens) < max(full_lens):
        L, padded, p0 = max(full_lens), [], []
        for b in range(B):
            p0.append(len(padded))
            padded += [(p, i) for p, i in zip(pieces[sample_piece0[b]:sample_piece0[b + 1]], piece_inst[sample_piece0[b]:sample_piece0[b + 1]])]
            padded.append((_neg_ids(L - full_lens[b]), -1))
        pieces, piece_inst = [p for p, _ in padded], [i for _, i in padded]
        sample_piece0, full_lens = p0 + [len(padded)], [L] * B
    full_lens = np.asarray(full_lens, dtype = np.int64)
    drop = 1 if return_loss else 0
    seq_lens = np.maximum(full_lens - drop, 0)
    cu = np.zeros(B + 1, dtype = np.int64); np.cumsum(seq_lens, out = cu[1:])
    M = int(cu[-1])

    type_base = np.concatenate([[0], np.cumsum(type_counts)]).astype(np.int64)
    S = int(type_base[-1])

    # ---- per-token metadata from the run-length description of the token stream: every array is np.repeat over the ~7 pieces per sample plus
    # elementwise arithmetic - no per-sample / per-instance NumPy calls and no fancy-index scatters (both cost ~10 ms at 128 x 1024 tokens)
    P = len(pieces)
    plen = np.fromiter((p.shape[0] for p in pieces), dtype = np.int64, count = P)
    pinst = np.asarray(piece_inst, dtype = np.int64)
    fed_pieces, lab_pieces = pieces, None
    if drop and P:
        # training shift (T.py:3135-3144): the LAST token of every sample is not fed and the FIRST is never a label
        fed_pieces, lab_pieces, plen = list(pieces), list(pieces), plen.copy()
        for b in range(B):
            lo, hi = sample_piece0[b], sample_piece0[b + 1]
            j = hi - 1
            while j >= lo and plen[j] == 0: j -= 1
            if j >= lo:
                fed_pieces[j] = fed_pieces[j][:-1]; plen[j] -= 1
            j = lo
            while j < hi and lab_pieces[j].shape[0] == 0: j += 1
            if j < hi:
                lab_pieces[j] = lab_pieces[j][1:]
    ar = np.arange(M, dtype = np.int64)
    pstart = np.cumsum(plen) - plen
    is_mod = np.repeat(pinst >= 0, plen)
    qfirst64 = np.where(is_mod, np.repeat(pstart, plen), ar)
    # a span sees up to its last FED token (= its last token, unless the shift cut it: then the fed part ends with the sample)
    kv_limit = np.where(is_mod, np.repeat(pstart + plen - 1, plen), ar).astype(np.int32)
    qfirst = qfirst64.astype(np.int32)
    n_type_tokens = [0] * n_types
    row_token = np.full(S, -1, dtype = np.int32); row_time = np.zeros(S, dtype = np.float32)
    cond_row = np.full(M, -1, dtype = np.int32); slot = np.full(M, -1, dtype = np.int32)
    if instances:
        ni = len(instances)
        il = np.fromiter((i.length for i in instances), dtype = np.int64, count = ni)
        ity = np.fromiter((i.modality_type for i in instances), dtype = np.int64, count = ni)
        ir0 = type_base[ity] + np.fromiter((i.row0 for i in instances), dtype = np.int64, count = ni)
        ic = np.fromiter((i.cond_row for i in instances), dtype = np.int64, count = ni)
        ct = np.asarray(cond_times, dtype = np.float32)
        ipiece = np.nonzero(pinst >= 0)[0]                               # piece of every instance (instances are numbered in piece order)
        cnt, tok0 = plen[ipiece], pstart[ipiece]                         # fed tokens of the instance, packed index of its first token
        for inst, c, t0 in zip(instances, cnt.tolist(), tok0.tolist()):
            if c:
                inst.token0 = t0
        pc = np.full(P, -1, dtype = np.int64); pc[ipiece] = ic
        pr = np.zeros(P, dtype = np.int64); pr[ipiece] = ir0 - tok0
        cond_row = np.repeat(pc, plen).astype(np.int32)
        slot = np.where(is_mod, np.repeat(pr, plen) + ar, -1).astype(np.int32)
        # compact rows: the instances tile [0, S) in (type, scan) order
        order = np.argsort(ir0, kind = 'stable')
        il_s, r0_s = il[order], ir0[order]
        rr = np.arange(S, dtype = np.int64) - np.repeat(r0_s, il_s)      # row index inside its instance
        row_token = np.where(rr < np.repeat(cnt[order], il_s), np.repeat(tok0[order], il_s) + rr, -1).astype(np.int32)
        row_time = np.repeat(ct[ic[order]], il_s)                        # the time of EVERY compact row (also of rows the shift dropped)
        n_type_tokens = [int(c) for c in np.bincount(ity, weights = cnt, minlength = n_types)]
    text_id = np.zeros(M, dtype = np.int32); label = np.full(M, -1, dtype = np.int32); rope_pos = np.zeros(M, dtype = np.int32)
    max_rope = 0
    if M:
        ids_fed = np.concatenate(fed_pieces)
        assert ids_fed.shape[0] == M
        text_id = np.maximum(ids_fed, 0).astype(np.int32)
        seq_of = np.repeat(np.arange(B), seq_lens)
        seq_start = cu[:-1][seq_of]
        ce = np.cumsum(is_mod & (ar != qfirst64))                        # transfusion.py:398-415: tokens of a span share the position of its first token
        before = np.where(seq_start > 0, ce[np.maximum(seq_start - 1, 0)], 0)
        pos = (ar - seq_start) - (ce - before)
        rope_pos = pos.astype(np.int32)
        max_rope = int(pos.max())
        if return_loss:
            lab = np.concatenate(lab_pieces).astype(np.int64)              # next token (transfusion.py:3144)
            assert lab.shape[0] == M
            lab[is_mod] = -1                                               # transfusion.py:3320
            lab[lab == model.null_text_id] = -1                            # transfusion.py:3323
            label = lab.astype(np.int32)

    rb = RaggedBatch(
        B = B, M = M, seq_lens = seq_lens, cu = cu, full_lens = full_lens, text_id = text_id, label = label, kv_limit = kv_limit,
        rope_pos = rope_pos, cond_row = cond_row, slot = slot, n_cond = len(cond_times),
        cond_times = np.asarray(cond_times, dtype = np.float32), n_types = n_types,
        type_rows = [(int(type_base[t]), int(type_base[t + 1])) for t in range(n_types)], row_token = row_token, row_time = row_time,
        latents = latents, instances = instances, modality_positions = modality_positions,
        total_tokens = int(total_tokens), n_type_tokens = n_type_tokens, max_rope_pos = max_rope, has_labels = return_loss)
    rb.n_valid = int((label >= 0).sum())
    add_pos = getattr(model, 'add_pos_emb', None)
    if add_pos is not None and any(add_pos) and instances:
        # axial positional embedding (T.py:2792-2796; MP.py:1003-1046): row-major coordinates of every latent row inside its instance; the engine
        # evaluates one factorised table per (type, axis) at the batch maximum and gathers with these
        coords = [np.full(S, -1, dtype = np.int32) for _ in range(3)]
        pmax = [None] * n_types
        for inst in instances:
            t = inst.modality_type
            if not add_pos[t]:
                continue
            ax = tuple(int(a) for a in inst.axial_shape)
            assert len(ax) <= 3, 'axial positional embeddings are implemented for up to 3 axes'
            r0 = int(type_base[t]) + inst.row0
            for a, c in enumerate(np.unravel_index(np.arange(inst.length), ax)):
                coords[a][r0:r0 + inst.length] = c
            pmax[t] = ax if pmax[t] is None else tuple(max(x, y) for x, y in zip(pmax[t], ax))
        rb.pos_c0, rb.pos_c1, rb.pos_c2 = coords
        rb.pos_max = tuple(None if m is None else tuple((x + 7) // 8 * 8 for x in m) for m in pmax)
    if getattr(model, 'has_recon_loss', False):
        build_recon_meta(rb)
    build_tiles(rb, qfirst)
    return rb


def build_recon_meta(rb: RaggedBatch) -> None:
    """Per-row instance index and per-instance weights of the reconstruction loss (T.py:3299-3308, 3420-3431): the loss of a type is the mean
    over its instances of each instance's MSE, so instance i weighs 1 / (K_t n_i) (K_t instances of its type, n_i rows).  Both arrays are
    sized by S, so their shapes depend only on the batch's shape signature; the values travel in the metadata upload (a replayed CUDA graph
    reads them from the device)."""
    S = rb.S
    row_inst = np.zeros(S, dtype = np.int32)
    inst_w = np.zeros(S, dtype = np.float32)
    if rb.instances:
        ni = len(rb.instances)
        il = np.fromiter((i.length for i in rb.instances), dtype = np.int64, count = ni)
        ity = np.fromiter((i.modality_type for i in rb.instances), dtype = np.int64, count = ni)
        base = np.asarray([s0 for s0, _ in rb.type_rows], dtype = np.int64)
        ir0 = base[ity] + np.fromiter((i.row0 for i in rb.instances), dtype = np.int64, count = ni)
        order = np.argsort(ir0, kind = 'stable')                        # compact rows hold the instances in (type, scan) order
        row_inst[:] = np.repeat(order, il[order])
        k = np.bincount(ity, minlength = rb.n_types)
        inst_w[:ni] = 1. / (k[ity] * np.maximum(il, 1))
    rb.row_inst, rb.inst_w = row_inst, inst_w


def pack_incremental(samples: list, times, model, *, slab: np.ndarray, base_len: np.ndarray, rope_base: np.ndarray, cap: int) -> RaggedBatch:
    """Descriptor of a kv-cache (incremental) forward: `samples[b]` are the NEW parts of sample b (a whole prompt for the prefill, one token
    for a text step, one `(type, latents)` for a modality step), appended to cache slab `slab[b]` which already holds `base_len[b]` rows.

    The token layout / mask / positions are those of `pack_batch(return_embed = True)` (no [meta] / [som] / [eom] are added around
    modalities, as in the reference's decode-time calls: T.py:2194-2201, 2389-2406) shifted into cache-row coordinates:
      * `kv_row[i]`   = slab start + base_len + local position            (where the QKVG epilogue appends the token's key / value)
      * `kv_limit[i]` = slab start + base_len + local limit               (the cached prefix - rows from the slab start - is always visible:
                                                                           decode-time attention is un-masked over the cache, T.py:938-939)
      * attention tiles: keys from the slab start up to the tile's largest limit
      * RoPE position  = local position (span-shared, T.py:398-415) + rope_base[b]   (`tokens_seen`, T.py:3211-3219)."""
    rb = pack_batch(samples, times, model, return_loss = False, return_embed = True)
    B, M = rb.B, rb.M
    slab, base_len, rope_base = (np.asarray(a, dtype = np.int64) for a in (slab, base_len, rope_base))
    assert slab.shape == base_len.shape == rope_base.shape == (B,)
    assert ((base_len + rb.seq_lens) <= cap).all(), 'kv cache slab overflow: a sample needs more rows than the slab capacity'
    off = slab * cap + base_len - rb.cu[:-1]                   # packed token index -> cache row
    seq = np.repeat(np.arange(B), rb.seq_lens)
    rb.kv_row = (np.arange(M, dtype = np.int64) + off[seq]).astype(np.int32)
    rb.kv_limit = (rb.kv_limit.astype(np.int64) + off[seq]).astype(np.int32)
    rb.rope_pos = (rb.rope_pos.astype(np.int64) + rope_base[seq]).astype(np.int32)
    rb.max_rope_pos = int(rb.rope_pos.max()) if M else 0
    for pre in ('tile', 't2'):
        q0 = getattr(rb, f'{pre}_q0')
        if q0.shape[0] == 0:
            continue
        ts = np.searchsorted(rb.cu, q0, side = 'right') - 1      # sequence of every query tile
        setattr(rb, f'{pre}_kv0', (slab[ts] * cap).astype(np.int32))
        setattr(rb, f'{pre}_kvend', (getattr(rb, f'{pre}_kvend').astype(np.int64) + off[ts]).astype(np.int32))
    rb.single_row_tiles = bool(M > 0 and (rb.seq_lens <= 1).all())
    return rb


def pack_text_only(text: Tensor, *, return_loss: bool, pos_offset: int = 0) -> RaggedBatch:
    """`Int[b, n]` pretraining path (transfusion.py:2585-2664): causal mask, arange positions."""
    t = text.detach().cpu().numpy().astype(np.int64)
    B, L = t.shape
    n = L - 1 if return_loss else L
    M = B * n
    cu = np.arange(B + 1, dtype = np.int64) * n
    tid = t[:, :n].reshape(-1)
    label = np.full(M, -1, dtype = np.int32)
    if return_loss:
        label = t[:, 1:].reshape(-1).astype(np.int32)
    rb = RaggedBatch(
        B = B, M = M, seq_lens = np.full(B, n, dtype = np.int64), cu = cu, full_lens = np.full(B, L, dtype = np.int64),
        text_id = np.where(tid < 0, 0, tid).astype(np.int32), label = label, kv_limit = np.arange(M, dtype = np.int32),
        rope_pos = (np.tile(np.arange(n, dtype = np.int32), B) + pos_offset).astype(np.int32), cond_row = np.full(M, -1, dtype = np.int32),
        slot = np.full(M, -1, dtype = np.int32), n_cond = 0, cond_times = np.zeros(0, dtype = np.float32), n_types = 0, type_rows = [],
        row_token = np.zeros(0, dtype = np.int32), row_time = np.zeros(0, dtype = np.float32), latents = [], instances = [],
        modality_positions = [[] for _ in range(B)], total_tokens = B * L, n_type_tokens = [], max_rope_pos = n - 1 + pos_offset,
        has_labels = return_loss)
    rb.n_valid = int((label >= 0).sum())
    build_tiles(rb, np.arange(M, dtype = np.int32))
    return rb


# --------------------------------------------------------------------------------------------- registry (API parity)
def _strategy(name):
    def fn(modalities, times, model, *, need_axial_pos_emb, return_loss, return_embed, pad_rows = False):
        return pack_batch(modalities, times, model, return_loss = return_loss, return_embed = return_embed, need_axial_pos_emb = need_axial_pos_emb,
                          pad_rows = pad_rows)
    fn.__name__ = f'process_modality_batch_{name}'
    return fn

PROCESSING_STRATEGIES: dict[str, Callable] = {name: _strategy(name) for name in ('naive', 'grouped', 'flat', 'hybrid', 'auto')}
DEFAULT_PROCESSING_STRATEGY = 'auto'


def get_processing_strategy(name: str):
    assert name in PROCESSING_STRATEGIES, f'unknown modality processing strategy `{name}`, available: {list(PROCESSING_STRATEGIES)}'
    return PROCESSING_STRATEGIES[name]
