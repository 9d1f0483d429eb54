"""GPU: the kernels around the block stack - loss, conditioning, bias gradients, weight repack, optimizer step, token / flow path
and the RoPE table - each called through the C ABI and compared with a float64 restatement of its formula.

Tolerances:
  - copies and casts are compared bit for bit (int16 / int32 views); torch's fp32 -> bf16 cast rounds to nearest even, like the kernels;
  - a bf16 output may differ from the float64 value by the rounding of the cast, |got - ref| <= 2^-8 |ref|, plus the few fp32 roundings the
    kernel makes before the cast (stated per test);
  - fp32 results and fp32 / fp64 accumulators: a relative error of about 1e-6.  One fp32 rounding is 2^-24 = 6e-8 relative; a kernel makes a
    handful of them per element, and a sum of many positive terms in fp32 partials drifts by ~sqrt(terms) roundings, so 1e-6 leaves room for
    that and is still four orders of magnitude below a wrong constant, a dropped term or a skipped row.
Shapes are large enough for every grid-stride / multi-row loop to run more than once: element-wise kernels cap their grid at
num_SMs x 16 blocks of 256 threads (n >= 4M), the warp-per-row kernels at num_SMs x 8 blocks of 8 warps (rows > 8448), CE at num_SMs x 64 warps.
Bytes a kernel must not touch (padding columns, skipped rows, a guard row past the end) hold a sentinel and are checked unchanged."""
import math

import numpy as np
import pytest
import torch

from transfusion_pytorch_b200 import _lib, engine as E

pytestmark = pytest.mark.gpu
BF16, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
FLT_MAX = float(np.finfo(np.float32).max)
U32 = 2.0 ** -24                      # one fp32 rounding, relative
DISPATCH_D = (128, 256, 384, 512, 768, 1024)      # TFX_DISPATCH_NCH


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


def gen(seed):
    return torch.Generator(device = 'cuda').manual_seed(seed)


def assert_bf16_close(got, ref, slack = 0.0, what = ''):
    """got (bf16) within the bf16 rounding of the float64 value ref, plus `slack` (absolute, broadcastable) for fp32 work before the cast"""
    err = (got.double() - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + slack + 1e-37
    bad = err > bound
    assert not bad.any(), f'{what}: {int(bad.sum())} bf16 values off, worst excess {(err - bound).max().item():.3e}'


def assert_close64(got, ref, scale, rel = 1e-6, what = ''):
    """|got - ref| <= rel * scale (+ a denormal floor): ref float64, scale the magnitude of the terms that produced ref"""
    err = (got.double() - ref).abs()
    bound = rel * scale + 1e-37
    bad = err > bound
    assert not bad.any(), f'{what}: {int(bad.sum())} values off, worst err / bound {(err / bound).max().item():.3e}'


def same_bits(a, b):
    view = {BF16: torch.int16, F32: torch.int32, torch.float16: torch.int16}
    return torch.equal(a.view(view[a.dtype]), b.view(view[b.dtype]))


def bf16_ties(x, g, frac = 8):
    """overwrite every `frac`-th value (random positions) with an fp32 value half-way between two bf16 values (round-to-nearest-even ties)"""
    flat = x.view(-1)
    idx = torch.randint(0, flat.numel(), (max(1, flat.numel() // frac),), device = x.device, generator = g)
    bits = flat[idx].view(torch.int32)
    flat[idx] = ((bits & ~0xFFFF) | 0x8000).view(F32)
    return x


# ------------------------------------------------------------------------------------------------ text cross-entropy
def ce_check(logits, labels, V, vlimit, gscale, dlog, what, chunk = 4096):
    """float64 restatement of T.py:3320-3331 (text-only 2653-2659, logits >= vlimit masked before the cross entropy).  Checks the
    gradient dlog[:, :V] of gscale * loss_row chunk by chunk and returns (sum of the row losses over rows with a label, their count)"""
    M = labels.shape[0]
    Vu = vlimit if vlimit > 0 else V
    loss, cnt = 0.0, 0
    for r0 in range(0, M, chunk):
        x = logits[r0:r0 + chunk, :Vu].double()
        lab = labels[r0:r0 + chunk].long()
        ok = lab >= 0
        lse = torch.logsumexp(x, dim = 1)
        p = torch.zeros(x.shape[0], V, dtype = F64, device = x.device)
        p[:, :Vu] = torch.softmax(x, dim = 1) * gscale
        p[~ok] = 0
        rows = torch.nonzero(ok).squeeze(1)
        loss += (lse[rows] - x[rows, lab[rows]]).sum().item()
        cnt += int(ok.sum())
        ref = p.clone()
        ref[rows, lab[rows]] -= gscale
        # softmax: __expf of (x - max) with |x - max| up to ~40 carries ~|x - max| * 2^-24 relative error before the subtraction and the cast
        assert_bf16_close(dlog[r0:r0 + x.shape[0], :V], ref, slack = 1e-5 * (p + ref.abs()), what = f'{what} rows {r0}..')
    return loss, cnt


@pytest.mark.parametrize('V', [390, 32768])        # the bench config's text vocabulary (256 tokens + specials), and a large one
def test_ce_fwd_bwd(ops, V):
    M, gscale = 20000, 0.37
    ld_l, ld_d = V + 5, (V + 7) // 8 * 8 + 8
    g = gen(1)
    logits = torch.full((M + 1, ld_l), 1e30, device = 'cuda')          # padding past V must never be read: 1e30 would own the max
    logits[:, :V] = 80. + 4. * torch.randn(M + 1, V, device = 'cuda', generator = g)
    for vlimit in (0, V * 3 // 4):
        Vu = vlimit or V
        labels = torch.randint(0, Vu, (M + 1,), device = 'cuda', generator = g, dtype = I32)
        labels[torch.rand(M + 1, device = 'cuda', generator = g) < 0.1] = -1
        dlog = torch.full((M + 1, ld_d), -7., device = 'cuda', dtype = BF16)
        loss = torch.tensor([123.5], device = 'cuda', dtype = F64)
        nval = torch.tensor([7], device = 'cuda', dtype = I32)
        ops.ce_fwd_bwd(logits, ld_l, labels, V, vlimit, gscale, dlog, ld_d, loss, nval, M)
        ref_loss, ref_cnt = ce_check(logits[:M], labels[:M], V, vlimit, gscale, dlog, f'dlogits V={V} vlimit={vlimit}')
        assert int(nval.item()) == 7 + ref_cnt
        # per row, lse is an fp32 value near 90 (one rounding ~5e-6 against a row loss of ~10), the sum over rows is double
        assert abs(loss.item() - (123.5 + ref_loss)) <= 2e-6 * (123.5 + ref_loss), (loss.item(), 123.5 + ref_loss)
        assert not dlog[:M, V:].float().any(), 'columns past V must be zero'
        assert torch.equal(dlog[M], torch.full_like(dlog[M], -7.)), 'row past M touched'
        ign = labels[:M] < 0
        assert not dlog[:M][ign].float().any(), 'ignored rows must be zero over the whole pitch'
        if vlimit:
            assert not dlog[:M, vlimit:].float().any(), 'masked vocabulary columns must get zero gradient'
    # a label at or above vlimit (text-only path): the reference sees the -FLT_MAX fill -> loss lse + FLT_MAX, gradient -gscale on its column
    vlimit = V * 3 // 4
    labels = torch.full((M,), -1, device = 'cuda', dtype = I32)
    rows = torch.tensor([5, 9000, M - 1], device = 'cuda')
    labels[rows] = torch.tensor([vlimit, V - 1, vlimit + 1], device = 'cuda', dtype = I32)
    dlog = torch.full((M, ld_d), -7., device = 'cuda', dtype = BF16)
    loss = torch.zeros(1, device = 'cuda', dtype = F64); nval = torch.zeros(1, device = 'cuda', dtype = I32)
    ops.ce_fwd_bwd(logits, ld_l, labels, V, vlimit, gscale, dlog, ld_d, loss, nval, M)
    x = logits[rows, :vlimit].double()
    want = (torch.logsumexp(x, 1) + FLT_MAX).sum().item()
    assert int(nval.item()) == 3 and abs(loss.item() - want) <= 1e-12 * want
    p = torch.softmax(x, 1) * gscale
    assert_bf16_close(dlog[rows, :vlimit], p, slack = 1e-5 * p, what = 'softmax of a row with a masked label')
    lab = labels[rows].long()
    assert torch.equal(dlog[rows, lab].float(), torch.full((3,), -gscale, device = 'cuda').to(BF16).float())
    dlog[rows, lab] = 0
    assert not dlog[:, vlimit:].float().any()
    assert not dlog[labels < 0].float().any()


# ------------------------------------------------------------------------------------------------ flow-match noise
@pytest.mark.parametrize('with_eps,with_f32', [(True, True), (True, False), (False, False)])
def test_flow_noise(ops, with_eps, with_f32):
    S, dl, ld = 42011, 100, 104
    g = gen(2)
    x = torch.randn(S, dl, device = 'cuda', generator = g)
    eps = torch.randn(S, dl, device = 'cuda', generator = g)
    t = torch.rand(S, device = 'cuda', generator = g)
    t[:3] = torch.tensor([0., 1., 0.5], device = 'cuda')
    noised = torch.full((S + 1, ld), -7., device = 'cuda', dtype = BF16)
    nf = torch.full((S, dl), 5., device = 'cuda'); flow = torch.full((S, dl), 5., device = 'cuda')
    ops.flow_noise(x, eps if with_eps else None, t, noised, ld, nf if with_f32 else None, flow if with_f32 else None, S, dl)
    if with_eps:
        tt = t.double()[:, None]
        ref = x.double() * tt + eps.double() * (1 - tt)
        scale = (x.double() * tt).abs() + (eps.double() * (1 - tt)).abs()          # a multiply-add in fp32: two roundings of the terms
        assert_bf16_close(noised[:S, :dl], ref, slack = 3 * U32 * scale, what = 'noised')
        if with_f32:
            assert_close64(nf, ref, scale, rel = 3 * U32, what = 'noised fp32')
            assert same_bits(flow, x - eps)                                          # one fp32 subtraction
        else:
            assert (nf == 5.).all() and (flow == 5.).all()
    else:
        assert same_bits(noised[:S, :dl], x.to(BF16))
    assert (noised[:S, dl:].float() == -7.).all() and (noised[S].float() == -7.).all()


# ------------------------------------------------------------------------------------------------ time features
@pytest.mark.parametrize('D', [128, 512, 1024])
def test_time_features(ops, D):
    half = D // 2
    Kt = (D + 1 + 63) // 64 * 64                       # the engine's padded K of the time-cond Linear
    n = -(-(4 << 20) // Kt)
    g = gen(3)
    t = torch.rand(n, device = 'cuda', generator = g)
    t[:2] = torch.tensor([0., 1.], device = 'cuda')
    w = torch.randn(half, device = 'cuda', generator = g)
    feats = torch.full((n + 1, Kt), -7., device = 'cuda', dtype = BF16)
    ops.time_features(t, w, feats, n, half, Kt)
    # RandomFourierEmbed (T.py:625-635) forms the angle in fp32 as t * w * 2 * pi; sin / cos of that fp32 angle in float64
    ang = (t[:, None] * w[None, :] * torch.tensor(2., device = 'cuda')) * torch.tensor(math.pi, device = 'cuda', dtype = F32)
    ref_s, ref_c = torch.sin(ang.double()), torch.cos(ang.double())
    assert same_bits(feats[:n, 0].contiguous(), t.to(BF16))
    assert_bf16_close(feats[:n, 1:half + 1], ref_s, slack = 2 * 2 * U32 * ref_s.abs(), what = 'sin')        # sinf / cosf: <= 2 ulp
    assert_bf16_close(feats[:n, half + 1:2 * half + 1], ref_c, slack = 2 * 2 * U32 * ref_c.abs(), what = 'cos')
    assert not feats[:n, 2 * half + 1:].float().any(), 'padding columns must be exactly zero'
    assert (feats[n].float() == -7.).all()


# ------------------------------------------------------------------------------------------------ conditioning table ops
def table_ref(op, a, b):
    """float64 restatement of the five table ops; returns (value, magnitude of the terms for the fp32 error bound)"""
    x = a.double()
    if op == 0:
        y = torch.sigmoid(x); return y, y.abs()
    if op == 1:
        y = x * torch.sigmoid(x); return y, y.abs()
    z = b.double()
    if op == 2:                                   # sigmoid backward: g * s * (1 - s), s = b
        y = x * z * (1 - z); return y, (x * z).abs() * (1 + z.abs())
    if op == 3:                                   # silu backward: g * s * (1 + z (1 - s)), s = sigmoid(z)
        s = torch.sigmoid(z)
        return x * (s * (1 + z * (1 - s))), x.abs() * s * (1 + z.abs() * (1 - s))
    return x, x.abs()


@pytest.mark.parametrize('op', [0, 1, 2, 3, 4])
def test_table_op(ops, op):
    rows, cols = 8203, 515                        # n = 4.2M, odd column count
    ld_a, ld_b, ld_of, ld_ob = 3 * cols + 3, cols + 17, cols + 5, cols + 9        # column slices of wider tables, as the engine passes them
    g = gen(4 + op)
    a = torch.randn(rows, ld_a, device = 'cuda', generator = g) * 3
    b = torch.randn(rows, ld_b, device = 'cuda', generator = g) * 3
    if op == 2:
        b = torch.rand(rows, ld_b, device = 'cuda', generator = g)      # a sigmoid output
    sat = torch.rand(rows, ld_a, device = 'cuda', generator = g) < 0.01
    a[sat] = 100. * torch.sign(torch.randn(int(sat.sum()), device = 'cuda', generator = g))
    if op == 3:
        satb = torch.rand(rows, ld_b, device = 'cuda', generator = g) < 0.01
        b[satb] = 100. * torch.sign(torch.randn(int(satb.sum()), device = 'cuda', generator = g))
    ref, scale = table_ref(op, a[:, :cols], b[:, :cols])
    for want_f32, want_bf16 in ((True, True), (True, False), (False, True)):
        of = torch.full((rows + 1, ld_of), 5., device = 'cuda')
        ob = torch.full((rows + 1, ld_ob), -7., device = 'cuda', dtype = BF16)
        ops.table_op(a, ld_a, b if op in (2, 3) else None, ld_b, of if want_f32 else None, ld_of, ob if want_bf16 else None, ld_ob, rows, cols, op)
        if want_f32:
            assert torch.isfinite(of[:rows, :cols]).all()
            assert_close64(of[:rows, :cols], ref, scale, rel = 1e-6, what = f'op {op} fp32')
            assert (of[:rows, cols:] == 5.).all() and (of[rows] == 5.).all()
        else:
            assert (of == 5.).all()
        if want_bf16:
            assert_bf16_close(ob[:rows, :cols], ref, slack = 1e-6 * scale, what = f'op {op} bf16')
            assert (ob[:rows, cols:].float() == -7.).all() and (ob[rows].float() == -7.).all()
        else:
            assert (ob.float() == -7.).all()


# ------------------------------------------------------------------------------------------------ column sums (bias gradients)
def col_map_with_holes(N, n_out, g):
    m = torch.randperm(n_out, device = 'cuda', generator = g)[:N].to(I32)
    m[torch.rand(N, device = 'cuda', generator = g) < 0.1] = -1
    m[-1] = n_out - 1                             # the odd last column lands somewhere
    return m


def colsum_expect(x64, col_map, out0):
    out = out0.double().clone()
    if col_map is None:
        return out + x64.sum(0), out0.double().abs() + x64.abs().sum(0)
    keep = col_map >= 0
    idx = col_map[keep].long()                    # two columns may share an output
    out.index_add_(0, idx, x64.sum(0)[keep])
    sc = out0.double().abs().index_add_(0, idx, x64.abs().sum(0)[keep])
    return out, sc


@pytest.mark.parametrize('mapped', [False, True])
def test_colsum_bf16(ops, mapped):
    M, N, ld = 20077, 1413, 1420                  # M not a multiple of the 256 rows per block; odd N; even ld (4-byte aligned column pairs)
    g = gen(10)
    x = (torch.randn(M, ld, device = 'cuda', generator = g) * 2).to(BF16)
    n_out = N + 7 if mapped else N
    cmap = col_map_with_holes(N, n_out, g) if mapped else None
    out = torch.randn(n_out, device = 'cuda', generator = g)
    want, scale = colsum_expect(x[:, :N].double(), cmap, out)
    out0 = out.clone()
    ops.colsum_bf16(x, ld, M, N, cmap, out)
    # fp32 partial sums over <= 256 rows per block, added with fp32 atomics: error relative to the sum of |terms|
    assert_close64(out, want, scale, rel = 1e-6, what = 'colsum_bf16')
    colsum_untouched(out, out0, cmap)


def colsum_untouched(out, out0, cmap):
    """outputs no column maps to keep their bits"""
    if cmap is None:
        return
    untouched = torch.ones(out.shape[0], dtype = torch.bool, device = 'cuda')
    untouched[cmap[cmap >= 0].long()] = False
    assert untouched.any() and same_bits(out[untouched], out0[untouched])


@pytest.mark.parametrize('mapped', [False, True])
def test_colsum_f32(ops, mapped):
    M, N, ld = 20033, 1413, 1415                  # M not a multiple of the 64 rows per block
    g = gen(11)
    x = torch.randn(M, ld, device = 'cuda', generator = g)
    n_out = N + 7 if mapped else N
    cmap = col_map_with_holes(N, n_out, g) if mapped else None
    out = torch.randn(n_out, device = 'cuda', generator = g)
    want, scale = colsum_expect(x[:, :N].double(), cmap, out)
    out0 = out.clone()
    ops.colsum_f32(x, ld, M, N, cmap, out)
    assert_close64(out, want, scale, rel = 1e-6, what = 'colsum_f32')
    colsum_untouched(out, out0, cmap)


# ------------------------------------------------------------------------------------------------ weight repack
def pack_expect(src2d, c_src, row_src, r_dst, c_dst):
    """fp32 [r_dst][c_dst] of a pack job: row gather (-1 = zero row), the first c_src columns of the source row, zero padding"""
    out = torch.zeros(r_dst, c_dst, device = 'cuda', dtype = F32)
    rs = row_src.long() if row_src is not None else torch.arange(r_dst, device = 'cuda')
    ok = rs >= 0
    out[ok, :c_src] = src2d[rs[ok], :c_src]
    return out


def strided(base, ld, rows, cols):
    return torch.as_strided(base, (rows, cols), (ld, 1))


def test_cast_pack_multi_paths(ops):
    g = gen(12)
    SENT = -7.
    jobs, checks = [], []

    def add(name, src_rows, ld_src, c_src, r_dst, c_dst, row_src = None, f32 = False, src_offset = 0, vec = None):
        base = bf16_ties(torch.randn(src_rows * ld_src + src_offset + 4, device = 'cuda', generator = g), g)
        src = base[src_offset:]
        dtype = F32 if f32 else BF16
        buf = torch.full((r_dst * c_dst + 64,), SENT, device = 'cuda', dtype = dtype)      # guard past the destination
        rs = torch.from_numpy(row_src.astype(np.int32)).cuda() if row_src is not None else None
        jobs.append((src, ld_src, c_src, rs, buf, r_dst, c_dst, 1 if f32 else 0))
        aligned = src.data_ptr() % 16 == 0
        path = c_dst % 8 == 0 and c_src % 4 == 0 and ld_src % 4 == 0 and not f32 and aligned
        assert vec is None or path == vec, name
        checks.append((name, buf, pack_expect(strided(src, ld_src, src_rows, ld_src), c_src, rs, r_dst, c_dst).to(dtype), r_dst * c_dst, rs))

    add('vector', 301, 512, 512, 301, 512, vec = True)                                            # 301 x 512: not a multiple of 2048
    add('vector, partial chunk and zero padding', 64, 1364, 1364, 64, 1408, vec = True)            # C_src < C_dst, the last source chunk is half full
    add('scalar, C_dst % 8 != 0', 257, 100, 90, 257, 100, vec = False)
    add('scalar, ld_src % 4 != 0 (time-cond weight, ld = D + 1)', 2048, 513, 513, 2048, 576, vec = False)
    add('scalar, ld_src % 4 == 3', 200, 515, 512, 200, 512, vec = False)
    add('scalar, misaligned source', 300, 512, 512, 300, 512, src_offset = 1, vec = False)
    for inner, D in ((1365, 512), (341, 128)):                                                    # GEGLU W1 / b1 interleave with -1 rows
        src = E.w1_row_src(inner)
        Ip2 = src.shape[0]
        add(f'W1 gather inner={inner}', 2 * inner, D, D, Ip2, D, row_src = src, vec = True)
        add(f'b1 gather inner={inner} (fp32)', 2 * inner, 1, 1, Ip2, 1, row_src = src, f32 = True, vec = False)
    add('fp32 destination', 100, 37, 37, 100, 40, f32 = True, vec = False)
    tab, blk_job, blk_first, nb = E.pack_job_table(jobs, torch.device('cuda'))
    ops.cast_pack_multi(tab, blk_job, blk_first, nb)
    for name, buf, want, n, rs in checks:
        assert same_bits(buf[:n], want.reshape(-1)), name
        assert (buf[n:].float() == SENT).all(), f'{name}: wrote past the destination'
        if rs is not None:
            assert not buf[:n].view(want.shape)[rs < 0].float().any(), f'{name}: -1 rows must be zero'


ENGINE_MODELS = {
    'd512': dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), transformer = dict(dim = 512, depth = 2)),
    'd128': dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), transformer = dict(dim = 128, depth = 2, heads = 2)),
    'd1536': dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)), transformer = dict(dim = 1536, depth = 2, heads = 8)),
    'd2048': dict(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)),
                  transformer = dict(dim = 2048, depth = 2, heads = 16, dim_head = 128)),
    'd384h3x128vres': dict(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,),
                           transformer = dict(dim = 384, depth = 3, heads = 3, dim_head = 128, use_value_residual = True)),
}


def packed_layout(eng):
    """every bf16 / fp32 GEMM operand of the engine rebuilt in torch from the fp32 parameters (the layouts of Engine._build_pack_jobs)"""
    D, HI, H, Ip, inner, P = eng.D, eng.HI, eng.H, eng.Ip, eng.inner, eng.P
    src = torch.from_numpy(E.w1_row_src(inner)).cuda()
    ok = src >= 0
    out = {}
    def pad(w, rows, cols):
        t = torch.zeros(rows, cols, device = 'cuda'); t[:w.shape[0], :w.shape[1]] = w; return t
    for i in range(eng.depth):
        pre = f'transformer.layers.{i}'
        wq = torch.zeros(eng.NQ, D, device = 'cuda')
        wq[:2 * HI] = P(f'{pre}.1.fn.to_qk.0.weight'); wq[2 * HI:3 * HI] = P(f'{pre}.1.fn.to_v.0.weight'); wq[3 * HI:3 * HI + H] = P(f'{pre}.1.fn.to_gates.0.weight')
        if f'{pre}.1.fn.to_learned_value_residual.0.weight' in eng.named:
            # the mix rows start at the first even row behind the gates, so that the bf16 pairs of their gradient columns stay 4-byte
            # aligned: one pad row between them at an odd head count (dim_head 128 only)
            mix = 3 * HI + H + H % 2
            wq[mix:mix + H] = P(f'{pre}.1.fn.to_learned_value_residual.0.weight')
        out[f'qkvg{i}'] = wq
        out[f'wo{i}'] = P(f'{pre}.1.fn.to_out.1.weight')
        w1 = torch.zeros(2 * Ip, D, device = 'cuda'); w1[ok] = P(f'{pre}.2.fn.net.0.weight')[src[ok]]
        b1 = torch.zeros(2 * Ip, device = 'cuda'); b1[ok] = P(f'{pre}.2.fn.net.0.bias')[src[ok]]
        out[f'w1{i}'], out[f'b1{i}'] = w1, b1
        out[f'w2{i}'] = pad(P(f'{pre}.2.fn.net.3.weight'), D, Ip)
        if f'{pre}.0.weight' in eng.named:
            out[f'wskip{i}'] = P(f'{pre}.0.weight')
    out['wvocab'] = P('to_text_logits.weight')
    for t, dlp in enumerate(eng.dlp):
        out[f'wm2l{t}'] = P(f'model_to_latent_projs.{t}.weight')
        if f'latent_to_model_projs.{t}.weight' in eng.named:
            out[f'wl2m{t}'] = pad(P(f'latent_to_model_projs.{t}.weight'), D, dlp)
    out['wt'] = pad(P('transformer.to_time_cond.1.weight'), 4 * D, eng.Kt)
    wfz, bfz = [], []
    for w in range(eng.W):
        i, j = divmod(w, 2)
        pre = f'transformer.layers.{i}.{j + 1}'
        wfz += [P(f'{pre}.to_film.weight'), P(f'{pre}.to_ada_ln_zero.weight')]
        bfz += [P(f'{pre}.to_film.bias'), P(f'{pre}.to_ada_ln_zero.bias')]
    out['wfz'], out['bfz'] = torch.cat(wfz), torch.cat(bfz)
    return out


@pytest.mark.parametrize('model', sorted(ENGINE_MODELS))
def test_cast_pack_multi_engine_layout(ops, model):
    from transfusion_pytorch_b200 import Transfusion
    torch.manual_seed(0)
    m = Transfusion(**ENGINE_MODELS[model]).cuda()
    eng = m.engine
    eng.ensure_attached()
    g = gen(13)
    for seed in range(2):                         # the second pack must overwrite every value of the first
        with torch.no_grad():
            eng.flat.copy_(bf16_ties(torch.randn(eng.flat.shape, device = 'cuda', generator = g), g))
        eng.pack_weights(force = True)
        want = packed_layout(eng)
        assert set(want) == set(eng.packed), sorted(set(want) ^ set(eng.packed))
        for name, w in want.items():
            got = eng.packed[name]
            assert got.shape == w.shape, name
            assert same_bits(got, w.to(got.dtype)), f'{name} (pass {seed})'


# ------------------------------------------------------------------------------------------------ casts, scale, axpy
def test_cast_scale_axpy(ops):
    n = (4 << 20) + 3
    g = gen(14)
    x = bf16_ties(torch.randn(n + 8, device = 'cuda', generator = g) * 3, g)
    x[:4] = torch.tensor([FLT_MAX, -FLT_MAX, 1e-40, -0.], device = 'cuda')       # overflow to inf, a denormal, negative zero
    out = torch.full((n + 8,), -7., device = 'cuda', dtype = BF16)
    ops.cast_bf16(x, out, n)
    assert same_bits(out[:n], x[:n].to(BF16)) and (out[n:].float() == -7.).all()
    p = (torch.randn(n + 8, device = 'cuda', generator = g) * 5).to(BF16)
    p0 = p.clone()
    s = torch.tensor([0.37], device = 'cuda')
    ops.scale_bf16(p, s, n)
    assert same_bits(p[:n], (p0[:n].float() * s).to(BF16)) and same_bits(p[n:], p0[n:])
    n4 = (4 << 20) + 4
    y = torch.randn(n4 + 4, device = 'cuda', generator = g) * 10
    xx = torch.randn(n4 + 4, device = 'cuda', generator = g)
    y0, a = y.clone(), -0.3
    ops.axpy_f32(y, xx, a, n4)
    a32 = float(np.float32(a))
    ref = y0[:n4].double() + a32 * xx[:n4].double()
    # one rounding if the compiler fuses the multiply-add, two if it does not
    assert_close64(y[:n4], ref, ref.abs() + (a32 * xx[:n4].double()).abs(), rel = 2 * U32, what = 'axpy')
    assert same_bits(y[n4:], y0[n4:])
    with pytest.raises(_lib.TfxError):
        ops.axpy_f32(y, xx, a, n4 - 2)            # n must be a multiple of 4: rejected before any launch
    assert same_bits(y[n4:], y0[n4:])


# ------------------------------------------------------------------------------------------------ fused Adam / AdamW
def torch_adam_step(p, m, v, grad, step, lr, betas, eps, wd, decoupled):
    """one float64 step of torch.optim.Adam / AdamW from the given state (copies): returns (param, exp_avg, exp_avg_sq)"""
    P = torch.nn.Parameter(p.double().clone())
    cls = torch.optim.AdamW if decoupled else torch.optim.Adam
    opt = cls([P], lr = lr, betas = betas, eps = eps, weight_decay = wd, foreach = False)
    opt.state[P] = dict(step = torch.tensor(float(step - 1)), exp_avg = m.double().clone(), exp_avg_sq = v.double().clone())
    P.grad = grad.double().clone()
    opt.step()
    st = opt.state[P]
    assert float(st['step']) == step
    return P.detach(), st['exp_avg'], st['exp_avg_sq']


def f32(x):
    return float(np.float32(x))


def check_adam(p_new, m_new, v_new, p, m, v, g_scaled, step, lr, betas, eps, wd, decoupled, what):
    """the kernel's step from state (p, m, v) against torch's float64 step from the same fp32 state and the same (fp32) hyper-parameters.
    Bounds: a few fp32 roundings of the terms of each update, plus the fp32 bias corrections: 1 - powf(beta, step) loses
    ~beta^step / (1 - beta^step) ulps to cancellation.  The update of p is compared relative to its own size, so a bias correction evaluated
    at step - 1 (0.14 % at step 300 for beta2 = 0.999, 0.05 % for beta1 = 0.99; infinite at step 1) fails."""
    rp, rm, rv = torch_adam_step(p, m, v, g_scaled, step, lr, betas, eps, wd, decoupled)
    b1, b2 = betas
    gd = g_scaled.double().abs() + (0 if decoupled else wd * p.double().abs())
    m_scale = b1 * m.double().abs() + (1 - b1) * gd
    assert_close64(m_new, rm, m_scale, rel = 1e-6, what = f'{what}: exp_avg')
    assert_close64(v_new, rv, b2 * v.double() + (1 - b2) * gd * gd, rel = 1e-6, what = f'{what}: exp_avg_sq')
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    rel_bc = 2 * U32 * (b1 ** step / bc1 + b2 ** step / bc2)
    upd = lr / bc1 * m_scale / (rv.sqrt() / math.sqrt(bc2) + eps)
    assert_close64(p_new, rp, 4 * U32 * rp.abs() + (1e-6 + rel_bc) * upd, rel = 1.0, what = f'{what}: param')


@pytest.mark.parametrize('decoupled', [0, 1])
def test_adam_step_host(ops, decoupled):
    n = (4 << 20) + 13
    lr, betas, eps, wd, gs = f32(1e-3), (f32(0.9), f32(0.999)), f32(1e-8), f32(0.1), 0.25
    g = gen(15 + decoupled)
    p = torch.randn(n, device = 'cuda', generator = g) * 0.02
    m = torch.zeros(n, device = 'cuda'); v = torch.zeros(n, device = 'cuda')
    for step in (1, 2, 3):
        grad = torch.randn(n, device = 'cuda', generator = g)
        g_used = grad * gs                         # grad_scale is applied before the decay term (exact: a power of two)
        p0, m0, v0 = p.clone(), m.clone(), v.clone()
        ops.adam_step(p, grad, m, v, n, lr, betas[0], betas[1], eps, wd, decoupled, step, gs, 1, None)
        assert not grad.any(), 'zero_grads = 1 must leave the gradients exactly zero'
        check_adam(p, m, v, p0, m0, v0, g_used, step, lr, betas, eps, wd, decoupled, f'host step {step}')
    grad = torch.randn(n, device = 'cuda', generator = g); g0 = grad.clone()
    ops.adam_step(p, grad, m, v, n, lr, betas[0], betas[1], eps, wd, decoupled, 4, 1.0, 0, None)
    assert same_bits(grad, g0), 'zero_grads = 0 must not touch the gradients'


@pytest.mark.parametrize('decoupled', [0, 1])
def test_adam_step_device_counter_graph(ops, decoupled):
    """the production path (DataParallelTrainer: device step counter, zero_grads, grad_scale = 1 / world, captured in the step graph):
    one launch captured once, replayed 300 times; every step is checked against torch's from the kernel's previous state"""
    n = (1 << 20) + 7
    lr, betas, eps, wd, gs = f32(1e-3), (f32(0.99), f32(0.999)), f32(1e-8), f32(0.05), 0.25
    g = gen(17 + decoupled)
    p = torch.randn(n, device = 'cuda', generator = g) * 0.02
    m = torch.zeros(n, device = 'cuda'); v = torch.zeros(n, device = 'cuda'); grad = torch.zeros(n, device = 'cuda')
    counter = torch.zeros(1, device = 'cuda', dtype = I32)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.adam_step(p, grad, m, v, n, lr, betas[0], betas[1], eps, wd, decoupled, 12345, gs, 1, counter)     # host step: ignored
    torch.cuda.synchronize()
    assert int(counter.item()) == 0, 'capture must not run the step'
    for step in range(1, 301):
        grad.copy_(torch.randn(n, device = 'cuda', generator = g))
        g_used = grad * gs
        p0, m0, v0 = p.clone(), m.clone(), v.clone()
        graph.replay()
        assert not grad.any()
        check_adam(p, m, v, p0, m0, v0, g_used, step, lr, betas, eps, wd, decoupled, f'graph step {step}')
    assert int(counter.item()) == 300


# ------------------------------------------------------------------------------------------------ global-norm clipping
def test_grad_sumsq_clip_by_norm(ops):
    n, n2 = 50_000_003, (4 << 20) + 1
    g = gen(19)
    a = torch.randn(n, device = 'cuda', generator = g)
    b = torch.randn(n2, device = 'cuda', generator = g) * 3
    sq_a = (a.double() ** 2).sum().item()
    sq_b = (b.double() ** 2).sum().item()
    acc = torch.zeros(1, device = 'cuda', dtype = F64)
    ops.grad_sumsq(a, n, acc)
    # per-thread partials in double, per-block sums in fp32, blocks added in double: the norm to ~1e-6
    assert abs(math.sqrt(acc.item()) - math.sqrt(sq_a)) <= 1e-6 * math.sqrt(sq_a)
    ops.grad_sumsq(b, n2, acc)                    # accumulates into the same scalar
    assert abs(math.sqrt(acc.item()) - math.sqrt(sq_a + sq_b)) <= 1e-6 * math.sqrt(sq_a + sq_b)
    acc_a = torch.tensor([sq_a], device = 'cuda', dtype = F64)
    for pre in (1.0, 1 / 8):                      # pre_scale = 1 / world when the buffer holds the all-reduced sum
        max_norm = 0.5 * pre * math.sqrt(sq_a)
        # torch.nn.utils.clip_grad_norm_ on the averaged gradient pre * a, in float64
        holder = torch.zeros(n, dtype = F64, device = 'cuda').requires_grad_(True)
        holder.grad = a.double() * pre
        torch.nn.utils.clip_grad_norm_([holder], max_norm)
        want = holder.grad / pre
        got = a.clone()
        ops.clip_by_norm(got, n, acc_a, max_norm, pre)
        # the coefficient is an fp32 value (~3 roundings), then one multiply per element
        assert_close64(got, want, want.abs(), rel = 1e-6, what = f'clip pre_scale={pre}')
        del holder, want
    got = a.clone()
    ops.clip_by_norm(got, n, acc_a, 10 * math.sqrt(sq_a), 1.0)
    assert same_bits(got, a), 'a norm below max_norm must leave the gradients bit for bit'
    for bad in (0.0, -1.0):
        with pytest.raises(_lib.TfxError):
            ops.clip_by_norm(got, n, acc_a, bad, 1.0)


# ------------------------------------------------------------------------------------------------ EMA
@pytest.mark.parametrize('decay', [0.999, 0.9, 0.0])
def test_ema_update(ops, decay):
    n = (4 << 20) + 5
    g = gen(20)
    ema = torch.randn(n, device = 'cuda', generator = g)
    p = torch.randn(n, device = 'cuda', generator = g)
    half = n // 2
    ema[:half] *= 1e-3; p[:half] *= 1e3           # |p| >> |ema| in the first half, |ema| >> |p| in the second
    ema[half:] *= 1e3; p[half:] *= 1e-3
    e0 = ema.clone()
    ops.ema_update(ema, p, n, decay)
    if decay == 0.0:
        assert same_bits(ema, p)
        return
    d = float(np.float32(decay))
    ref = d * e0.double() + (1 - d) * p.double()
    # within one fp32 ulp of the larger operand
    assert_close64(ema, ref, torch.maximum(e0.abs(), p.abs()).double(), rel = 2.0 ** -23, what = f'ema decay={decay}')


# ------------------------------------------------------------------------------------------------ token assemble / flow-head rows
@pytest.mark.parametrize('D', DISPATCH_D)
def test_embed_scatter_clean_flow(ops, D):
    M, S, V, n_cond = 12000, 9000, 300, 37        # 9000 > 8448 warps of the capped grid: every warp walks two rows
    eps = 1e-2
    g = gen(21 + D)
    emb = torch.randn(V, D, device = 'cuda', generator = g)
    modtok = torch.randn(S, D, device = 'cuda', generator = g)
    text_id = torch.randint(-3, V, (M,), device = 'cuda', generator = g, dtype = I32)           # negative ids read row 0
    slot = torch.full((M,), -1, device = 'cuda', dtype = I32)
    rows = torch.randperm(M, device = 'cuda', generator = g)[:S]
    slot[rows] = torch.arange(S, device = 'cuda', dtype = I32)
    # ---- embed_assemble: a pure copy (+ its bf16 cast)
    want = emb[text_id.clamp(min = 0).long()]
    want_m = want.clone(); want_m[rows] = modtok
    for sl, w in ((slot, want_m), (None, want)):
        for with_bf16 in (True, False):
            x0 = torch.full((M + 1, D), 5., device = 'cuda'); xb = torch.full((M + 1, D), -7., device = 'cuda', dtype = BF16)
            ops.embed_assemble(text_id, emb, modtok, sl, x0, xb if with_bf16 else None, M, D)
            assert same_bits(x0[:M], w) and (x0[M] == 5.).all()
            if with_bf16:
                assert same_bits(xb[:M], w.to(BF16)) and (xb[M].float() == -7.).all()
            else:
                assert (xb.float() == -7.).all()
    # ---- scatter_add_rows: dst[row_map[s]] += src[s], -1 rows skipped
    row_map = rows.to(I32).clone()
    row_map[torch.rand(S, device = 'cuda', generator = g) < 0.1] = -1
    dst = torch.randn(M + 1, D, device = 'cuda', generator = g); d0 = dst.clone()
    src = torch.randn(S, D, device = 'cuda', generator = g)
    ops.scatter_add_rows(dst, src, row_map, S, D)
    want = d0.clone()
    keep = row_map >= 0
    want[row_map[keep].long()] += src[keep]       # one fp32 add per element: bit exact
    assert same_bits(dst, want)
    # ---- clean_flow fwd / bwd: t = cond_times[cond_row[row_token[s]]], 1 / max(1 - t, eps)
    cond_times = torch.rand(n_cond, device = 'cuda', generator = g)
    cond_times[:4] = torch.tensor([1.0, 0.9995, 0.995, 0.0], device = 'cuda')                 # eps clamp active for the first three
    cond_times = cond_times[torch.randperm(n_cond, device = 'cuda', generator = g)]
    cond_row = torch.randint(0, n_cond, (M,), device = 'cuda', generator = g, dtype = I32)
    row_token = rows.to(I32).clone()
    row_token[torch.rand(S, device = 'cuda', generator = g) < 0.1] = -1
    out = torch.randn(M, D, device = 'cuda', generator = g)
    omod = torch.full((S + 1, D), -7., device = 'cuda', dtype = BF16)
    ops.clean_flow_fwd(out, row_token, modtok, cond_times, cond_row, eps, omod, S, D)
    ok = row_token >= 0
    tok = row_token[ok].long()
    t = cond_times[cond_row[tok].long()].double()
    inv = 1 / torch.clamp(1 - t, min = float(np.float32(eps)))
    assert (inv > 99).any(), 'the eps clamp is not exercised'
    diff = out[tok].double() - modtok[ok].double()
    ref = diff * inv[:, None]
    # (a - b), 1 - t, 1 / x, * inv: four fp32 roundings
    assert_bf16_close(omod[:S][ok], ref, slack = 4 * U32 * ref.abs(), what = f'clean_flow_fwd D={D}')
    assert not omod[:S][~ok].float().any() and (omod[S].float() == -7.).all()
    dmod = torch.randn(S + 1, D, device = 'cuda', generator = g); dm0 = dmod.clone()
    dneg = torch.full((S + 1, D), 5., device = 'cuda')
    ops.clean_flow_bwd(dmod, dneg, row_token, cond_times, cond_row, eps, S, D)
    ref = dm0[:S][ok].double() * inv[:, None]
    assert_close64(dmod[:S][ok], ref, ref.abs(), rel = 3 * U32, what = f'clean_flow_bwd D={D}')
    assert torch.equal(dneg[:S], -dmod[:S])
    assert not dmod[:S][~ok].any() and not dneg[:S][~ok].any(), 'skipped rows get a zero gradient'
    assert same_bits(dmod[S], dm0[S]) and (dneg[S] == 5.).all()


# ------------------------------------------------------------------------------------------------ RoPE table
def test_rope_table(ops):
    max_pos, nf = 8192, 32                        # well past the positions the sampler reaches for the bench config (max_length 512)
    freqs = 1. / (10000 ** (torch.arange(0, 64, 2)[:32].float() / 64))          # the model's RoPE frequencies (fp32)
    freqs = freqs.cuda()
    cs = torch.full((max_pos + 1, nf, 2), 5., device = 'cuda'); cst = torch.full((nf, max_pos, 2), 5., device = 'cuda')
    ops.rope_table(freqs, cs, cst, max_pos, nf)
    # rotary_embedding_torch forms the angle in fp32: fp32(p) * freqs[f]; cos / sin of that fp32 angle in float64
    ang = torch.arange(max_pos, device = 'cuda').float()[:, None] * freqs[None, :]
    ref = torch.stack((torch.cos(ang.double()), torch.sin(ang.double())), dim = -1)
    err = (cs[:max_pos].double() - ref).abs().max().item()
    assert err <= 2.5e-7, err                     # cosf / sinf: <= 2 ulp of a value <= 1
    assert (cs[max_pos] == 5.).all()
    assert same_bits(cst, cs[:max_pos].transpose(0, 1).contiguous())
