"""GPU: tfx_gemm_store, the plain GEMM behind every dgrad and wgrad product of a train step, against float64.

    out_f32 (+)= alpha A B^T + bias   (rows at m ld_f32, or at row_off[m] with -1 = skip; accumulate: fp32 atomics, split-K over k_splits)
    out_bf16    = bf16(alpha A B^T + bias)

Two tests:
  - the replay: every distinct gemm_store call of one eager forward + backward of seven models (d128 with two modality types and one
    condition row, a d512 config-2-like model over 4096 tokens, a text-only d128 model, a Self-Flow model, the d1536 (8 heads of 64) and
    d2048 (16 heads of 128) models of the wide training-step fixtures, a d384 model with 3 heads of 128 and the learned value residual),
    recorded on the engine's Ops instance and replayed with fresh operands of the same geometry, pitches, output alignment (address mod 16),
    row offsets, alpha, accumulate and split-K.  The test asserts that the recorded set still holds the edge cases below, so it cannot lose
    them silently when the engine changes: K < 64, N < 32, M <= 2, K <= 2 with both operands MN-major, odd N through row_off, a row offset
    that is not a multiple of 4, k_splits > 1, a bf16-only output, a dgrad (A K-major, B MN-major, no split) over more than 128 k-blocks
    (du = dvg W1 at d2048: 172), a wgrad with more than 8192 output rows through row_off with -1 rows (W1 at d2048: 11008 rows, 86 of them
    pad), and one -1 row between mapped rows (the QKVG wgrad at an odd head count, whose value-residual mix rows start at an even row).
  - explicit edges the ABI allows, under every schedule a launch can take (ping-pong single CTA, ping-pong 2-CTA clusters, the 256 x 128
    wide tile): K in {1, 8, 63, 64, 65, 390}, M in {1, 2, 127, 129, 257, 300, 40000} (40000: several tiles per CTA, an odd tile count),
    N in {1, 31, 33, 390, 1365}, all four operand majors; each case stores fp32 + bf16 with alpha and bias (bf16 pitch not a multiple of
    8: the scalar bf16 path), a staged bf16-only output, an accumulate with alpha and bias into a non-zero fp32 output at an unaligned
    address, a split-K accumulate and a plain store through row_off (offsets 0, -1 and not multiples of 4).

Operands: every operand is stored at its real pitch and the columns between its logical extent (K for K-major, M or N for MN-major) and the
pitch hold NaN.  The tensor maps are built with the logical extent, so a read of padding shows up as NaN in the output.

Reference and bound (|got - ref| <= bound element-wise, worst err / bound printed with -s):
  ref = alpha (A @ B^T) + bias (+ the initial value when accumulating), in float64 from the same bf16 operands; mag = |alpha| |A| @ |B|^T.
  bound = C_ACC(kb) mag + (s + 2) 2^-24 (mag + |bias| + |initial|)   (the fp32 accumulator over kb k-blocks per work item, then the alpha
          product, the bias add and one atomic add per split), plus 2^-8 |ref| for bf16 outputs.
  Bytes a call must not write (a guard row past M, the columns between N and the pitch, the flat-buffer entries no row offset reaches, a
  tail past the last row) hold a sentinel - or the initial value when accumulating - and are compared bit for bit."""
import pytest
import torch

from helpers import SENT, Checks as _Checks, c_acc, gen, load_golden, show_c_acc
from test_selfflow_cpu import selfflow_noise, selfflow_wrapper
from transfusion_pytorch_b200 import Transfusion, _lib, synth

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
U8, U24 = 2.0 ** -8, 2.0 ** -24
# fp32 accumulation of the wgmma main loop: c_acc(kb) of helpers.py, C_ACC0 = 1.6e-6 of |A| |B|^T up to 43 k-blocks, growing with
# sqrt(kb / 43) above that.  Measured here on an H100 80GB HBM3 (700 W power limit): at most 1.4e-6 of |A| |B|^T (kb = 384, K = 24576: the
# conditioning dgrad of the d2048 model), 0.29 of C_ACC(kb) over every call of the file.
# Measured worst err / bound (same run): bf16 outputs 0.98 - 0.996 (the cast's rounding, which the bound states exactly); fp32 outputs of
# the replay <= 0.33 (the K = 1 wgrads through row_off), of the explicit edges <= 0.43.  Recording the seven models takes 15 s, the replay
# 1.3 s.
# The float64 reference and checks of one call run over row chunks of at most REF_VALUES outputs (a dozen [rows, N] float64 / int64 arrays
# each): every explicit edge and every call of the d512 and smaller models is one chunk; the largest product, the d2048 model's
# conditioning-table wgrad (24576 x 8192 outputs), takes 12.  Measured on the same H100: whole, its checks peaked at 20.3 GiB of device
# memory; in chunks the replay's checks peak at 4.6 GiB, over the 5.8 GiB that recording the seven models leaves allocated.
REF_VALUES = 1 << 24

SHOWN = {}


@pytest.fixture(scope = 'module')
def ops():
    return _lib.Ops()


@pytest.fixture(scope = 'module', autouse = True)
def _report():
    yield
    for name, r in sorted(SHOWN.items()):
        print(f'worst over the file: {name:40s} {r:.3g}')


def Checks(what):
    return _Checks(what, SHOWN)


def pad(x, m):
    return (x + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ one checked call
def operand(rows, cols, pitch, g):
    """bf16 [rows, pitch]: the logical [rows, cols] random, the padding columns NaN"""
    t = torch.full((rows, pitch), float('nan'), dtype = BF16, device = 'cuda')
    t[:, :cols] = torch.randn(rows, cols, device = 'cuda', generator = g).to(BF16)
    return t


def logical(t, mn_major, ext, K):
    """[ext, K] float64 of a stored operand (MN-major: stored [K][pitch])"""
    return t[:K, :ext].double().t() if mn_major else t[:ext, :K].double()


class Out:
    """an output matrix inside a flat buffer: `pre` elements put its address at `align` mod 16; rows at m ld or at row_off[m]; the buffer
    holds `init` (a sentinel, or random initial values to accumulate into) everywhere, including a guard row / tail no row may reach"""

    def __init__(self, M, N, ld, dtype, align, row_off, init, g):
        esz = torch.finfo(dtype).bits // 8
        assert align % esz == 0
        self.pre, self.N = align // esz, N
        self.offs = row_off.long() if row_off is not None else torch.arange(M, device = 'cuda') * ld
        self.valid = self.offs >= 0
        end = int(self.offs[self.valid].max()) + N if bool(self.valid.any()) else 0
        if row_off is None:
            end = max(end, (M + 1) * ld)
        size = self.pre + end + 37
        if init == 'sentinel':
            self.flat = torch.full((size,), SENT, dtype = dtype, device = 'cuda')
        else:
            self.flat = torch.randn(size, device = 'cuda', generator = g).to(dtype)
        assert self.flat.data_ptr() % 16 == 0
        self.flat0 = self.flat.clone()
        self.ptr = self.flat[self.pre:]
        self.written = torch.zeros_like(self.flat, dtype = torch.bool)

    def idx(self, rows):
        """flat indices of the stored rows among `rows` (a slice of the M output rows)"""
        offs = self.offs[rows]
        return self.pre + offs[offs >= 0][:, None] + torch.arange(self.N, device = 'cuda')[None]

    def got(self, rows):
        i = self.idx(rows)
        self.written[i.reshape(-1)] = True
        return self.flat[i]

    def initial(self, rows):
        return self.flat0[self.idx(rows)].double()

    def rest_untouched(self):
        """every entry no got() call covered still holds its initial bytes"""
        view = {BF16: torch.int16, F32: torch.int32}[self.flat.dtype]
        return not bool(((self.flat.view(view) != self.flat0.view(view)) & ~self.written).any())


def run_gemm(ops, ck, tag, c, g):
    """one tfx_gemm_store call described by c (the recorded / explicit geometry) on fresh operands, checked against float64 in row chunks
    of at most REF_VALUES outputs"""
    M, N, K, a_mn, b_mn, lda, ldb = c['M'], c['N'], c['K'], c['a_mn'], c['b_mn'], c['lda'], c['ldb']
    alpha, acc, ks, row_off = c['alpha'], c['acc'], c['ks'], c['row_off']
    A = operand(K if a_mn else M, M if a_mn else K, lda, g)
    B = operand(K if b_mn else N, N if b_mn else K, ldb, g)
    a64, b64 = logical(A, a_mn, M, K), logical(B, b_mn, N, K)
    bias = torch.randn(N, device = 'cuda', generator = g) * 0.5 if c['bias'] else None
    init = 'random' if acc else 'sentinel'
    of = Out(M, N, c['ld_f32'], F32, c['align_f32'], row_off, init, g) if c['f32'] else None
    ob = Out(M, N, c['ld_bf16'], BF16, c['align_bf16'], None, 'sentinel', g) if c['bf16'] else None
    ops.gemm_store(A, lda, a_mn, B, ldb, b_mn, M, N, K, of.ptr if of else None, c['ld_f32'], ob.ptr if ob else None, c['ld_bf16'], bias, row_off,
                   alpha, acc, ks)
    _, kb, _, s = _lib.gemm_store_items(M, N, K, a_mn, b_mn, ks)
    step = max(1, REF_VALUES // max(N, 1))
    for r0 in range(0, M, step):
        rs = slice(r0, min(r0 + step, M))
        a = a64[rs]
        mag = abs(alpha) * (a.abs() @ b64.abs().t())
        ref = alpha * (a @ b64.t())
        extra = mag
        if bias is not None:
            ref = ref + bias.double()
            extra = mag + bias.double().abs()
        E = c_acc(kb) * mag + (s + 2) * U24 * extra
        if of is not None:
            v = of.valid[rs]
            want, Ef = ref[v], E[v]
            if acc:
                init = of.initial(rs)
                want, Ef = want + init, Ef + (s + 2) * U24 * init.abs()
            got = of.got(rs)
            ck(f'{tag} fp32', got, want, Ef, row0 = int(of.valid[:r0].sum()))    # rows counted among the stored ones
            rest = (got.double() - want).abs() - (Ef - c_acc(kb) * mag[v])
            measured = (rest.clamp_min(0) / mag[v].clamp_min(1e-300)).max().item() if got.numel() else 0.
            SHOWN['c_acc (measured) / C_ACC(kb)'] = max(SHOWN.get('c_acc (measured) / C_ACC(kb)', 0.), measured / c_acc(kb))
            show_c_acc(SHOWN, kb, measured)
        if ob is not None:
            ck(f'{tag} bf16', ob.got(rs), ref, U8 * ref.abs() + (1 + U8) * E, row0 = r0)
    if of is not None:
        ck.true(f'{tag} fp32: bytes no row reaches untouched', of.rest_untouched())
    if ob is not None:
        ck.true(f'{tag} bf16: bytes no row reaches untouched', ob.rest_untouched())


def call(M, N, K, a_mn, b_mn, lda, ldb, f32 = None, bf16 = None, bias = False, row_off = None, alpha = 1.0, acc = 0, ks = 1):
    """f32 / bf16: (pitch, address mod 16) of the output"""
    return dict(M = M, N = N, K = K, a_mn = a_mn, b_mn = b_mn, lda = lda, ldb = ldb, f32 = f32 is not None, ld_f32 = f32[0] if f32 else 0,
                align_f32 = f32[1] if f32 else 0, bf16 = bf16 is not None, ld_bf16 = bf16[0] if bf16 else 0, align_bf16 = bf16[1] if bf16 else 0,
                bias = bias, row_off = row_off, alpha = alpha, acc = acc, ks = ks)


# ================================================================================================ replay of the engine's calls
def _record(calls, label, model, run):
    o = model.engine.ops
    orig = o.gemm_store

    def rec(A, lda, a_mn, B, ldb, b_mn, M, N, K, of, ld_f32, ob, ld_bf16, bias, row_off, alpha, acc, ks):
        ro = row_off.clone() if row_off is not None else None
        c = call(M, N, K, a_mn, b_mn, lda, ldb, (ld_f32, of.data_ptr() % 16) if of is not None else None,
                 (ld_bf16, ob.data_ptr() % 16) if ob is not None else None, bias is not None, ro, alpha, acc, ks)
        key = tuple(v for k, v in sorted(c.items()) if k != 'row_off') + ((ro.cpu().numpy().tobytes(),) if ro is not None else ())
        calls.setdefault(key, dict(c, where = label))
        orig(A, lda, a_mn, B, ldb, b_mn, M, N, K, of, ld_f32, ob, ld_bf16, bias, row_off, alpha, acc, ks)

    o.gemm_store = rec
    try:
        run()
    finally:
        o.gemm_store = orig


@pytest.fixture(scope = 'module')
def recorded():
    """every distinct gemm_store call of one eager forward + backward of seven models"""
    calls = {}
    # (a) d128, two modality types (dim_latent 32, 16), one modality instance: n_cond = 1
    torch.manual_seed(0)
    m = Transfusion(num_text_tokens = 64, dim_latent = (32, 16), modality_default_shape = ((4,), (2,)), prob_uncond = 0.,
                    transformer = dict(dim = 128, depth = 2, heads = 2))
    synth.fill_parameters_(m, seed = 3)
    m = m.cuda().eval()
    g = torch.Generator().manual_seed(1)
    batch = [[torch.randint(0, 64, (5,), generator = g), (1, torch.randn(9, 16, generator = g)), torch.randint(0, 64, (4,), generator = g)],
             [torch.randint(0, 64, (12,), generator = g)]]
    _record(calls, 'd128 n_cond=1', m, lambda: m(batch, times = torch.tensor([[0.3], [0.]])).backward())
    # (b) d512 config-2-like, 4096 tokens, 8 condition rows
    torch.manual_seed(0)
    m = Transfusion(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,), prob_uncond = 0., transformer = dict(dim = 512, depth = 2))
    synth.fill_parameters_(m, seed = 4)
    m = m.cuda().eval()
    _record(calls, 'd512 config2', m, lambda: m(synth.config2_batch(4, seed = 5), times = synth.config2_times(4, seed = 5)).backward())
    # (c) text-only d128: n_cond = 0
    torch.manual_seed(0)
    m = Transfusion(num_text_tokens = 256, transformer = dict(dim = 128, depth = 2))
    synth.fill_parameters_(m, seed = 6)
    m = m.cuda().eval()
    _record(calls, 'd128 text-only', m, lambda: m(synth.text_batch(2, 65, seed = 3)).backward())
    # (d) Self-Flow: the representation head's GEMMs
    fx = load_golden('small_selfflow')
    w = selfflow_wrapper(fx, 'cuda')

    def selfflow():
        total, _ = w(synth.dropout_batch(), times = fx['times'], noise = selfflow_noise(fx, 0), teacher_noise = selfflow_noise(fx, 1),
                     dropout_key = fx['dropout_key'])
        total.backward()
    _record(calls, 'self-flow', w.student, selfflow)
    # (e) d1536 with 8 heads of 64 and (f) d2048 with 16 heads of 128, the models of the wide training-step fixtures, on their two-modality
    # batch: the dgrad du = dvg W1 over K = 2 Ip = 8192 / 11008, the W1 wgrad with 8192 / 11008 output rows through row_off
    two_type_batch = lambda: synth.config4_batch(2, seed = 2, total_len = 300, dims = (32, 16), text_vocab = 64)
    for name in ('small_wide1536', 'small_wide2048'):
        fx = load_golden(name)
        torch.manual_seed(0)
        m = Transfusion(**fx['ctor'])
        synth.fill_parameters_(m, seed = fx['seed'])
        m = m.cuda().eval()
        _record(calls, name[6:], m, lambda: m(two_type_batch(), times = fx['times']).backward())
    # (g) dim_head 128, an odd head count and the learned value residual: the QKVG wgrad maps the mix rows at 3 HI + 4 (one pad row behind
    # the 3 gate rows)
    torch.manual_seed(0)
    m = Transfusion(num_text_tokens = 64, dim_latent = 32, modality_default_shape = (4,), prob_uncond = 0.,
                    transformer = dict(dim = 384, depth = 3, heads = 3, dim_head = 128, use_value_residual = True))
    synth.fill_parameters_(m, seed = 8)
    m = m.cuda().eval()
    batch = synth.small_batch(3, seed = 1, dim_latent = 32, text_vocab = 64)
    times = torch.rand(3, 3, generator = torch.Generator().manual_seed(5))             # up to 3 modality instances per sample
    _record(calls, 'd384 h3x128 vres', m, lambda: m(batch, times = times).backward())
    torch.cuda.synchronize()
    return list(calls.values())


def test_recorded_calls_keep_their_edge_cases(recorded):
    def has(pred):
        return sorted({c['where'] for c in recorded if pred(c)})
    splits = lambda c: _lib.gemm_store_items(c['M'], c['N'], c['K'], c['a_mn'], c['b_mn'], c['ks'])[3]
    kblocks = lambda c: _lib.gemm_store_items(c['M'], c['N'], c['K'], c['a_mn'], c['b_mn'], c['ks'])[1]

    def lone_gap(r):
        on = r >= 0
        return bool((on[:-2] & ~on[1:-1] & on[2:]).any())
    want = {
        'K < 64': has(lambda c: c['K'] < 64),
        'N < 32': has(lambda c: c['N'] < 32),
        'M <= 2': has(lambda c: c['M'] <= 2),
        'K <= 2, both operands MN-major': has(lambda c: c['K'] <= 2 and c['a_mn'] and c['b_mn']),
        'odd N through row_off': has(lambda c: c['N'] % 2 and c['row_off'] is not None),
        'a row offset not a multiple of 4': has(lambda c: c['row_off'] is not None and bool(((c['row_off'] >= 0) & (c['row_off'] % 4 != 0)).any())),
        'k_splits > 1': has(lambda c: splits(c) > 1),
        'bf16-only output': has(lambda c: c['bf16'] and not c['f32']),
        'a dgrad (A K-major, B MN-major, no split) over more than 128 k-blocks and 256 token rows':
            has(lambda c: not c['a_mn'] and c['b_mn'] and splits(c) == 1 and kblocks(c) > 128 and c['M'] >= 256),
        'a wgrad with more than 8192 output rows through row_off, with -1 rows':
            has(lambda c: c['row_off'] is not None and c['M'] > 8192 and bool((c['row_off'] == -1).any())),
        'one -1 row between mapped rows (the mix rows behind an odd head count)': has(lambda c: c['row_off'] is not None and lone_gap(c['row_off'])),
    }
    for k, v in want.items():
        print(f'{k}: {", ".join(v)}')
    missing = [k for k, v in want.items() if not v]
    assert not missing, f'the recorded train steps no longer contain: {missing}'


def test_replay_engine_calls_vs_float64(ops, recorded):
    ck = Checks('replay')
    g = gen(5)
    for i, c in enumerate(recorded):
        print(f"replay {c['where']} #{i}: M={c['M']} N={c['N']} K={c['K']} mn={c['a_mn']}{c['b_mn']} lda={c['lda']} ldb={c['ldb']} ks={c['ks']}"
              + (' row_off' if c['row_off'] is not None else '') + (' acc' if c['acc'] else ''))
        run_gemm(ops, ck, f"replay {c['where']}", c, g)
    print(f'replayed {len(recorded)} distinct calls')
    ck.done()


# ================================================================================================ explicit edges under every schedule
SCHEDULES = {'single': (1, 3), 'paired': (2, 3), 'wide': (1, 2)}           # (tfx_gemm_set_cluster_mode, tfx_gemm_set_wide_mode)
SHAPES = [(1, 1365, 390), (127, 31, 65), (129, 33, 63), (257, 1, 8), (2, 1365, 1), (129, 31, 64), (300, 390, 520), (40000, 33, 390)]
MAJORS = [(0, 0), (0, 1), (1, 1), (1, 0)]


@pytest.fixture(params = list(SCHEDULES), ids = list(SCHEDULES))
def schedule(ops, request):
    cm, wm = SCHEDULES[request.param]
    assert ops.lib.tfx_gemm_set_cluster_mode(cm) == 0 and ops.lib.tfx_gemm_set_wide_mode(wm) == 0
    yield request.param
    ops.lib.tfx_gemm_set_cluster_mode(1)
    ops.lib.tfx_gemm_set_wide_mode(1)


def row_offsets(M, N, g):
    """row m at perm[m] (N + 5): rows never overlap, row 0 at offset 0 exactly, row 1 skipped (-1), most offsets not multiples of 4"""
    perm = torch.randperm(M, device = 'cuda', generator = g)
    perm[(perm == 0).nonzero().squeeze(1)] = perm[0].clone()
    perm[0] = 0
    off = perm.long() * (N + 5)
    if M > 1:
        off[1] = -1
    return off


@pytest.mark.parametrize('a_mn,b_mn', MAJORS, ids = [f'mn{a}{b}' for a, b in MAJORS])
@pytest.mark.parametrize('M,N,K', SHAPES, ids = [f'M{m}N{n}K{k}' for m, n, k in SHAPES])
def test_gemm_store_edges_vs_float64(ops, schedule, M, N, K, a_mn, b_mn):
    ck = Checks(f'edges {schedule} M={M} N={N} K={K} mn={a_mn}{b_mn}')
    g = gen(M * 7 + N * 3 + K + 11 * a_mn + 13 * b_mn)
    lda = pad(M if a_mn else K, 8) + 8
    ldb = pad(N if b_mn else K, 8) + 8
    geo = dict(M = M, N = N, K = K, a_mn = a_mn, b_mn = b_mn, lda = lda, ldb = ldb)
    cases = [
        ('store fp32 + bf16 (scalar bf16 path), alpha, bias', call(**geo, f32 = (pad(N, 4) + 4, 0), bf16 = (pad(N, 8) + 3, 0), bias = True, alpha = 0.75)),
        ('store bf16 only (staged)', call(**geo, bf16 = (pad(N, 8) + 8, 0))),
        ('accumulate, alpha, bias, unaligned fp32', call(**geo, f32 = (N + 1, 4), bias = True, alpha = -1.5, acc = 1)),
        ('split-K 4 accumulate through row_off', call(**geo, f32 = (0, 0), row_off = row_offsets(M, N, g), acc = 1, ks = 4)),
        ('store through row_off, alpha, bias', call(**geo, f32 = (0, 0), row_off = row_offsets(M, N, g), bias = True, alpha = 0.5)),
    ]
    for name, c in cases:
        run_gemm(ops, ck, name, c, g)
    ck.done()
