"""CPU: `tools/bench_step.py` builds, for every arm, the model and batch the per-option step scripts it replaced built, and counts the
AttentionResidual and row-kernel bytes as they did (the old values are written out literally)."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location('bench_step', os.path.join(ROOT, 'tools', 'bench_step.py'))
bench_step = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(bench_step)

C2 = dict(num_text_tokens = 256, dim_latent = 384, modality_default_shape = (256,))
C4 = dict(num_text_tokens = 256, dim_latent = (384, 192), modality_default_shape = ((4,), (2,)))

# (arm, the constructor the old script built, batch kind, batch size); an old script's baseline arm is its run with the option at its default
OLD = [
    # bench_dh128_step.py
    ('512x8x128:dim_head=128', dict(C2, transformer = dict(dim = 512, depth = 8, heads = 4, dim_head = 128)), 'config2', 128),
    ('512x8x128', dict(C2, transformer = dict(dim = 512, depth = 8, heads = 8, dim_head = 64)), 'config2', 128),
    # bench_noqknorm_step.py
    ('512x8x128', dict(C2, transformer = dict(dim = 512, depth = 8, qk_rmsnorm = True)), 'config2', 128),
    ('512x8x128:qk_rmsnorm=0', dict(C2, transformer = dict(dim = 512, depth = 8, qk_rmsnorm = False)), 'config2', 128),
    # bench_dropout_step.py --dropout 0 / 0.1
    ('512x8x128', dict(C2, transformer = dict(dim = 512, depth = 8, ff_kwargs = dict(dropout = 0.))), 'config2', 128),
    ('512x8x128:dropout=0.1', dict(C2, transformer = dict(dim = 512, depth = 8, ff_kwargs = dict(dropout = 0.1))), 'config2', 128),
    # bench_recon_step.py --config 4 --weight 0 / 0.1
    ('512x8x128:data=config4', dict(C4, transformer = dict(dim = 512, depth = 8), reconstruction_loss_weight = 0.), 'config4', 128),
    ('512x8x128:data=config4,recon=0.1', dict(C4, transformer = dict(dim = 512, depth = 8), reconstruction_loss_weight = 0.1), 'config4', 128),
    # bench_depth.py
    ('512x8x64', dict(C2, transformer = dict(dim = 512, depth = 8, heads = 8)), 'config2', 64),
    ('512x16x64', dict(C2, transformer = dict(dim = 512, depth = 16, heads = 8)), 'config2', 64),
    ('768x12x32', dict(C2, transformer = dict(dim = 768, depth = 12, heads = 12)), 'config2', 32),
    ('1024x24x6', dict(C2, transformer = dict(dim = 1024, depth = 24, heads = 16)), 'config2', 6),
    ('1024x32x4', dict(C2, transformer = dict(dim = 1024, depth = 32, heads = 16)), 'config2', 4),
    # bench_wide_step.py (its model builder was bench_depth.py's)
    ('1536x16x4', dict(C2, transformer = dict(dim = 1536, depth = 16, heads = 24)), 'config2', 4),
    ('2048x8x2', dict(C2, transformer = dict(dim = 2048, depth = 8, heads = 32)), 'config2', 2),
]


def with_defaults(ctor):
    """the constructor with the defaults of the options an arm can set written out (`Transformer`: dim_head 64, heads 8, qk_rmsnorm True, no FFN
    dropout; `Transfusion`: no reconstruction loss), so that writing a default out and leaving it to the constructor compare equal"""
    tr = dict(dict(dim_head = 64, heads = 8, qk_rmsnorm = True, ff_kwargs = dict(dropout = 0.)), **ctor['transformer'])
    return dict(dict(reconstruction_loss_weight = 0.), **dict(ctor, transformer = tr))


@pytest.mark.parametrize('spec,ctor,data,batch', OLD, ids = [f'{i}-{o[0]}' for i, o in enumerate(OLD)])
def test_arm_builds_what_the_old_script_built(spec, ctor, data, batch):
    got, got_data, got_batch = bench_step.parse_arm(spec)
    assert (with_defaults(got), got_data, got_batch) == (with_defaults(ctor), data, batch)


def test_arm_writes_only_the_options_it_is_given():
    ctor, _, _ = bench_step.parse_arm('512x8x128:dim_head=128')
    assert ctor == dict(C2, transformer = dict(dim = 512, depth = 8, dim_head = 128, heads = 4))
    ctor, _, _ = bench_step.parse_arm('1536x16x4:heads=12,qk_rmsnorm=1,dropout=0.2,recon=0.5,data=config2')
    assert ctor == dict(C2, transformer = dict(dim = 1536, depth = 16, dim_head = 64, heads = 12, qk_rmsnorm = True, ff_kwargs = dict(dropout = 0.2)),
                        reconstruction_loss_weight = 0.5)


@pytest.mark.parametrize('spec', ['512x8x128:lr=1e-3', '512x8x128:depth=4', '512x8x128:qk_rmsnorm=2', '512x8x128:data=config3', '512x8',
                                  '512x8x128:heads'])
def test_bad_arm_is_an_error(spec):
    with pytest.raises(ValueError):
        bench_step.parse_arm(spec)


def test_row_bytes_match_the_old_counts():
    old = {512: (3080, 8200, 4096, 6144), 1024: (6152, 16392, 8192, 12288), 2048: (12296, 32776, 16384, 24576)}
    for D, want in old.items():
        assert tuple(bench_step.row_bytes(n, D) for n in ('adaln_fwd', 'adaln_bwd', 'resid_bwd', 'rmsnorm_bwd')) == want
        assert bench_step.row_bytes('rmsnorm_fwd', D) is None


def test_attention_residual_bytes_match_the_old_counts():
    # depth 10 -> 11 adds a second chunk to the x0 assembly; depth 32 runs up to four chunks per launch
    old = {(512, 8): (69664, 171904), (512, 10): (97320, 245072), (512, 11): (112684, 291420), (1024, 24): (811104, 2385024),
           (1024, 32): (1343616, 4090368), (2048, 8): (278560, 684928)}
    for (D, L), want in old.items():
        assert bench_step.ares_bytes_per_token(D, L) == want
    assert bench_step.step_bytes('attn_residual_fwd_h16', 512, 11, 1000, 11) == 112684 * 1000
    assert bench_step.step_bytes('attn_residual_bwd2', 512, 11, 1000, 12) == 291420 * 1000
    assert bench_step.step_bytes('adaln_bwd', 512, 11, 1000, 22) == 8200 * 1000 * 22
    assert bench_step.step_bytes('gemm_store', 512, 11, 1000, 100) is None
