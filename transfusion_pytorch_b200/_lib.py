"""ctypes binding of libtfx_b200.so (include/tfx_b200.h).  PyTorch is used only for device memory
(`tensor.data_ptr()`) and the current CUDA stream; no torch types cross the boundary.

The library is loaded lazily and LOUDLY: there is no CPU / eager fallback in the product path.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_void_p, c_int, c_longlong, c_ulonglong, c_float, c_char_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libtfx_b200.so')

_lib = None

VP, I, LL, F, ULL = c_void_p, c_int, c_longlong, c_float, c_ulonglong

# name -> argtypes, mirrors include/tfx_b200.h exactly (order matters)
SIGNATURES = {
    'tfx_init': [I],
    'tfx_gemm_set_cluster_mode': [I],
    'tfx_gemm_set_wide_mode': [I],
    'tfx_gemm_store_items': [I, I, I, I, I, I, VP],
    'tfx_gemm_store': [VP, LL, I, VP, LL, I, I, I, I, VP, LL, VP, LL, VP, VP, F, I, I, VP],
    'tfx_gemm_qkvg': [VP, LL, VP, LL, I, I, I, VP, VP, VP, VP, VP, VP, VP, VP, VP, I, VP, VP, VP],
    'tfx_gemm_qkvg_rope': [VP, LL, VP, LL, I, I, I, VP, VP, VP, VP, VP, VP, I, VP, VP, VP],
    'tfx_gemm_qkvg_d128': [VP, LL, VP, LL, I, I, I, VP, VP, VP, VP, VP, VP, VP, VP, VP, I, VP, VP, VP],
    'tfx_gemm_qkvg_rope_d128': [VP, LL, VP, LL, I, I, I, VP, VP, VP, VP, VP, VP, I, VP, VP, VP],
    'tfx_gemm_resid': [VP, LL, VP, LL, I, VP, LL, I, I, I, VP, VP, VP, VP, VP, VP, VP, LL, VP, VP],
    'tfx_gemm_geglu': [VP, LL, VP, LL, VP, I, I, I, VP, VP, VP],
    'tfx_gemm_geglu_drop': [VP, LL, VP, LL, VP, I, I, I, VP, VP, VP, F, I, VP],
    'tfx_attn_fwd': [VP, VP, VP, LL, LL, LL, VP, I, VP, VP, VP, VP, VP, I, VP, LL, VP, I, F, F, VP, VP],
    'tfx_attn_fwd_tc': [VP, VP, VP, LL, LL, LL, VP, I, VP, VP, VP, VP, VP, I, VP, LL, VP, I, I, F, F, VP, VP],
    'tfx_attn_fast_params': [VP, VP, I, F, F, VP, VP],
    'tfx_attn_bwd_prep': [VP, VP, VP, VP, VP, VP, VP, I, I, VP],
    'tfx_attn_bwd': [VP, VP, VP, VP, LL, LL, LL, LL, VP, VP, VP, VP, VP, VP, VP, I, VP, VP, VP, LL, I, I, F, F, VP, VP],
    'tfx_attn_bwd_tc': [VP, VP, VP, VP, LL, LL, LL, LL, VP, VP, VP, VP, VP, VP, VP, VP, I, VP, VP, VP, LL, I, I, F, F, VP, VP],
    'tfx_attn_fwd_d128': [VP, VP, VP, LL, LL, LL, VP, I, VP, VP, VP, VP, VP, I, VP, LL, VP, I, F, F, VP],
    'tfx_attn_bwd_prep_d128': [VP, VP, VP, VP, VP, VP, VP, I, I, VP],
    'tfx_attn_bwd_d128': [VP, VP, VP, VP, LL, LL, LL, LL, VP, VP, VP, VP, VP, VP, VP, I, VP, VP, VP, LL, I, I, F, F, VP],
    'tfx_qk_bwd_pack': [VP, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP, LL, VP, VP, I, I, VP],
    'tfx_qk_bwd_pack_rope': [VP, VP, VP, VP, VP, VP, VP, LL, I, I, VP],
    'tfx_qk_bwd_pack_d128': [VP, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP, LL, VP, VP, I, I, VP],
    'tfx_qk_bwd_pack_rope_d128': [VP, VP, VP, VP, VP, VP, VP, LL, I, I, VP],
    'tfx_adaln_fwd': [VP, VP, VP, LL, VP, VP, VP, I, I, VP],
    'tfx_adaln_bwd': [VP, VP, VP, VP, VP, LL, VP, VP, VP, LL, VP, I, I, VP],
    'tfx_resid_bwd': [VP, VP, VP, VP, LL, VP, VP, VP, LL, VP, VP, I, I, VP],
    'tfx_attn_residual_bwd2': [VP, I, I, VP, VP, VP, VP, I, VP, VP, VP, VP, VP, I, VP, VP, VP, I, I, VP],
    'tfx_attn_residual_fwd_h16': [VP, I, VP, VP, VP, VP, VP, I, I, VP],
    'tfx_rmsnorm_fwd': [VP, VP, VP, VP, VP, VP, I, I, VP],
    'tfx_rmsnorm_bwd': [VP, VP, VP, VP, VP, I, I, VP],
    'tfx_rep_cos_fwd_bwd': [VP, VP, I, VP, I, VP, VP, VP, VP, I, I, VP],
    'tfx_embed_assemble': [VP, VP, VP, VP, VP, VP, I, I, VP],
    'tfx_embed_bwd': [VP, VP, VP, VP, VP, I, I, VP],
    'tfx_scatter_add_rows': [VP, VP, VP, I, I, VP],
    'tfx_flow_noise': [VP, VP, VP, VP, LL, VP, VP, LL, I, VP],
    'tfx_time_features': [VP, VP, VP, I, I, I, VP],
    'tfx_table_op': [VP, LL, VP, LL, VP, LL, VP, LL, LL, I, I, VP],
    'tfx_geglu_bwd': [VP, VP, VP, LL, I, VP, VP, VP, VP],
    'tfx_geglu_bwd_drop': [VP, VP, VP, LL, I, VP, VP, VP, VP, F, I, VP],
    'tfx_ce_fwd_bwd': [VP, LL, VP, I, I, F, VP, LL, VP, VP, I, VP],
    'tfx_mse_fwd_bwd': [VP, LL, VP, VP, LL, F, VP, LL, I, VP],
    'tfx_mse_recon_fwd_bwd': [VP, LL, VP, VP, VP, I, VP, VP, VP, LL, F, F, VP, VP, VP, LL, I, VP],
    'tfx_colsum_bf16': [VP, LL, LL, I, VP, VP, VP],
    'tfx_colsum_f32': [VP, LL, LL, I, VP, VP, VP],
    'tfx_cast_pack_multi': [VP, VP, VP, I, VP],
    'tfx_cast_bf16': [VP, VP, LL, VP],
    'tfx_scale_bf16': [VP, VP, LL, VP],
    'tfx_axpy_f32': [VP, VP, F, LL, VP],
    'tfx_rope_table': [VP, VP, VP, I, I, VP],
    'tfx_grad_sumsq': [VP, LL, VP, VP],
    'tfx_clip_by_norm': [VP, LL, VP, F, F, VP],
    'tfx_ema_update': [VP, VP, LL, F, VP],
    'tfx_adam_step': [VP, VP, VP, VP, LL, F, F, F, F, F, I, I, F, I, VP, VP],
    'tfx_decode_prep': [VP, I, I, I, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP],
    'tfx_attn_decode': [VP, VP, VP, LL, LL, LL, VP, I, VP, VP, VP, VP, I, VP, LL, F, F, VP],
    'tfx_attn_decode_d128': [VP, VP, VP, LL, LL, LL, VP, I, VP, VP, VP, VP, I, VP, LL, F, F, VP],
    'tfx_sample_tokens': [VP, LL, VP, I, I, VP, I, VP, I, I, VP, I, I, F, F, ULL, VP, I, VP],
    'tfx_ode_pre': [VP, VP, VP, LL, I, VP, VP, VP, I, VP],
    'tfx_ode_post': [VP, VP, VP, VP, F, LL, VP, VP, VP],
    'tfx_counter_inc': [VP, VP],
    'tfx_clean_flow_fwd': [VP, VP, VP, VP, VP, F, VP, I, I, VP],
    'tfx_clean_flow_bwd': [VP, VP, VP, VP, VP, F, I, I, VP],
    'tfx_laser_v_fwd': [VP, LL, VP, VP, LL, I, I, F, VP],
    'tfx_laser_out_fwd': [VP, VP, VP, I, I, VP],
    'tfx_laser_bwd_prep': [VP, VP, VP, VP, VP, VP, VP, I, I, VP],
    'tfx_laser_v_bwd': [VP, LL, VP, LL, I, I, F, VP],
    'tfx_vmix_fwd': [VP, LL, VP, VP, LL, VP, VP, I, I, VP],
    'tfx_vmix_bwd': [VP, LL, VP, LL, VP, LL, VP, VP, VP, VP, LL, I, I, VP],
    'tfx_add_f32_into_bf16': [VP, LL, VP, LL, I, I, VP],
    'tfx_laser_out_fwd_d128': [VP, VP, VP, I, I, VP],
    'tfx_laser_bwd_prep_d128': [VP, VP, VP, VP, VP, VP, VP, I, I, VP],
    'tfx_vmix_fwd_d128': [VP, LL, VP, VP, LL, VP, VP, I, I, VP],
    'tfx_vmix_bwd_d128': [VP, LL, VP, LL, VP, LL, VP, VP, VP, VP, LL, I, I, VP],
}

EXPORTED = ['tfx_last_error', 'tfx_version', 'tfx_geglu_bwd_rows_per_block', 'tfx_attn_residual_bwd_workspace_floats', 'tfx_rep_cos_blocks'] + list(SIGNATURES)


class TfxError(RuntimeError):
    pass


def library_present() -> bool:
    return os.path.isfile(LIB_PATH)


def load():
    """Load libtfx_b200.so, declaring every prototype.  Raises if the extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not library_present():
        raise TfxError(
            f'{LIB_PATH} is missing: the sm_90a CUDA extension has not been built. '
            'Run `python -c "import __graft_entry__ as g; g.build()"` (or `make -C transfusion_pytorch_b200/csrc`). '
            'There is no CPU / eager fallback.')
    lib = ctypes.CDLL(LIB_PATH)
    lib.tfx_last_error.restype = c_char_p
    lib.tfx_last_error.argtypes = []
    lib.tfx_version.restype = c_int
    lib.tfx_version.argtypes = []
    lib.tfx_geglu_bwd_rows_per_block.restype = c_int
    lib.tfx_geglu_bwd_rows_per_block.argtypes = []
    lib.tfx_attn_residual_bwd_workspace_floats.restype = c_longlong
    lib.tfx_attn_residual_bwd_workspace_floats.argtypes = [c_int, c_int]
    lib.tfx_rep_cos_blocks.restype = c_int
    lib.tfx_rep_cos_blocks.argtypes = [c_int]
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = c_int
    _lib = lib
    return lib


def check(rc: int, name: str):
    if rc != 0:
        msg = _lib.tfx_last_error().decode(errors = 'replace') if _lib is not None else ''
        raise TfxError(f'{name} failed (code {rc}): {msg}')


def gemm_store_items(M: int, N: int, K: int, a_mn: int, b_mn: int, k_splits: int):
    """(work items, k-blocks per item, tile rows, split-K factor) of a `tfx_gemm_store` launch with these arguments; launches nothing"""
    lib = load()
    geo = (c_int * 4)()
    check(lib.tfx_gemm_store_items(M, N, K, a_mn, b_mn, k_splits, geo), 'tfx_gemm_store_items')
    return tuple(geo)


class Ops:
    """Thin callable facade: `ops.adaln_fwd(...)` -> `tfx_adaln_fwd(..., stream)` with error checking.
    Tensor arguments are converted with `.data_ptr()`; None becomes NULL."""

    def __init__(self):
        self.lib = load()
        import torch
        self._torch = torch
        self.launches = 0            # kernels launched through the C ABI (every entry point launches exactly one)
        self.timing = None           # when a dict: name -> list of (start_event, end_event), filled per call
        self.order = None            # when a list (and timing is on): entry-point names in launch order

    def stream(self):
        return self._torch.cuda.current_stream().cuda_stream

    def __getattr__(self, name):
        fn = getattr(self.lib, 'tfx_' + name)
        torch = self._torch

        def call(*args):
            conv = []
            for a in args:
                if a is None:
                    conv.append(None)
                elif torch.is_tensor(a):
                    conv.append(a.data_ptr())
                else:
                    conv.append(a)
            self.launches += 1
            if self.timing is not None:
                e0, e1 = torch.cuda.Event(enable_timing = True), torch.cuda.Event(enable_timing = True)
                e0.record()
                rc = fn(*conv, self.stream())
                e1.record()
                self.timing.setdefault(name, []).append((e0, e1, args))
                if self.order is not None:
                    self.order.append(name)
            else:
                rc = fn(*conv, self.stream())
            if rc != 0:
                check(rc, 'tfx_' + name)
        call.__name__ = name
        setattr(self, name, call)
        return call
