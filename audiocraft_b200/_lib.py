"""ctypes binding of libaudiocraft_b200.so (the C-ABI declared in include/audiocraft_b200.h).

There is NO CPU or PyTorch fallback: if the library is missing or a call fails, this raises.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('ACB_LIB') or os.path.join(_HERE, 'libaudiocraft_b200.so')   # ACB_LIB: another build (e.g. an ACB_BUILD_VARIANT one) for A/B runs

CONV_FP32, CONV_TF32X3, CONV_TF32X3_MMASYNC = 0, 1, 2
CONV_T6_FLUSH = 3   # host-side selector only: every layer acb_conv1d_t6 supports goes through it, the rest fp32 FMA
CONV_T6_AUTO = 4    # host-side selector only: acb_conv1d_t6 where it is faster (k > 1, >= 128 output channels), else fp32 FMA
ACB_LM_MAX_SPLIT = 8
ACB_LM_PART_SLOTS = 16
ACB_LM_PREFILL_ROWS = 64
ACB_LM_MAX_ROWS = 256
ACB_LM_SLOT_STRIDE = 8
ACB_LM_SLOT_SAMPLING_STRIDE = 8
ACB_LM_MAX_SLOTS = 128
ACB_LM_KV_PAGE = 64
ACB_LM_MAX_PAGES_PER_ROW = 188


class LMConfig(C.Structure):
    """acb_lm_config.  `_fields_` lists the fields up to positional_embedding, and callers build the structure from that
    list; every instance also carries the trailing `int weight_dtype` (0, fp16, unless given), so whatever builds it, the
    library never reads past its end."""
    _fields_ = [('dim', C.c_int), ('num_heads', C.c_int), ('num_layers', C.c_int), ('ffn_dim', C.c_int),
                ('n_q', C.c_int), ('card', C.c_int), ('cross_attention', C.c_int), ('max_rows', C.c_int),
                ('max_seq', C.c_int), ('max_text', C.c_int), ('pos_scale', C.c_float), ('positional_embedding', C.c_int)]

    def __init__(self, *args, weight_dtype: int = 0, **kw):
        super().__init__(*args, **kw)
        C.resize(self, C.sizeof(LMConfig) + C.sizeof(C.c_int))   # the added bytes are zero
        self.weight_dtype = weight_dtype

    @property
    def weight_dtype(self) -> int:
        return C.c_int.from_address(C.addressof(self) + C.sizeof(LMConfig)).value

    @weight_dtype.setter
    def weight_dtype(self, v: int):
        C.c_int.from_address(C.addressof(self) + C.sizeof(LMConfig)).value = int(v)


class LMWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('emb', 'inv_freq', 'w_qkv', 'w_o', 'w_cq', 'w_ckv', 'w_co', 'w_ff1',
                                           'w_ff2', 'ln', 'out_norm', 'heads', 'rope_freq', 's_qkv', 's_o', 's_cq', 's_ckv',
                                           's_co', 's_ff1', 's_ff2')]


class LMBuffers(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('x', 'h16', 'a16', 'f16', 'q32', 'part', 'logits', 'k_cache', 'v_cache',
                                           'ck_cache', 'cv_cache', 'cross16', 'seq', 'seq_mask', 'pos', 'noise', 'slot_sampling',
                                           'slot_state', 'slot_mask')]


class LMSampling(C.Structure):
    _fields_ = [('use_sampling', C.c_int), ('temp', C.c_float), ('top_k', C.c_int), ('top_p', C.c_float),
                ('cfg_coef', C.c_float), ('seed', C.c_uint64), ('noise_from_buffer', C.c_int), ('cfg_coef_beta', C.c_float)]


class T5Config(C.Structure):
    _fields_ = [('d_model', C.c_int), ('d_kv', C.c_int), ('num_heads', C.c_int), ('num_layers', C.c_int), ('d_ff', C.c_int),
                ('vocab_size', C.c_int), ('num_buckets', C.c_int), ('out_dim', C.c_int), ('eps', C.c_float)]


class T5Weights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('shared', 'w_qkv', 'w_o', 'w_i', 'w_fo', 'ln', 'final_ln', 'rel_bias', 'proj_w',
                                           'proj_b')]


_lib = None


def lib():
    """Load the library (once). Raises with build instructions when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: the CUDA kernels are not built. Run `python -m audiocraft_b200.build` "
            "(nvcc, sm_90a). There is no CPU / PyTorch fallback for this path.")
    L = C.CDLL(LIB_PATH)
    vp, ci, cf, i64 = C.c_void_p, C.c_int, C.c_float, C.c_int64
    L.acb_last_error.restype = C.c_char_p
    L.acb_version.restype = ci
    L.acb_device_sm_count.argtypes = [ci]
    L.acb_weight_norm_fold.argtypes = [vp, vp, vp, ci, ci, vp]
    L.acb_conv1d.argtypes = [vp, vp, vp, vp, vp] + [ci] * 13 + [vp]
    L.acb_convtr1d.argtypes = [vp, vp, vp, vp, vp] + [ci] * 10 + [vp]
    L.acb_conv1d_t6.argtypes = [vp, vp, vp, vp, vp] + [ci] * 12 + [vp]
    L.acb_conv1d_t6_tile.argtypes = [ci]
    L.acb_resblock_supported.argtypes = [ci, ci, ci]
    L.acb_resblock.argtypes = [vp] * 6 + [ci] * 8 + [vp]
    L.acb_lstm_recurrent.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, vp]
    L.acb_lstm_recurrent_carry.argtypes = [vp] * 7 + [ci, ci, ci, vp]
    L.acb_lstm_state_bytes.argtypes = [ci, ci]
    L.acb_lstm_state_bytes.restype = i64
    L.acb_rvq_encode.argtypes = [vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]
    L.acb_rvq_decode.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, vp]
    L.acb_groupnorm_workspace_bytes.argtypes = [ci, ci, ci]
    L.acb_groupnorm_workspace_bytes.restype = i64
    L.acb_groupnorm_stats.argtypes = [vp, vp, vp, ci, ci, ci, cf, vp]
    L.acb_groupnorm_apply.argtypes = [vp, vp, vp, vp, ci, ci, vp, vp, vp, vp, vp, vp, ci, ci, ci, vp]
    L.acb_overlap_add.argtypes = [vp, vp, vp, vp] + [ci] * 7 + [vp]
    L.acb_lm_create.argtypes = [C.POINTER(LMConfig), C.POINTER(LMWeights), C.POINTER(LMBuffers), C.POINTER(vp)]
    L.acb_lm_destroy.argtypes = [vp]
    L.acb_lm_begin.argtypes = [vp, vp, ci, ci, ci, ci, C.POINTER(LMSampling), vp]
    L.acb_lm_begin_prefix.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, C.POINTER(LMSampling), vp]
    L.acb_lm_steps.argtypes = [vp, ci, vp]
    L.acb_lm_begin_slots.argtypes = [vp, ci, ci, ci, C.POINTER(LMSampling), vp]
    L.acb_lm_admit.argtypes = [vp, ci, vp, ci, ci, C.c_uint64, C.POINTER(LMSampling), vp]
    L.acb_lm_admit_prefix.argtypes = [vp, ci, vp, ci, vp, ci, ci, C.c_uint64, C.POINTER(LMSampling), vp]
    L.acb_lm_retire.argtypes = [vp, ci, vp]
    L.acb_lm_begin_slots_paged.argtypes = [vp, ci, ci, ci, ci, vp, vp, ci, vp, ci, vp, vp, C.POINTER(LMSampling), vp]
    L.acb_lm_begin_slots_paged_fp8.argtypes = [vp, ci, ci, ci, ci, vp, vp, vp, vp, ci, vp, ci, vp, vp, C.POINTER(LMSampling), vp]
    L.acb_lm_admit_paged.argtypes = [vp, ci, vp, ci, vp, ci, ci, C.c_uint64, C.POINTER(LMSampling), vp, ci, vp]
    L.acb_lm_admit_prompt.argtypes = [vp, ci, vp, ci, vp, ci, ci, ci, C.c_uint64, C.POINTER(LMSampling), vp, ci, vp]
    L.acb_lm_slot_status.argtypes = [vp, vp, vp]
    L.acb_lm_prefill.argtypes = [vp, ci, ci, vp]
    L.acb_lm_step_logits.argtypes = [vp, vp, vp]
    L.acb_lm_launches_per_step.argtypes = [vp]
    L.acb_lm_rows_pad.argtypes = [ci]
    L.acb_lm_uses_pdl.argtypes = [vp]
    L.acb_lm_debug_gemms.argtypes = [vp, vp, C.POINTER(ci)]
    L.acb_sample.argtypes = [vp, vp, vp, ci, ci, ci, ci, C.POINTER(LMSampling), C.c_uint64, vp]
    L.acb_lm_forward_workspace_bytes.argtypes = [C.POINTER(LMConfig), ci, ci, ci, ci]
    L.acb_lm_forward_workspace_bytes.restype = i64
    L.acb_lm_forward.argtypes = [C.POINTER(LMConfig), C.POINTER(LMWeights), vp, vp, vp, ci, ci, ci, ci, vp, vp, i64, vp]
    L.acb_t5_workspace_bytes.argtypes = [C.POINTER(T5Config), ci, ci]
    L.acb_t5_workspace_bytes.restype = i64
    L.acb_t5_encode.argtypes = [C.POINTER(T5Config), C.POINTER(T5Weights), vp, vp, vp, ci, ci, vp, vp, vp, i64, vp]
    for name in ('acb_weight_norm_fold', 'acb_conv1d', 'acb_convtr1d', 'acb_lstm_recurrent', 'acb_lstm_recurrent_carry',
                 'acb_rvq_encode',
                 'acb_rvq_decode', 'acb_lm_create', 'acb_lm_destroy', 'acb_lm_begin', 'acb_lm_begin_prefix', 'acb_lm_steps',
                 'acb_lm_step_logits', 'acb_lm_launches_per_step', 'acb_lm_rows_pad', 'acb_sample',
                 'acb_device_sm_count', 'acb_lm_debug_gemms', 'acb_lm_uses_pdl',
                 'acb_conv1d_t6', 'acb_conv1d_t6_tile', 'acb_lm_prefill',
                 'acb_resblock', 'acb_resblock_supported', 'acb_lm_forward', 'acb_t5_encode', 'acb_groupnorm_stats',
                 'acb_groupnorm_apply', 'acb_overlap_add', 'acb_lm_begin_slots', 'acb_lm_admit', 'acb_lm_slot_status', 'acb_lm_retire',
                 'acb_lm_admit_prefix', 'acb_lm_begin_slots_paged', 'acb_lm_admit_paged', 'acb_lm_admit_prompt',
                 'acb_lm_begin_slots_paged_fp8'):
        getattr(L, name).restype = ci
    _lib = L
    return L


# every symbol include/audiocraft_b200.h declares (checked by tests/test_host.py against the header text)
EXPORTS = ['acb_version', 'acb_last_error', 'acb_device_sm_count', 'acb_weight_norm_fold', 'acb_conv1d', 'acb_convtr1d',
           'acb_lstm_recurrent', 'acb_lstm_state_bytes', 'acb_rvq_encode', 'acb_rvq_decode', 'acb_lm_create',
           'acb_lm_destroy', 'acb_lm_begin', 'acb_lm_begin_prefix', 'acb_lm_steps', 'acb_lm_step_logits', 'acb_lm_rows_pad',
           'acb_lm_launches_per_step', 'acb_lm_debug_gemms', 'acb_lm_uses_pdl', 'acb_sample', 'acb_conv1d_t6', 'acb_conv1d_t6_tile',
           'acb_lm_prefill', 'acb_resblock', 'acb_resblock_supported', 'acb_lm_forward_workspace_bytes', 'acb_lm_forward',
           'acb_t5_workspace_bytes', 'acb_t5_encode', 'acb_groupnorm_workspace_bytes', 'acb_groupnorm_stats',
           'acb_groupnorm_apply', 'acb_overlap_add', 'acb_lstm_recurrent_carry', 'acb_lm_begin_slots', 'acb_lm_admit',
           'acb_lm_slot_status', 'acb_lm_retire', 'acb_lm_admit_prefix', 'acb_lm_begin_slots_paged', 'acb_lm_admit_paged',
           'acb_lm_admit_prompt', 'acb_lm_begin_slots_paged_fp8']


def check(rc: int, what: str = ''):
    if rc != 0:
        msg = lib().acb_last_error().decode(errors='replace')
        raise RuntimeError(f"audiocraft_b200 {what} failed (status {rc}): {msg}")


def ptr(t) -> int:
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), "the C-ABI takes contiguous CUDA tensors"
    return t.data_ptr()


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def require_cuda(device):
    if not torch.cuda.is_available():
        raise RuntimeError("audiocraft_b200 runs on CUDA (H100, sm_90a) only; no CPU fallback exists")
    return torch.device(device if device is not None else 'cuda')
