"""ctypes binding of `libpipeedge_b200.so` (the C-ABI declared in `include/pipeedge_b200.h`).

There is no CPU fallback: if the library is missing this module raises at import, and every call on a
machine without an sm_90 (H100) GPU fails with `PipeEdgeB200Error` (PE_ERR_DEVICE).
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_longlong, c_size_t, c_uint64, c_ulonglong, c_void_p

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, 'libpipeedge_b200.so')

PE_OK = 0
PE_FAMILY = {'vit': 0, 'deit': 1, 'bert': 2}
PE_EPI_F16, PE_EPI_GELU_F16, PE_EPI_RESID_F32, PE_EPI_F32, PE_EPI_TANH_F32 = range(5)
PE_EPI_STATIC_W = 0x100   # OR-able flag: W is a model weight (not produced by pending work on the stream)
PE_CLAMP_NONE, PE_CLAMP_AUTO, PE_CLAMP_LAPLACE, PE_CLAMP_GELU = range(4)
PE_STAGE_DEFER_ADD = 2        # OR-able into pe_stage_forward's use_graph (eager only)
PE_LINK_HEADER_BYTES = 16384
PE_LINK_PATH_COPY, PE_LINK_PATH_FUSED, PE_LINK_PATH_STAGED = range(3)   # pe_debug_link_put_plan
PE_ABI_VERSION = 2
PE_PIPE_STAMP_DEPTH = 256
PE_STAMP_OVERLAPPED, PE_STAMP_FUSED, PE_STAMP_STAGED = 1, 2, 4   # pe_pipe_record.flags


class PipeEdgeB200Error(RuntimeError):
    """A C-ABI call returned a negative status."""


class BlockWeights(Structure):
    """`pe_block_weights`."""
    _fields_ = [(n, c_void_p) for n in ('w_qkv', 'b_qkv', 'w_o', 'b_o', 'w_fc1', 'b_fc1', 'w_fc2', 'b_fc2',
                                        'ln1_w', 'ln1_b', 'ln2_w', 'ln2_b')]


class StageDesc(Structure):
    """`pe_stage_desc`."""
    _fields_ = [('family', c_int), ('hidden', c_int), ('heads', c_int), ('inter', c_int), ('tokens', c_int),
                ('eps', c_float), ('layer_start', c_int), ('layer_end', c_int), ('max_ubatch', c_int)]


class PipeRecord(Structure):
    """`pe_pipe_record`: one micro-batch's device timestamps (%globaltimer ns) on a pipe with stamps on."""
    _fields_ = [(n, c_ulonglong) for n in ('index', 't_start', 't_got', 't_stage', 't_send_start', 't_encoded',
                                           't_send_end', 'bytes_out')] + \
               [(n, c_int) for n in ('items', 'bit_out', 'bit_in', 'flags')]


# name -> (restype, argtypes); every symbol declared in include/pipeedge_b200.h
SYMBOLS = {
    'pe_abi_version': (c_int, []),
    'pe_last_error': (c_char_p, []),
    'pe_launch_count': (c_uint64, []),
    'pe_layernorm': (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    'pe_residual_layernorm': (c_int, [c_void_p] * 4 + [c_float] + [c_void_p] * 3 + [c_int, c_int, c_void_p]),
    'pe_linear': (c_int, [c_void_p] * 5 + [c_int] * 4 + [c_void_p]),
    'pe_linear_residual_layernorm': (c_int, [c_void_p] * 6 + [c_float, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int,
                                             c_void_p]),
    'pe_linear_ln_cluster': (c_int, [c_int]),
    'pe_attention': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    'pe_cast_f32_to_f16': (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    'pe_cast_f16_to_f32': (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    'pe_quant_words': (c_size_t, [c_size_t, c_int]),
    'pe_quant_workspace_bytes': (c_size_t, [c_int, c_size_t]),
    'pe_quant_encode': (c_int, [c_void_p, c_int, c_size_t, c_int, c_int] + [c_void_p] * 6),
    'pe_quant_alpha': (c_int, [c_void_p, c_int, c_size_t, c_int, c_int] + [c_void_p] * 5),
    'pe_quant_decode': (c_int, [c_void_p, c_int, c_size_t, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'pe_quant_clamp_factor': (c_float, [c_int, c_int]),
    'pe_stage_create': (c_int, [POINTER(StageDesc), POINTER(BlockWeights), c_int, POINTER(c_void_p)]),
    'pe_stage_destroy': (c_int, [c_void_p]),
    'pe_stage_forward': (c_int, [c_void_p] * 5 + [c_int, c_int, c_void_p]),
    'pe_stage_profile': (c_int, [c_void_p] * 5 + [c_int, c_void_p, POINTER(c_float), POINTER(c_int), c_int,
                                 POINTER(c_int)]),
    'pe_stage_kernel_count': (c_int, [c_void_p]),
    'pe_stage_deferred': (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_void_p)]),
    'pe_patch_embed': (c_int, [c_void_p] * 7 + [c_int] * 6 + [c_void_p]),
    'pe_bert_embed': (c_int, [c_void_p] * 7 + [c_float, c_void_p, c_int, c_int, c_int, c_void_p]),
    'pe_hop_available': (c_int, []),
    'pe_hop_open': (c_int, [c_int, c_int, POINTER(c_void_p)]),
    'pe_hop_close': (c_int, [c_void_p]),
    'pe_hop_send': (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_size_t), c_int, c_void_p, c_void_p, c_void_p, c_int]),
    'pe_hop_wait_envelope': (c_int, [c_void_p, POINTER(c_longlong)]),
    'pe_hop_recv': (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_size_t), POINTER(c_void_p), c_int, c_void_p, c_void_p]),
    'pe_link_open': (c_int, [c_int, c_int, c_size_t, c_int, c_int, POINTER(c_void_p)]),
    'pe_link_open_local': (c_int, [c_size_t, c_int, c_int, POINTER(c_void_p)]),
    'pe_link_open_host': (c_int, [c_size_t, c_int, POINTER(c_void_p)]),
    'pe_link_close': (c_int, [c_void_p]),
    'pe_link_slot_bytes': (c_size_t, [c_void_p]),
    'pe_link_put': (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_size_t, c_int, c_int, c_int,
                            c_void_p]),
    'pe_quant_encode_send': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_size_t, c_int, c_int, c_void_p]),
    'pe_link_get': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_size_t, c_size_t, c_void_p]),
    'pe_link_get_raw': (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    'pe_link_feed': (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_void_p]),
    'pe_link_ticket_send': (c_int, [c_void_p, c_longlong, c_longlong]),
    'pe_link_ticket_recv': (c_int, [c_void_p, POINTER(c_longlong)]),
    'pe_link_check': (c_int, [c_void_p]),
    'pe_link_debug_read': (c_int, [c_void_p, c_ulonglong, c_size_t, c_void_p, c_size_t]),
    'pe_hostring_create': (c_int, [c_int, c_char_p, c_int, c_size_t, c_int, POINTER(c_void_p)]),
    'pe_hostring_attach': (c_int, [c_int, c_int, c_size_t, c_int, POINTER(c_void_p)]),
    'pe_hostring_close': (c_int, [c_void_p]),
    'pe_hostring_slot_bytes': (c_size_t, [c_void_p]),
    'pe_hostring_publish': (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_longlong]),
    'pe_hostring_close_input': (c_int, [c_void_p]),
    'pe_hostring_next': (c_int, [c_void_p, POINTER(c_longlong)]),
    'pe_hostring_wait': (c_int, [c_void_p, c_int, c_size_t, POINTER(c_void_p)]),
    'pe_hostring_release': (c_int, [c_void_p]),
    'pe_link_is_shm': (c_int, [c_void_p]),
    'pe_link_shm_wait': (c_int, [c_void_p, c_int, c_size_t, POINTER(c_void_p)]),
    'pe_link_shm_release': (c_int, [c_void_p, c_void_p]),
    'pe_pipe_create': (c_int, [c_void_p, c_void_p, c_void_p, POINTER(c_void_p)]),
    'pe_pipe_destroy': (c_int, [c_void_p]),
    'pe_pipe_stream': (c_void_p, [c_void_p]),
    'pe_pipe_copy_stream': (c_void_p, [c_void_p]),
    'pe_pipe_has_graph': (c_int, [c_void_p, c_int, c_longlong]),
    'pe_pipe_set_send_bit': (c_int, [c_void_p, c_int]),
    'pe_pipe_has_variant': (c_int, [c_void_p, c_int, c_longlong, c_int]),
    'pe_pipe_capture_begin': (c_int, [c_void_p, c_int, c_longlong, c_int, c_void_p, c_void_p, c_size_t, c_size_t, c_size_t]),
    'pe_pipe_capture_end': (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_size_t, c_int, c_int,
                                    c_int, c_int, POINTER(c_int)]),
    'pe_pipe_capture_relay': (c_int, [c_void_p, c_int, c_longlong, c_size_t, POINTER(c_int)]),
    'pe_pipe_capture_abort': (c_int, [c_void_p]),
    'pe_pipe_invalidate': (c_int, [c_void_p]),
    'pe_pipe_set_out_dim': (c_int, [c_void_p, c_longlong]),
    'pe_pipe_submit': (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_int, c_longlong]),
    'pe_pipe_close_input': (c_int, [c_void_p]),
    'pe_pipe_run': (c_int, [c_void_p, POINTER(c_longlong)]),
    'pe_pipe_next_result': (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_int), POINTER(c_size_t)]),
    'pe_pipe_sync': (c_int, [c_void_p]),
    'pe_pipe_timing_reset': (c_int, [c_void_p]),
    'pe_pipe_timing': (c_int, [c_void_p, POINTER(c_float), POINTER(c_float), POINTER(c_ulonglong),
                               POINTER(c_ulonglong)]),
    'pe_pipe_enable_stamps': (c_int, [c_void_p, c_int]),
    'pe_pipe_drain_stamps': (c_int, [c_void_p, POINTER(PipeRecord), c_int, POINTER(c_int), POINTER(c_ulonglong)]),
    'pe_link_payload_bytes': (c_size_t, [c_int, c_size_t, c_int, c_int]),
    'pe_debug_gemm_trace': (c_int, [c_void_p]),
    'pe_debug_gemm_plan': (c_int, [c_int] * 4 + [c_void_p]),
    'pe_debug_link_put_plan': (c_int, [c_int, c_size_t, c_int, c_int, c_void_p]),
    'pe_debug_linear_simt': (c_int, [c_void_p] * 5 + [c_int] * 4 + [c_void_p]),
}


def _load() -> ctypes.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -m pipeedge_b200.build` "
                          "(pipeedge_b200 has no CPU or PyTorch fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SYMBOLS.items():
        fn = getattr(lib, name)   # AttributeError if the .so lacks a declared symbol
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


LIB = _load()


def check(status: int) -> None:
    """Raise `PipeEdgeB200Error` with the library's message on a negative status."""
    if status != PE_OK:
        raise PipeEdgeB200Error(f"status {status}: {LIB.pe_last_error().decode()}")
