"""ctypes binding of libnts_b200.so - the C ABI declared in include/nts_b200.h - and the plumbing every caller shares:
status and handle checks, the current stream, borrowed device arrays and caller ids.

There is no fallback: if the shared object is missing or a call fails, we raise.
"""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np
import torch

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
LIB_PATH = os.path.join(PKG, "lib", "libnts_b200.so")
HEADER = os.path.join(ROOT, "include", "nts_b200.h")

_vp = C.c_void_p
_u32 = C.c_uint32
_u64 = C.c_uint64
_int = C.c_int
_sz = C.c_size_t

# name -> (restype, argtypes).  Pointers are passed as integers (device addresses from torch .data_ptr()).
SIGNATURES = {
    "nts_version": (_int, []),
    "nts_last_error": (C.c_char_p, []),
    "nts_device_count": (_int, []),
    "nts_set_device": (_int, [_int]),
    "nts_device_sm_count": (_int, [C.POINTER(_int)]),
    "nts_device_synchronize": (_int, []),
    "nts_device_reset": (_int, []),
    "nts_malloc_device": (_vp, [_sz]),
    "nts_free_device": (_int, [_vp]),
    "nts_malloc_pinned": (_vp, [_sz]),
    "nts_free_pinned": (_int, [_vp]),
    "nts_pinned_device_pointer": (_vp, [_vp]),
    "nts_memcpy_h2d": (_int, [_vp, _vp, _sz, _vp, _int]),
    "nts_memcpy_d2h": (_int, [_vp, _vp, _sz, _vp, _int]),
    "nts_memcpy_d2d": (_int, [_vp, _vp, _sz, _vp]),
    "nts_zero": (_int, [_vp, _sz, _vp]),
    "nts_stream_create": (_vp, [_int]),
    "nts_stream_destroy": (_int, [_vp]),
    "nts_stream_synchronize": (_int, [_vp]),
    "nts_event_create": (_vp, [_int]),
    "nts_event_destroy": (_int, [_vp]),
    "nts_event_record": (_int, [_vp, _vp]),
    "nts_stream_wait_event": (_int, [_vp, _vp]),
    "nts_event_elapsed_ms": (_int, [_vp, _vp, C.POINTER(C.c_float)]),
    "nts_segment_gather_sum": (_int, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _u64, _u32, _vp]),
    "nts_gather_by_dst_from_src": (_int, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _u32, _u32, _u32, _u32, _u32, _int, _vp]),
    "nts_gather_by_src_from_dst": (_int, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _u32, _u32, _u32, _u32, _u32, _int, _vp]),
    "nts_segment_gather_sum_range": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _u64, _u64, _u32, _vp]),
    "nts_segment_gather_sum_bf16": (_int, [_vp, _u32, _vp, _vp, _vp, _vp, _u32, _u64, _u32, _vp]),
    "nts_segment_gather_sum_sharded": (_int, [_vp, _vp, _int, _vp, _int, _u32, _vp, _vp, _vp, _u32, _u64, _u64, _u32,
                                              _vp]),
    "nts_gat_softmax_stats_sharded": (_int, [_vp, _vp, _vp, _vp, _int, _u32, _vp, _vp, _vp, _u32, _u64, _u64, _u32,
                                             C.c_float, _vp]),
    "nts_gat_aggregate_sharded": (_int, [_vp, _vp, _int, _vp, _int, _u32, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _u32,
                                         _u64, _u64, _u32, _u32, C.c_float, _vp]),
    "nts_gather_plan_pick_slabs": (_int, [_u32, _u64, _u32, _u32, _u64]),
    "nts_gather_plan_create_hybrid": (_vp, [_vp, _vp, _vp, _vp, _u32, _u32, _u64, _u32, _int, _int, _int, _vp]),
    "nts_gather_plan_create_parts": (_vp, [_vp, _int, _u32, _u32, _int, _u32, _vp]),
    "nts_gather_plan_tuned_ms": (C.c_float, [_vp]),
    "nts_gather_plan_destroy": (_int, [_vp]),
    "nts_gather_plan_slabs": (_int, [_vp]),
    "nts_gather_plan_hubs": (_int, [_vp, C.POINTER(_int), C.POINTER(_int)]),
    "nts_gather_plan_overlap": (_int, [_vp]),
    "nts_gather_plan_set_overlap": (_int, [_vp, _int]),
    "nts_gather_plan_bytes": (_u64, [_vp]),
    "nts_gather_plan_run_ex": (_int, [_vp, _vp, _u32, _vp, _u32, _int, _vp]),
    "nts_gather_plan_run_bf16_ex": (_int, [_vp, _vp, _int, _u32, _vp, _u32, _int, _vp]),
    "nts_gather_plan_create_tuned_ex": (_vp, [_vp, _vp, _vp, _vp, _u32, _u32, _u64, _u32, _u32, _int, _int, _vp]),
    "nts_gather_plan_last_launch": (_int, [_vp] + [C.POINTER(_int)] * 5),
    "nts_gather_plan_set_tuning": (_int, [_int, _int, _int]),
    "nts_gather_plan_set_variant": (_int, [_int]),
    "nts_segment_gather_sum_slots": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _u32, _u64, _u32, _vp]),
    "nts_segment_gather_sum_heads": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _u64, _u32, _u32, _vp]),
    "nts_aggregate_set_variant": (_int, [_int, _int]),
    "nts_aggregate_last_launch": (_int, [C.POINTER(_int)] * 4),
    "nts_aggregate_last_shape": (_int, [C.POINTER(_int)] * 5),
    "nts_kernel_launch_count": (_u64, []),
    "nts_scatter_src_mirror_to_msg": (_int, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_gather_msg_to_src_mirror": (_int, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_scatter_dst_to_msg": (_int, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_gather_msg_to_dst": (_int, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_edge_softmax_forward": (_int, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_edge_softmax_backward": (_int, [_vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_scatter_grad_back_to_message": (_int, [_vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_aggregate_dst_fuse_weight_backward": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_aggregate_dst_fuse_weight_backward_heads": (_int, [_vp] * 8 + [_u32, _u32, _u32, _vp]),
    "nts_gat_softmax_stats": (_int, [_vp] * 7 + [_u32, _u32, C.c_float, _vp]),
    "nts_gat_fused_aggregate_forward": (_int, [_vp] * 9 + [_u32, _u64, _u32, _u32, C.c_float, _vp]),
    "nts_gat_fused_aggregate_backward": (_int, [_vp] * 13 + [_u32, _u32, _u32, C.c_float, _vp]),
    "nts_gat_fused_aggregate_backward_two_pass": (_int, [_vp] * 16 + [_u32, _u32, _u32, _u32, C.c_float, _vp]),
    "nts_gat_fused_aggregate_forward_bf16": (_int, [_vp] * 9 + [_u32, _u64, _u32, _u32, _u32, C.c_float, _vp]),
    "nts_gat_fused_aggregate_backward_two_pass_bf16": (_int, [_vp] * 16 + [_u32] * 5 + [C.c_float, _vp]),
    "nts_rows_to_bf16": (_int, [_vp, _int, _u32, _vp, _u32, _u32, _u32, _vp]),
    "nts_deserialize_records": (_int, [_vp, _vp, _u32, _u32, _u32, _u32, _vp]),
    "nts_aggregate_records": (_int, [_vp, _vp, _u32, _u32, _u32, _u32, _vp]),
    "nts_gather_rows": (_int, [_vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_gather_rows_sharded": (_int, [_vp, _vp, _vp, _int, _u32, _vp, _u32, _u32, _vp]),
    "nts_gather_rows_sharded_bf16": (_int, [_vp, _int, _u32, _vp, _vp, _int, _u32, _vp, _u32, _u32, _vp]),
    "nts_scatter_add_rows": (_int, [_vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_scatter_add_rows_atomic": (_int, [_vp, _vp, _vp, _u32, _u32, _vp]),
    "nts_ipc_get_handle": (_int, [_vp, C.c_char_p]),
    "nts_ipc_open_handle": (_vp, [C.c_char_p]),
    "nts_ipc_close_handle": (_int, [_vp]),
    "nts_adam_update": (_int, [_vp, _vp, _vp, _vp, _u64] + [C.c_float] * 5 + [_vp]),
    "nts_embedding_step": (_int, [_vp] * 7 + [_int, _u32, _u32, _u32, _u32, _u32] + [C.c_float] * 5 + [_vp]),
    "nts_signal_set": (_int, [_vp, _u32, _vp]),
    "nts_signal_wait_geq": (_int, [_vp, _u32, _vp]),
    "nts_host_degrees": (_int, [_vp, _u64, _u32, _vp, _vp]),
    "nts_host_partition_offsets": (_int, [_vp, _u64, _u32, _int, _vp]),
    "nts_host_chunk_edge_counts": (_int, [_vp, _u64, _vp, _int, _int, _vp]),
    "nts_host_build_chunk": (_int, [_vp, _u64, _u32, _vp, _int, _int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nts_host_mirror_index": (_int, [_vp, _u64, _u32, _vp, _int, _vp, _vp]),
    "nts_host_read_feature_label_mask": (_int, [C.c_char_p, C.c_char_p, C.c_char_p, _u32, _u32, _u32, _vp, _vp, _vp]),
    "nts_host_read_feature_binary": (_int, [C.c_char_p, _u32, _u32, _u32, _vp]),
    "nts_graph_build_from_file": (_vp, [C.c_char_p, _u32, _int, _int, _vp, _u64, _int, _vp]),
    "nts_graph_build_from_device": (_vp, [_vp, _vp, _int, _u64, _u32, _int, _int, _vp, _vp, _vp, _int, _vp]),
    "nts_graph_build_info": (_int, [_vp] * 6),
    "nts_graph_build_export_chunk": (_int, [_vp, _int] + [_vp] * 8),
    "nts_graph_build_export_dist": (_int, [_vp] * 5),
    "nts_graph_build_export_degrees": (_int, [_vp] * 4),
    "nts_graph_build_destroy": (_int, [_vp]),
}



class ExchangeChunk(C.Structure):
    """nts_exchange_chunk of include/nts_b200.h (device arrays of one remote chunk)."""
    _fields_ = [
        ("column_offset", _vp), ("slots", _vp), ("weight_forward", _vp), ("row_offset_compact", _vp),
        ("column_indices", _vp), ("weight_backward", _vp), ("edges", _u64),
    ]


class ExchangeDesc(C.Structure):
    """nts_exchange_desc of include/nts_b200.h."""
    _fields_ = [
        ("partitions", _int), ("rank", _int), ("owned_vertices", _u32), ("dst_start", _u32),
        ("local_column_offset", _vp), ("local_row_indices", _vp), ("local_row_offset", _vp),
        ("local_column_indices", _vp), ("local_weight_forward", _vp), ("local_weight_backward", _vp),
        ("local_edges", _u32),
        ("chunks", C.POINTER(ExchangeChunk)),
        ("need_count", C.POINTER(_u32)), ("send_count", C.POINTER(_u32)),
        ("send_rows_all", _vp), ("fwd_push_offset", C.POINTER(_u32)), ("bwd_push_offset", C.POINTER(_u32)),
        ("local_need", _vp), ("local_need_count", _u32),
    ]


class DeviceChunk(C.Structure):
    """nts_device_chunk of include/nts_b200.h."""
    _fields_ = [
        ("column_offset", _vp), ("row_indices", _vp), ("row_offset", _vp), ("column_indices", _vp),
        ("edge_weight_forward", _vp), ("edge_weight_backward", _vp),
    ]


SIGNATURES.update({
    "nts_exchange_create": (_vp, [C.POINTER(ExchangeDesc)]),
    "nts_exchange_destroy": (_int, [_vp]),
    "nts_exchange_required_floats": (_u64, [_vp, _u32]),
    "nts_exchange_capacity_floats": (_u64, [_vp]),
    "nts_exchange_release_peers": (_int, [_vp]),
    "nts_exchange_reserve": (_int, [_vp, _u64, _int]),
    "nts_exchange_handles": (_int, [_vp, C.c_char_p, C.c_char_p]),
    "nts_exchange_open_peers": (_int, [_vp, C.c_char_p, C.c_char_p]),
    "nts_exchange_forward": (_int, [_vp, _vp, _vp, _u32, _vp]),
    "nts_exchange_backward": (_int, [_vp, _vp, _vp, _u32, _vp]),
    "nts_exchange_forward_bf16": (_int, [_vp, _vp, _int, _vp, _u32, _vp]),
    "nts_exchange_backward_bf16": (_int, [_vp, _vp, _vp, _u32, _vp]),
    "nts_exchange_required_floats_bf16": (_u64, [_vp, _u32]),
    "nts_exchange_set_trace": (_int, [_vp, _int]),
    "nts_exchange_last_timeline": (_int, [_vp, C.POINTER(C.c_float), _int]),
    "nts_exchange_last_paths": (_int, [_vp] + [C.POINTER(_int)] * 4 + [C.POINTER(_u32)] * 2 +
                                [C.POINTER(_int), C.POINTER(_u32), C.POINTER(_int)]),
    "nts_exchange_fetch_mirrors": (_int, [_vp, _vp, _vp, _u32, _vp]),
    "nts_exchange_return_mirror_grads": (_int, [_vp, _vp, _vp, _u32, _vp]),
})



class HostChunk(C.Structure):
    """nts_host_chunk of include/nts_b200.h (host arrays of one CSC_segment_pinned)."""
    _fields_ = [
        ("column_offset", _vp), ("row_indices", _vp), ("row_offset", _vp), ("column_indices", _vp),
        ("edge_weight_forward", _vp), ("edge_weight_backward", _vp),
        ("src_start", _u32), ("src_end", _u32), ("dst_start", _u32), ("dst_end", _u32), ("edges", _u64),
    ]


class ExchangePlanView(C.Structure):
    """nts_exchange_plan_view of include/nts_b200.h."""
    _fields_ = [
        ("partitions", _int), ("rank", _int),
        ("owned_vertices", _u32), ("recv_total", _u32), ("send_total", _u32), ("backward_rows", _u32),
        ("remote_edges", _u64),
        ("need_count", C.POINTER(_u32)), ("send_count", C.POINTER(_u32)), ("peer_bwd_offset", C.POINTER(_u32)),
        ("fwd_push_offset", C.POINTER(_u32)), ("bwd_push_offset", C.POINTER(_u32)),
        ("remote_column_offset", C.POINTER(_u32)), ("remote_slots", C.POINTER(_u32)),
        ("remote_weight", C.POINTER(C.c_float)),
        ("backward_offsets", C.POINTER(_u32)), ("backward_indices", C.POINTER(_u32)),
        ("backward_weight", C.POINTER(C.c_float)),
        ("send_rows_all", C.POINTER(_u32)),
    ]


SIGNATURES.update({
    "nts_exchange_plan_create": (_vp, [C.POINTER(HostChunk), _int, _int]),
    "nts_exchange_plan_destroy": (None, [_vp]),
    "nts_exchange_plan_need": (C.POINTER(_u32), [_vp, _int, C.POINTER(_u32)]),
    "nts_exchange_plan_packed_rows": (_u64, [_vp]),
    "nts_exchange_plan_pack_needs": (_int, [_vp, _vp, _vp]),
    "nts_exchange_plan_set_peer_needs": (_int, [_vp, _int, _vp, _vp]),
    "nts_exchange_plan_finalize": (_int, [_vp]),
    "nts_exchange_plan_get_view": (_int, [_vp, C.POINTER(ExchangePlanView)]),
    "nts_exchange_plan_chunk": (_int, [_vp, _int, C.POINTER(C.POINTER(_u32)), C.POINTER(C.POINTER(_u32))]),
    "nts_exchange_create_from_plan": (_vp, [_vp, C.POINTER(DeviceChunk)]),
})


class SampleHopView(C.Structure):
    """nts_sample_hop_view of include/nts_b200.h (device arrays of one sampled hop)."""
    _fields_ = [
        ("n_dst", _u32), ("n_src", _u32), ("n_edges", _u64),
        ("dst", _vp), ("column_offset", _vp), ("row_indices", _vp), ("row_global", _vp), ("weight", _vp),
        ("src", _vp), ("row_offset", _vp), ("column_indices", _vp), ("weight_backward", _vp),
    ]


SIGNATURES.update({
    "nts_sampler_create": (_vp, [_vp, _vp, _vp, _u32, _u64, _u32, _int, C.POINTER(_int), _vp]),
    "nts_sampler_create_ex": (_vp, [_vp, _vp, _vp, _u32, _u64, _u32, _int, C.POINTER(_int), _u32, _vp]),
    "nts_sampler_sample": (_int, [_vp, _vp, _u32, _u64, _u64, _vp]),
    "nts_sampler_hop_view": (_int, [_vp, _int, C.POINTER(SampleHopView)]),
    "nts_sampler_hop_dst_pos": (_int, [_vp, _int, C.POINTER(_vp)]),
    "nts_sampler_bytes": (_u64, [_vp]),
    "nts_sampler_destroy": (_int, [_vp]),
    "nts_sample_transpose": (_int, [_vp, _vp, _vp, _u32, _u32, _u64, _vp, _vp, _vp, _vp]),
    "nts_sampler_create_sharded": (_vp, [C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_u32), _int, _u32,
                                         _int, C.POINTER(_int), _u32, _vp]),
    "nts_merge_chunk_csc": (_int, [C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), _int, _u32, _u64, _vp, _vp, _vp,
                                   _vp]),
})

_lib = None


class NtsError(RuntimeError):
    pass


def header_symbols():
    """Every function name declared in include/nts_b200.h (used by the CPU tests)."""
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(nts_[a-z0-9_]+)\s*\(", text)))


def load():
    """dlopen libnts_b200.so (building it is `python -m neutronstarlite_b200.build`). Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NtsError("libnts_b200.so not found at %s - run `python -m neutronstarlite_b200.build` "
                       "(there is no CPU fallback)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error():
    """The text of the library's last failure on this thread."""
    return load().nts_last_error().decode(errors="replace")


def check(rc, what=""):
    if rc != 0:
        raise NtsError("libnts_b200 %s failed (rc=%d): %s" % (what, rc, last_error()))


def call(name, *args):
    """Invoke an int-returning ABI function and raise on a non-zero status."""
    rc = getattr(load(), name)(*args)
    check(rc, name)


def checked(handle, what):
    """A handle or pointer an ABI function returned; NtsError with the library's reason when it is null."""
    if not handle:
        raise NtsError("%s failed: %s" % (what, last_error()))
    return handle


def stream(device=None):
    """The current CUDA stream of `device` (default: the current device), as the ABI's stream argument."""
    return torch.cuda.current_stream(device).cuda_stream


class _DeviceArray:
    """A borrowed 1-D device array for torch.as_tensor (the CUDA array interface; no copy, no stream sync)."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2, "strides": None}


_TYPESTR = {torch.int32: "<i4", torch.float32: "<f4"}


def borrowed(ptr, n, dtype, device):
    """A tensor over n int32 or float32 values of device memory at ptr that the library owns (no copy); an empty tensor
    when n == 0, whatever ptr is."""
    if n == 0:
        return torch.empty(0, dtype=dtype, device=device)
    return torch.as_tensor(_DeviceArray(ptr, n, _TYPESTR[dtype]), device=device)


def device_ids(ids, bound, device, name, what):
    """Caller ids (an integer tensor, numpy array or list) as a contiguous int32 tensor on `device`.  Ids outside
    [0, bound) raise NtsError ("<what> must be in [0, bound)") before any device work for host ids; device ids are
    checked in the caller's dtype, since a cast first could wrap an int64 id >= 2^32 into range."""
    if torch.is_tensor(ids) and ids.is_cuda:
        if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
            raise NtsError("%s must be an integer tensor, not %s" % (name, ids.dtype))
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= bound):
            raise NtsError("%s must be in [0, %d)" % (what, bound))
        return ids.reshape(-1).to(device=device, dtype=torch.int32).contiguous()
    a = np.asarray(ids.numpy() if torch.is_tensor(ids) else ids).reshape(-1).astype(np.int64)
    if a.size and (a.min() < 0 or a.max() >= bound):
        raise NtsError("%s must be in [0, %d)" % (what, bound))
    return torch.from_numpy(a.astype(np.int32)).to(device)
