"""ctypes loader for libenoki_b200.so (the C ABI declared in include/enoki_b200.h).

There is deliberately no fallback: if the CUDA extension has not been built the
import fails loudly (build it with ``python -c 'import __graft_entry__ as g; g.build()'``
or ``make -C enoki_b200/csrc``).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libenoki_b200.so")

c_u32, c_u64, c_sz, c_int, c_vp = (ctypes.c_uint32, ctypes.c_uint64, ctypes.c_size_t,
                                   ctypes.c_int, ctypes.c_void_p)


class ek_stats(ctypes.Structure):
    _fields_ = [("launches", c_u64), ("sweep_launches", c_u64), ("adjoint_launches", c_u64),
                ("ops_evaluated", c_u64), ("edge_adjoints", c_u64), ("bytes_in", c_u64),
                ("bytes_out", c_u64), ("last_kernel_ms", ctypes.c_float),
                ("total_kernel_ms", ctypes.c_float), ("fast_launches", c_u64), ("partition_device", c_u64)]


# name -> (restype, argtypes); every symbol include/enoki_b200.h declares
SIGNATURES = {
    "ek_init": (c_int, []),
    "ek_dist_unique_id": (c_int, [c_vp]),
    "ek_dist_init": (c_int, [c_int, c_int, c_vp]),
    "ek_dist_rank": (c_int, []),
    "ek_dist_world": (c_int, []),
    "ek_allreduce": (c_int, [c_int, c_vp, c_sz]),
    "ek_allreduce_scalars": (c_int, [c_vp, c_sz]),
    "ek_dist_shutdown": (None, []),
    "ek_set_fast_mode": (None, [c_int]),
    "ek_fast_mode": (c_int, []),
    "ek_shutdown": (None, []),
    "ek_last_error": (ctypes.c_char_p, []),
    "ek_device_count": (c_int, []),
    "ek_set_device": (c_int, [c_int]),
    "ek_version": (ctypes.c_char_p, []),
    "ek_trace_append": (c_u32, [c_int, c_int, c_u32, c_u32, c_u32, c_u64]),
    "ek_trace_printf": (c_int, [ctypes.c_char_p, c_u32, ctypes.POINTER(c_u32)]),
    "ek_inc_ref_ext": (None, [c_u32]),
    "ek_dec_ref_ext": (None, [c_u32]),
    "ek_var_size": (c_sz, [c_u32]),
    "ek_var_ptr": (c_vp, [c_u32]),
    "ek_var_type": (c_int, [c_u32]),
    "ek_var_set_size": (c_u32, [c_u32, c_sz, c_int]),
    "ek_var_mark_dirty": (c_int, [c_u32]),
    "ek_var_set_label": (c_int, [c_u32, ctypes.c_char_p]),
    "ek_var_mark_side_effect": (c_int, [c_u32]),
    "ek_set_scatter_gather_operand": (c_int, [c_u32, c_int]),
    "ek_var_copy_to_device": (c_u32, [c_int, c_sz, c_vp]),
    "ek_var_register_ptr": (c_u32, [c_vp]),
    "ek_var_register": (c_u32, [c_int, c_sz, c_vp, c_int]),
    "ek_fetch_element": (c_int, [c_vp, c_u32, c_sz, c_sz]),
    "ek_make_managed": (c_int, [c_u32]),
    "ek_eval": (c_int, []),
    "ek_eval_var": (c_int, [c_u32]),
    "ek_sync": (None, []),
    "ek_register_callback": (c_int, [c_vp, c_vp]),
    "ek_unregister_callback": (c_int, [c_vp, c_vp]),
    "ek_set_log_level": (None, [c_u32]),
    "ek_log_level": (c_u32, []),
    "ek_whos": (c_vp, []),
    "ek_hsum": (c_vp, [c_int, c_sz, c_vp]),
    "ek_hprod": (c_vp, [c_int, c_sz, c_vp]),
    "ek_hmax": (c_vp, [c_int, c_sz, c_vp]),
    "ek_hmin": (c_vp, [c_int, c_sz, c_vp]),
    "ek_psum": (c_vp, [c_int, c_sz, c_vp]),
    "ek_count": (c_sz, [c_sz, c_vp]),
    "ek_all": (c_int, [c_sz, c_vp]),
    "ek_any": (c_int, [c_sz, c_vp]),
    "ek_compress": (c_int, [c_int, c_sz, c_vp, c_vp, ctypes.POINTER(c_vp), ctypes.POINTER(c_sz)]),
    "ek_partition": (c_int, [c_sz, c_vp, c_vp, c_vp, c_vp]),
    "ek_fill": (None, [c_vp, c_sz, c_u64, c_sz]),
    "ek_reverse": (None, [c_vp, c_vp, c_sz, c_sz]),
    "ek_malloc": (c_vp, [c_sz]),
    "ek_managed_malloc": (c_vp, [c_sz]),
    "ek_host_malloc": (c_vp, [c_sz]),
    "ek_free": (None, [c_vp]),
    "ek_host_free": (None, [c_vp]),
    "ek_malloc_trim": (None, []),
    "ek_mem_get_info": (None, [ctypes.POINTER(c_sz), ctypes.POINTER(c_sz)]),
    "ek_memcpy_to_device": (None, [c_vp, c_vp, c_sz]),
    "ek_memcpy_to_device_async": (None, [c_vp, c_vp, c_sz]),
    "ek_memcpy_from_device": (None, [c_vp, c_vp, c_sz]),
    "ek_memcpy_from_device_async": (None, [c_vp, c_vp, c_sz]),
    "ek_memcpy_from_device_overlapped": (None, [c_vp, c_vp, c_sz]),
    "ek_memcpy_device_async": (None, [c_vp, c_vp, c_sz]),
    "ek_dlpack_export": (c_vp, [c_u32, c_int, c_vp]),
    "ek_dlpack_import": (c_u32, [c_vp, c_int]),
    "ek_device": (c_int, []),
    "ek_stream_wait_external": (c_int, [c_vp]),
    "ek_stream_signal_external": (c_int, [c_vp]),
    "ek_tape_append_node": (c_u32, [c_int, c_sz, ctypes.c_char_p]),
    "ek_tape_append_leaf": (c_u32, [c_int, c_sz]),
    "ek_tape_append_edge": (c_int, [c_int, c_u32, c_u32, c_u32]),
    "ek_tape_append": (c_u32, [c_int, ctypes.c_char_p, c_sz, c_u32, ctypes.POINTER(c_u32), ctypes.POINTER(c_u32)]),
    "ek_tape_append_gather": (c_u32, [c_int, c_u32, c_u32]),
    "ek_tape_append_scatter": (c_int, [c_int, c_u32, c_u32, c_u32, c_int]),
    "ek_tape_append_psum": (c_u32, [c_int, c_u32]),
    "ek_tape_append_reverse": (c_u32, [c_int, c_u32]),
    "ek_tape_inc_ref_ext": (None, [c_int, c_u32]),
    "ek_tape_dec_ref_ext": (None, [c_int, c_u32]),
    "ek_tape_set_scatter_gather_operand": (c_int, [c_int, ctypes.POINTER(c_u32), c_sz, c_int]),
    "ek_tape_set_gradient": (c_int, [c_int, c_u32, c_u32, c_int]),
    "ek_tape_backward": (c_int, [c_int, c_u32, c_int]),
    "ek_tape_forward": (c_int, [c_int, c_u32, c_int]),
    "ek_tape_backward_static": (c_int, [c_int, c_int]),
    "ek_tape_forward_static": (c_int, [c_int, c_int]),
    "ek_tape_gradient": (c_u32, [c_int, c_u32]),
    "ek_tape_set_label": (c_int, [c_int, c_u32, ctypes.c_char_p]),
    "ek_tape_push_prefix": (None, [c_int, ctypes.c_char_p]),
    "ek_tape_pop_prefix": (c_int, [c_int]),
    "ek_tape_set_log_level": (None, [c_int, c_u32]),
    "ek_tape_set_graph_simplification": (None, [c_int, c_int]),
    "ek_tape_simplify": (c_int, [c_int]),
    "ek_tape_graphviz": (c_vp, [c_int, c_sz, ctypes.POINTER(c_u32)]),
    "ek_tape_whos": (c_vp, [c_int]),
    "ek_tape_node_count": (c_sz, [c_int]),
    "ek_tape_clear": (None, [c_int]),
    "ek_stats_reset": (None, []),
    "ek_stats_get": (None, [ctypes.POINTER(ek_stats)]),
    "ek_set_timing": (None, [c_int]),
    "ek_stream": (c_vp, []),
    "ek_timer_start": (None, []),
    "ek_timer_stop": (ctypes.c_float, []),
    "ek_flush_l2": (None, []),
    # debugging aid (host-only, not part of the reference-facing ABI)
    "ek_debug_plan": (c_vp, []),
    "ek_debug_program": (c_vp, []),
    "ek_debug_discard_side_effects": (None, []),
    "ek_debug_tape_edge_weight": (c_u32, [c_int, c_u32, c_u32]),
}

_lib = None


def load():
    """Load the shared library once and attach prototypes. Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: the CUDA extension is not built. "
            "Run `python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback).")
    lib = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def take_string(ptr):
    """Convert a malloc'd char* returned by the library into str and free() it."""
    if not ptr:
        return None
    s = ctypes.string_at(ptr).decode()
    ctypes.CDLL(None).free(ctypes.c_void_p(ptr))
    return s
