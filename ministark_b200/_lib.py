"""ctypes binding of libministark_b200.so (include/ministark_b200.h).

The library is the product: if it is missing or no CUDA device is present, everything here
fails loudly — there is no CPU fallback and nothing from oracle/ is ever imported.
"""
import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MS_LIB_PATH") or os.path.join(_HERE, "libministark_b200.so")   # MS_LIB_PATH: A/B builds
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_b200.h")
STREAM_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_stream.h")
CHECK_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_check.h")
EXTENSION_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_extension.h")
LOOKUP_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_lookup.h")
PERMUTATION_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_permutation.h")
BF_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_bf.h")
DEVICE_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_device.h")
HOST_NODES_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_host_nodes.h")
RESCUE_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_rescue.h")
RESCUE_HASH_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_rescue_hash.h")
RESCUE_MERKLE_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_rescue_merkle.h")
RESCUE_MERKLE_UPDATES_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_rescue_merkle_updates.h")
RESCUE_ROLLUP_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_rescue_rollup.h")
RESCUE_WOTS_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ministark_rescue_wots.h")

u64 = C.c_uint64
vp = C.c_void_p
sz = C.c_size_t
ui = C.c_uint
ci = C.c_int

_SIGS = {
    "ms_ctx_create": (ci, [ci, C.POINTER(vp)]),
    "ms_ctx_destroy": (ci, [vp]),
    "ms_ctx_set_stream": (ci, [vp, vp]),
    "ms_ctx_sync": (ci, [vp]),
    "ms_last_error": (C.c_char_p, [vp]),
    "ms_version": (C.c_char_p, []),
    "ms_launch_count": (u64, [vp]),
    "ms_set_option": (ci, [vp, C.c_char_p, C.c_int64]),
    "ms_alloc_device": (ci, [vp, sz, C.POINTER(vp)]),
    "ms_alloc_host_pinned": (ci, [vp, sz, C.POINTER(vp)]),
    "ms_free": (ci, [vp, vp]),
    "ms_copy": (ci, [vp, vp, vp, sz]),
    "ms_ntt_plan_create": (ci, [vp, ci, ui, ci, u64, C.POINTER(vp)]),
    "ms_ntt_encode": (ci, [vp, vp]),
    "ms_ntt_execute": (ci, [vp]),
    "ms_ntt_plan_destroy": (ci, [vp]),
    "ms_ntt_batch": (ci, [vp, ci, vp, sz, ui, ui, ci, u64]),
    "ms_ntt_batch_to": (ci, [vp, ci, vp, sz, vp, sz, ui, ui, ci, u64]),
    "ms_lde_batch": (ci, [vp, ci, vp, sz, vp, sz, ui, ui, ui, u64, ci]),
    "ms_bit_reverse": (ci, [vp, ci, vp, sz, ui, ui]),
    "ms_pointwise": (ci, [vp, ci, ci, vp, ci, vp, ci, vp, sz, sz, u64]),
    "ms_pointwise_const": (ci, [vp, ci, ci, vp, ci, vp, ci, vp, sz]),
    "ms_sum_columns": (ci, [vp, ci, vp, sz, ui, sz, vp]),
    "ms_hash_rows_sha256": (ci, [vp, ci, vp, sz, ui, sz, vp]),
    "ms_merkle_nodes_sha256": (ci, [vp, vp, sz, vp]),
    "ms_merkle_commit_sha256": (ci, [vp, ci, vp, sz, ui, sz, vp, vp, vp]),
    "ms_merkle_commit_rows_sha256": (ci, [vp, vp, ui, sz, vp, vp, vp]),
    "ms_pow_grind_sha256": (ci, [vp, vp, ui, C.POINTER(u64)]),
    "ms_merkle_prove_sha256": (ci, [vp, vp, vp, sz, vp, ui, vp, vp, vp, vp]),
    "ms_matrix_from_rows": (ci, [vp, ci, vp, sz, ui, vp, sz]),
    "ms_gather_rows": (ci, [vp, ci, vp, sz, ui, sz, vp, ui, vp]),
    "ms_gather_rows_rowmajor": (ci, [vp, vp, ui, sz, vp, ui, vp]),
    "ms_debug_lazy_ops": (ci, [vp, vp, vp, sz, vp]),
    "ms_lde_batch_scatter": (ci, [vp, ci, vp, sz, ui, ui, ui, u64, vp, sz, vp, sz, vp, sz]),
    "ms_ipc_export": (ci, [vp, vp, vp]),
    "ms_ipc_open": (ci, [vp, vp, C.POINTER(vp)]),
    "ms_ipc_close": (ci, [vp, vp]),
    "ms_scan_affine": (ci, [vp, ci, vp, ci, vp, vp, ci, sz, vp, ci, vp]),
    "ms_fri_fold": (ci, [vp, ci, vp, ui, ui, u64, vp, vp]),
    "ms_eval_constraints": (ci, [vp, vp, ui, vp, ui, vp, sz, ui, vp, sz, ui, ci, ui, u64, ci, ci, vp]),
    "ms_eval_constraints_ptrs": (ci, [vp, vp, ui, vp, ui, vp, vp, ui, ci, ui, u64, ci, ci, vp]),
    "ms_eval_jit_check": (ci, [vp, ui, vp, ui, ci, C.c_char_p, sz]),
    "ms_poly_eval": (ci, [vp, ci, vp, sz, ui, sz, vp, ui, vp]),
    "ms_fill_random": (ci, [vp, vp, sz, u64]),
}

# include/ministark_stream.h: the entry points of the streamed prover residency
_STREAM_SIGS = {
    "ms_merkle_commit_block_sha256": (ci, [vp, ci, vp, sz, ui, ui, ui, sz, vp, vp]),
    "ms_lde_rows": (ci, [vp, ci, vp, sz, ui, ui, ui, u64, vp, ui, vp]),
}

# include/ministark_check.h: the constraint check behind the prover's optional validation (validate.py)
_CHECK_SIGS = {
    "ms_check_constraints": (ci, [vp, vp, ui, vp, ui, vp, vp, ui, ci, ui, ui, vp, vp]),
}

# include/ministark_extension.h: extension columns declared by the AIR (air.RunningColumn), built on the device
_EXTENSION_SIGS = {
    "ms_extension_columns": (ci, [vp, vp, ui, vp, ui, vp, vp, ui, ci, ui, ui, vp, vp, vp]),
}

# include/ministark_lookup.h: multiplicity columns of the LogUp lookups an AIR declares (air.Lookup), filled on the device
_LOOKUP_SIGS = {
    "ms_lookup_workspace_bytes": (ci, [ui, ui, ui, C.POINTER(sz)]),
    "ms_lookup_multiplicities": (ci, [vp, vp, ui, vp, ui, vp, vp, ui, ui, ui, ui, vp, sz, vp, vp]),
}

# include/ministark_permutation.h: target columns of the sorted-copy permutations an AIR declares (air.Permutation), filled
# on the device
_PERMUTATION_SIGS = {
    "ms_permutation_workspace_bytes": (ci, [ui, ui, C.POINTER(sz)]),
    "ms_permutation_fill": (ci, [vp, vp, ui, vp, ui, vp, vp, ui, ui, ui, vp, vp, sz]),
}

# include/ministark_bf.h: the execution trace of examples/brainfuck (VM on the host, tables on the device)
_BF_SIGS = {
    "ms_bf_run": (ci, [vp, sz, vp, sz, u64, vp, vp, vp]),
    "ms_bf_trace_sizes": (ci, [vp, vp, sz, vp, sz, vp]),
    "ms_bf_trace_fill": (ci, [vp, vp, sz, vp, sz, vp, vp, vp]),
    "ms_bf_helper_columns": (ci, [vp, vp, sz, vp]),
}

# include/ministark_device.h: free device memory, for sizing a proof before anything is allocated
_DEVICE_SIGS = {
    "ms_device_memory": (ci, [vp, C.POINTER(sz), C.POINTER(sz)]),
}

# include/ministark_host_nodes.h: block subtrees of a streamed commitment copied to pinned host memory
_HOST_NODES_SIGS = {
    "ms_merkle_commit_block_sha256_host": (ci, [vp, ci, vp, sz, ui, ui, vp, vp]),
}

# include/ministark_rescue.h: the trace of examples/rescue (Rescue-Prime permutation chains) built on the device
_RESCUE_SIGS = {
    "ms_rescue_chains": (ci, [vp, vp, u64, u64, vp]),
}

# include/ministark_rescue_hash.h: the trace of examples/rescue's hash claim (the Rescue-Prime sponge over K messages)
_RESCUE_HASH_SIGS = {
    "ms_rescue_hash": (ci, [vp, vp, u64, u64, vp]),
}

# include/ministark_rescue_merkle.h: examples/merkle's Rescue-Prime Merkle tree and authentication-path trace
_RESCUE_MERKLE_SIGS = {
    "ms_rescue_merkle_tree": (ci, [vp, vp, ui, vp]),
    "ms_rescue_merkle_paths": (ci, [vp, vp, ui, vp, u64, vp]),
}

# include/ministark_rescue_merkle_updates.h: the trace of examples/merkle's K ordered leaf writes, and the heap after them
_RESCUE_MERKLE_UPDATES_SIGS = {
    "ms_rescue_merkle_updates": (ci, [vp, vp, ui, vp, vp, u64, vp, vp]),
}

# include/ministark_rescue_rollup.h: the trace of examples/rollup's K balance transfers, and the heap after them
_RESCUE_ROLLUP_SIGS = {
    "ms_rescue_rollup": (ci, [vp, vp, ui, vp, u64, vp, vp]),
}

# include/ministark_rescue_wots.h: examples/wots's K one-time signatures, and the trace that proves them valid
_RESCUE_WOTS_SIGS = {
    "ms_rescue_wots_sign": (ci, [vp, vp, vp, vp, u64, vp, vp]),
    "ms_rescue_wots_trace": (ci, [vp, vp, vp, vp, u64, vp]),
}


def bind(lib, sigs):
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args


def header_symbols(path=HEADER_PATH):
    """every function name declared in include/ministark_b200.h (or in the header at `path`)"""
    text = open(path).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ms_[a-z0-9_]+)\s*\(", text)))


_lib = None


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        bind(lib, _SIGS)
        bind(lib, _STREAM_SIGS)
        bind(lib, _CHECK_SIGS)
        bind(lib, _EXTENSION_SIGS)
        bind(lib, _LOOKUP_SIGS)
        bind(lib, _PERMUTATION_SIGS)
        bind(lib, _BF_SIGS)
        bind(lib, _DEVICE_SIGS)
        bind(lib, _HOST_NODES_SIGS)
        bind(lib, _RESCUE_SIGS)
        bind(lib, _RESCUE_HASH_SIGS)
        bind(lib, _RESCUE_MERKLE_SIGS)
        bind(lib, _RESCUE_MERKLE_UPDATES_SIGS)
        bind(lib, _RESCUE_ROLLUP_SIGS)
        bind(lib, _RESCUE_WOTS_SIGS)
        if b"sm_90a" not in lib.ms_version():      # only the CUDA build is ever used: there is no CPU path in the product
            raise RuntimeError(f"{LIB_PATH} is not the sm_90a build of libministark_b200 ({lib.ms_version()!r})")
        _lib = lib
    return _lib
