"""ctypes binding of libdblink_b200.so (the C ABI in include/dblink_b200.h).

There is no CPU fallback: if the shared library is missing or cannot be built/loaded this module raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("DBL_LIB") or os.path.join(_HERE, "libdblink_b200.so")  # DBL_LIB: experiment builds

OK, ERR_INVALID, ERR_CUDA, ERR_ZERO_MASS, ERR_STATE = 0, -1, -2, -3, -4
PCG_I, PCG_II, GIBBS, GIBBS_SEQ = 0, 1, 2, 3
SAMPLERS = {"PCG-I": PCG_I, "PCG-II": PCG_II, "Gibbs": GIBBS, "Gibbs-Sequential": GIBBS_SEQ}  # ProjectStep.scala:35
MAX_ATTRS = 32
SIM_CONSTANT, SIM_LEVENSHTEIN, SIM_JARO_WINKLER = 0, 1, 2  # DBL_SIM_*

i32p = C.POINTER(C.c_int32)
i64p = C.POINTER(C.c_int64)
u8p = C.POINTER(C.c_uint8)
u64p = C.POINTER(C.c_uint64)
COMM_BLOB_BYTES = 192
f64p = C.POINTER(C.c_double)
vp = C.c_void_p


class ModelDesc(C.Structure):
    _fields_ = [
        ("num_attrs", C.c_int32),
        ("num_files", C.c_int32),
        ("indexes", C.POINTER(vp)),
        ("alpha", f64p),
        ("beta", f64p),
        ("tree", vp),
        ("seed", C.c_uint64),
        ("rank", C.c_int32),
        ("world_size", C.c_int32),
    ]


class SummaryHead(C.Structure):
    _fields_ = [
        ("iteration", C.c_int64),
        ("num_isolates", C.c_int64),
        ("log_likelihood", C.c_double),
        ("pairs_scored", C.c_int64),
    ]


# name -> (restype, argtypes): exactly the entry points declared in include/dblink_b200.h
SIGNATURES = {
    "dbl_index_build": (C.c_int, [C.POINTER(vp), C.POINTER(C.c_char_p), f64p, C.c_int32, C.c_int, C.c_double, C.c_double, C.c_int32]),
    "dbl_index_from_tables": (C.c_int, [C.POINTER(vp), C.c_int32, C.c_int, f64p, i32p, i32p, f64p, C.c_int32]),
    "dbl_index_free": (None, [vp]),
    "dbl_index_num_values": (C.c_int32, [vp]),
    "dbl_index_nnz": (C.c_int32, [vp]),
    "dbl_index_value_id": (C.c_int32, [vp, C.c_char_p]),
    "dbl_index_value": (C.c_char_p, [vp, C.c_int32]),
    "dbl_index_tables": (C.c_int, [vp, f64p, f64p, i32p, i32p, f64p]),
    "dbl_index_base_tables": (C.c_int, [vp, i32p, f64p, f64p, f64p, f64p, f64p]),
    "dbl_index_exp_sim": (C.c_double, [vp, C.c_int32, C.c_int32]),
    "dbl_similarity": (C.c_double, [C.c_int, C.c_char_p, C.c_char_p, C.c_double, C.c_double]),
    "dbl_kdtree_fit": (C.c_int, [C.POINTER(vp), i32p, C.c_int64, C.c_int32, C.c_int32, i32p, C.c_int32]),
    "dbl_kdtree_from_arrays": (C.c_int, [C.POINTER(vp), C.c_int32, i32p, i32p, i32p, i32p, i32p, i32p]),
    "dbl_kdtree_free": (None, [vp]),
    "dbl_kdtree_num_nodes": (C.c_int32, [vp]),
    "dbl_kdtree_num_leaves": (C.c_int32, [vp]),
    "dbl_kdtree_set_len": (C.c_int32, [vp]),
    "dbl_kdtree_export": (C.c_int, [vp, i32p, i32p, i32p, i32p, i32p, i32p]),
    "dbl_kdtree_partition_id": (C.c_int32, [vp, i32p]),
    "dbl_set_device": (C.c_int, [C.c_int32]),
    "dbl_device_count": (C.c_int32, []),
    "dbl_ctx_create": (C.c_int, [C.POINTER(vp), C.POINTER(ModelDesc)]),
    "dbl_ctx_destroy": (None, [vp]),
    "dbl_last_error": (C.c_char_p, [vp]),
    "dbl_set_partitioner": (C.c_int, [vp, vp]),
    "dbl_num_partitions": (C.c_int32, [vp]),
    "dbl_state_init": (C.c_int, [vp, C.c_int64, i32p, i32p, C.c_int64]),
    "dbl_state_upload": (C.c_int, [vp, C.c_int64, C.c_int64, i32p, i32p, u8p, i32p, i32p, f64p, C.c_int64]),
    "dbl_state_download": (C.c_int, [vp, u8p, i32p, i32p, f64p, i32p]),
    "dbl_num_records": (C.c_int64, [vp]),
    "dbl_num_entities": (C.c_int64, [vp]),
    "dbl_iteration": (C.c_int64, [vp]),
    "dbl_chains_init": (C.c_int, [vp, C.c_int32, u64p, C.c_int64, i32p, i32p, C.c_int64]),
    "dbl_chains_upload": (C.c_int, [vp, C.c_int32, u64p, C.c_int64, C.c_int64, i32p, i32p, u8p, i32p, i32p, f64p,
                                    C.c_int64]),
    "dbl_num_chains": (C.c_int32, [vp]),
    "dbl_chains_download": (C.c_int, [vp, u8p, i32p, i32p, f64p, i32p]),
    "dbl_chain_summary": (C.c_int, [vp, C.c_int32, C.POINTER(SummaryHead), i64p, i64p, f64p]),
    "dbl_sweep": (C.c_int, [vp, C.c_int, C.c_int32]),
    "dbl_links_download": (C.c_int, [vp, i32p, i32p]),
    "dbl_summary": (C.c_int, [vp, C.POINTER(SummaryHead), i64p, i64p, f64p]),
    "dbl_set_block_owners": (C.c_int, [vp, i32p]),
    "dbl_block_sweep_begin": (C.c_int, [vp, C.c_int]),
    "dbl_update_block": (C.c_int, [vp, C.c_int32]),
    "dbl_block_sweep_end": (C.c_int, [vp]),
    "dbl_sweep_begin": (C.c_int, [vp, C.c_int, i64p, i64p]),
    "dbl_exchange_pack": (C.c_int, [vp, vp, vp]),
    "dbl_exchange_unpack": (C.c_int, [vp, vp, C.c_int64, vp, C.c_int64]),
    "dbl_sweep_end": (C.c_int, [vp, i64p, C.c_double, C.c_int32]),
    "dbl_summary_words": (C.c_int32, [vp]),
    "dbl_partial_summary": (C.c_int, [vp, i64p, f64p]),
    "dbl_sweep_async": (C.c_int, [vp, C.c_int, C.c_int32]),
    "dbl_sync": (C.c_int, [vp]),
    "dbl_state_hash": (C.c_int, [vp, u64p]),
    "dbl_block_owners": (C.c_int, [vp, i32p]),
    "dbl_comm_export": (C.c_int, [vp, vp]),
    "dbl_comm_import": (C.c_int, [vp, vp, C.c_int32]),
    "dbl_set_rebalance": (C.c_int, [vp, C.c_int32, C.c_double]),
    "dbl_last_exchange": (C.c_int, [vp, i64p, i64p, i64p]),
    "dbl_download_owned": (C.c_int, [vp, i64p, i32p, i32p, i32p, i64p, i32p, i32p, u8p]),
    "dbl_det_log": (C.c_double, [C.c_double]),
    "dbl_det_exp": (C.c_double, [C.c_double]),
    "dbl_draw_theta": (C.c_int, [C.c_int32, C.c_int32, f64p, f64p, C.c_uint64, i64p, i64p, C.c_int64, f64p]),
    "dbl_export_owned_dev": (C.c_int, [vp, vp, vp, vp, vp]),
    "dbl_owned_masks": (C.c_int, [vp, u8p, u8p]),
    "dbl_kernel_launches": (C.c_int64, [vp]),
    "dbl_set_link_mode": (C.c_int, [vp, C.c_int]),
    "dbl_link_kernel": (C.c_int, [vp, C.c_int]),
    "dbl_set_link_mass_capture": (C.c_int, [vp, C.c_int]),
    "dbl_link_mass": (C.c_int, [vp, f64p]),
    "dbl_index_hash_slots": (C.c_int32, [vp]),
    "dbl_index_slot_codes": (C.c_int, [vp, i32p]),
    "dbl_index_pairs_on_device": (C.c_int32, [vp]),
    "dbl_set_graph_mode": (C.c_int, [vp, C.c_int]),
    "dbl_last_sweep_ms": (C.c_double, [vp]),
    "dbl_link_kernel_ms": (C.c_double, [vp, i64p]),
    "dbl_phase_ms": (C.c_int64, [vp, C.POINTER(C.c_double)]),
    "dbl_posterior_create": (C.c_int, [C.POINTER(vp), C.c_int64, C.c_int32]),
    "dbl_posterior_free": (None, [vp]),
    "dbl_posterior_add_sample": (C.c_int, [vp, vp]),
    "dbl_posterior_num_samples": (C.c_int32, [vp]),
    "dbl_posterior_smpc": (C.c_int, [vp, i32p, f64p]),
    "dbl_pairs_create": (C.c_int, [C.POINTER(vp), C.c_int64, C.c_int64]),
    "dbl_pairs_free": (None, [vp]),
    "dbl_pairs_add_sample": (C.c_int, [vp, vp]),
    "dbl_pairs_num_samples": (C.c_int32, [vp]),
    "dbl_pairs_count": (C.c_int, [vp, C.c_int32, i64p]),
    "dbl_pairs_read": (C.c_int, [vp, C.c_int32, vp, vp, vp]),
    "dbl_pairs_score_sample": (C.c_int, [vp, vp, i64p, i64p]),
    "dbl_pairs_binder_search": (C.c_int, [vp, C.c_int64, C.c_int64, vp, C.c_int32, vp, i32p, i32p, i64p, i64p, i64p,
                                          i64p, i64p]),
    "dbl_eval_create": (C.c_int, [C.POINTER(vp), C.c_int64, vp, C.c_int32]),
    "dbl_eval_free": (None, [vp]),
    "dbl_eval_add_sample": (C.c_int, [vp, vp]),
    "dbl_eval_num_samples": (C.c_int32, [vp]),
    "dbl_eval_read": (C.c_int, [vp, i64p, i64p, i64p]),
    "dbl_vi_create": (C.c_int, [C.POINTER(vp), C.c_int64, C.c_int32]),
    "dbl_vi_free": (None, [vp]),
    "dbl_vi_add_sample": (C.c_int, [vp, vp]),
    "dbl_vi_num_samples": (C.c_int32, [vp]),
    "dbl_vi_set_batch_keys": (C.c_int, [vp, C.c_int64]),
    "dbl_vi_cross": (C.c_int, [vp, C.c_int64, vp]),
    "dbl_version": (C.c_char_p, []),
}

_LIB = None


def load(build_if_missing=True):
    """Load libdblink_b200.so; build it in-tree with nvcc when absent/stale.  Raises on failure."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if build_if_missing and (not os.path.exists(SO_PATH) or os.environ.get("DBL_REBUILD") == "1"):
        # the in-tree library travels to the GPU box prebuilt; rebuild only when it is absent (or on request)
        from . import build as _build

        try:
            _build.build(force=True)
        except Exception as e:
            raise RuntimeError(f"libdblink_b200.so is missing and could not be built: {e}") from e
    if not os.path.exists(SO_PATH):
        raise RuntimeError(
            "libdblink_b200.so not found: build it with `python -m dblink_b200.build` (needs nvcc). "
            "dblink_b200 has no CPU fallback."
        )
    lib = C.CDLL(SO_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = the library does not export the declared ABI
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib
