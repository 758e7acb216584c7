"""ctypes binding of include/dlrm_b200.h -- the one and only way Python reaches the kernels.

There is NO fallback: if the shared library is missing (and cannot be built) or a call fails,
a RuntimeError is raised.  Nothing here imports oracle/ or computes on the CPU.
"""
import ctypes as C
import os

from . import _build

MAX_TABLES = 64
ACT_NONE, ACT_RELU, ACT_SIGMOID = 0, 1, 2
LOSS_MSE, LOSS_BCE, LOSS_WBCE = 0, 1, 2
OPT_SGD, OPT_RWSADAGRAD, OPT_ADAGRAD = 0, 1, 2
GEMM_SIMT_FP32, GEMM_TC_BF16X3, GEMM_TC_BF16 = 0, 1, 2
DTYPE_F32, DTYPE_F16, DTYPE_Q8, DTYPE_Q4 = 0, 1, 2, 3
TUNE = dict(emb_bags_per_group=0, emb_unroll=1, head_rows=6, interact_bwd_cols=7, pdl=8, upd_lean=10, upd_debug=11)


class EmbFwdTable(C.Structure):
    _fields_ = [("weight", C.c_void_p), ("indices", C.c_void_p), ("offsets", C.c_void_p),
                ("row_weights", C.c_void_p), ("nnz", C.c_int64), ("rows", C.c_int64), ("ld", C.c_int64),
                ("out_off", C.c_int64), ("out_stride", C.c_int64), ("row_lo", C.c_int64), ("row_n", C.c_int64),
                ("weight_dtype", C.c_int32)]


class EmbBwdTable(C.Structure):
    _fields_ = [("weight", C.c_void_p), ("momentum", C.c_void_p), ("head", C.c_void_p),
                ("indices", C.c_void_p), ("offsets", C.c_void_p), ("nnz", C.c_int64),
                ("rows", C.c_int64), ("pair_base", C.c_int64), ("ld", C.c_int64), ("mom_stride", C.c_int64),
                ("use_dy_off", C.c_int64), ("dy_off", C.c_int64), ("row_lo", C.c_int64), ("row_n", C.c_int64),
                ("head_stride", C.c_int64), ("mark", C.c_void_p), ("weight_dtype", C.c_int32),
                ("round_key", C.c_uint64), ("row_weights", C.c_void_p), ("row_weight_sum", C.c_void_p)]


class EmbRemoteTable(C.Structure):
    _fields_ = [("shard_weight", C.c_void_p * 8), ("num_shards", C.c_int32), ("rows_per_shard", C.c_int64),
                ("rows", C.c_int64), ("ld", C.c_int64), ("indices", C.c_void_p), ("offsets", C.c_void_p),
                ("nnz", C.c_int64), ("out_off", C.c_int64), ("out_stride", C.c_int64), ("weight_dtype", C.c_int32)]


class EmbDedup(C.Structure):
    _fields_ = [("filter", C.c_void_p), ("log2_size", C.c_int32), ("flags", C.c_void_p), ("suspects", C.c_void_p)]


class HostTable(C.Structure):
    _fields_ = [("weight", C.c_void_p), ("momentum", C.c_void_p), ("acc_ew", C.c_void_p), ("indices", C.c_void_p),
                ("offsets", C.c_void_p), ("nnz", C.c_int64), ("rows", C.c_int64), ("pos_base", C.c_int64),
                ("map", C.c_void_p)]


class HostStage(C.Structure):
    _fields_ = [("weight", C.c_void_p), ("momentum", C.c_void_p), ("head", C.c_void_p), ("acc_ew", C.c_void_p),
                ("slot_idx", C.c_void_p), ("list", C.c_void_p), ("key", C.c_void_p), ("count", C.c_void_p),
                ("capacity", C.c_int64), ("ld", C.c_int64), ("head_col", C.c_int64),
                # row cache (all zero: none)
                ("cache_rows", C.c_int64), ("cache_tag", C.c_void_p), ("cache_used", C.c_void_p), ("step", C.c_void_p),
                ("set_head", C.c_void_p), ("set_next", C.c_void_p), ("sets", C.c_void_p), ("num_sets", C.c_void_p),
                ("stats", C.c_void_p), ("forward_only", C.c_int64)]


class GemmTcDesc(C.Structure):
    _fields_ = [("A_hi", C.c_void_p), ("A_lo", C.c_void_p), ("lda", C.c_int64), ("a_mn_major", C.c_int),
                ("B_hi", C.c_void_p), ("B_lo", C.c_void_p), ("ldb", C.c_int64), ("b_mn_major", C.c_int),
                ("M", C.c_int64), ("N", C.c_int64), ("K", C.c_int64),
                ("mode_x3", C.c_int), ("split_k", C.c_int), ("tile_n", C.c_int), ("act", C.c_int),
                ("mask_act", C.c_int),
                ("mask_hi", C.c_void_p), ("mask_lo", C.c_void_p), ("ldmask", C.c_int64),
                ("out_f32", C.c_void_p), ("ld_f32", C.c_int64), ("slab_stride", C.c_int64),
                ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("ld_out", C.c_int64),
                ("outT_hi", C.c_void_p), ("outT_lo", C.c_void_p), ("ld_outT", C.c_int64),
                ("out_col", C.c_void_p), ("col_index", C.c_int64), ("col_slab_stride", C.c_int64),
                ("bias", C.c_void_p), ("tile_m", C.c_int)]


class DenseLayer(C.Structure):
    _fields_ = [("W", C.c_void_p), ("b", C.c_void_p), ("sW", C.c_void_p), ("sb", C.c_void_p),
                ("dW", C.c_void_p), ("db", C.c_void_p), ("pack_hi", C.c_void_p), ("pack_lo", C.c_void_p),
                ("slab_stride", C.c_int64), ("N", C.c_int64), ("K", C.c_int64), ("ld_pack", C.c_int64),
                ("num_slabs", C.c_int64)]


_lib = None

# every symbol include/dlrm_b200.h declares (tests check the .so exports all of them)
SYMBOLS = [
    "dlrm_b200_abi_version", "dlrm_b200_last_error", "dlrm_b200_device_info", "dlrm_b200_check_device_errors",
    "dlrm_b200_emb_bag_fwd", "dlrm_b200_emb_bag_fwd_train", "dlrm_b200_emb_bwd_link",
    "dlrm_b200_emb_bwd_update", "dlrm_b200_head_scratch_bytes", "dlrm_b200_head_fused",
    "dlrm_b200_interact_fwd_ex", "dlrm_b200_interact_bwd_ex", "dlrm_b200_interact_bwd_p2p", "dlrm_b200_act_bwd",
    "dlrm_b200_emb_bag_fwd_p2p", "dlrm_b200_emb_bwd_update_p2p", "dlrm_b200_emb_bwd_classify",
    "dlrm_b200_p2p_barrier", "dlrm_b200_p2p_allreduce_mean", "dlrm_b200_enable_peer_access",
    "dlrm_b200_ipc_export", "dlrm_b200_ipc_open", "dlrm_b200_ipc_close",
    "dlrm_b200_linear_fwd", "dlrm_b200_linear_dgrad", "dlrm_b200_linear_wgrad",
    "dlrm_b200_interact_fwd", "dlrm_b200_interact_bwd", "dlrm_b200_loss_fwd_bwd",
    "dlrm_b200_dense_update",
    "dlrm_b200_gemm_tc_plan_create", "dlrm_b200_gemm_tc_plan_info", "dlrm_b200_gemm_tc_run",
    "dlrm_b200_gemm_tc_plan_destroy",
    "dlrm_b200_emb_bwd_small_scratch_bytes", "dlrm_b200_emb_bwd_small_update", "dlrm_b200_emb_reduce_partials",
    "dlrm_b200_block_copy", "dlrm_b200_gen_multihot", "dlrm_b200_set_tunable", "dlrm_b200_emb_bag_fwd_remote", "dlrm_b200_split_bf16", "dlrm_b200_dense_update_pack",
    "dlrm_b200_decode_records", "dlrm_b200_gather_records", "dlrm_b200_ingest_records",
    "dlrm_b200_host_stage_in", "dlrm_b200_host_write_back", "dlrm_b200_host_release", "dlrm_b200_host_register",
    "dlrm_b200_host_unregister", "dlrm_b200_host_cache_flush",
    "dlrm_b200_emb_bwd_update_lr_dev", "dlrm_b200_emb_bwd_small_update_lr_dev", "dlrm_b200_dense_update_lr_dev",
    "dlrm_b200_dense_update_pack_lr_dev", "dlrm_b200_emb_quantize_rows",
]


def _declare(lib):
    i64, i32, f32, vp = C.c_int64, C.c_int, C.c_float, C.c_void_p
    lib.dlrm_b200_abi_version.restype = i32
    lib.dlrm_b200_last_error.restype = C.c_char_p
    lib.dlrm_b200_set_tunable.argtypes = [i32, i32]
    lib.dlrm_b200_check_device_errors.argtypes = [vp]
    lib.dlrm_b200_device_info.argtypes = [i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    lib.dlrm_b200_emb_bag_fwd.argtypes = [C.POINTER(EmbFwdTable), i32, i32, i64, i32, i32, vp, i64, i64, vp]
    lib.dlrm_b200_emb_bag_fwd_train.argtypes = [C.POINTER(EmbFwdTable), C.POINTER(EmbBwdTable), i32, i32, i64, i32,
                                                i32, vp, vp, i64, i64, C.POINTER(EmbDedup), vp]
    lib.dlrm_b200_emb_bwd_classify.argtypes = [C.POINTER(EmbBwdTable), i32, i64, i32, i32, vp, C.POINTER(EmbDedup), vp]
    lib.dlrm_b200_head_scratch_bytes.argtypes = [i64, i64]
    lib.dlrm_b200_head_fused.argtypes = [vp, i64, vp, vp, vp, vp, i64, i64, i32, i32, i32, f32, vp, vp, vp, vp, vp,
                                         vp, i64, vp, vp, i64, vp, vp]
    lib.dlrm_b200_interact_fwd_ex.argtypes = [vp, i64, vp, i64, vp, vp, i64, i64, i32, i32, i32, vp]
    lib.dlrm_b200_interact_bwd_ex.argtypes = [vp, i64, vp, i64, vp, i64, i64, i32, i32, i32, i32, vp, vp, i64, vp]
    lib.dlrm_b200_emb_bag_fwd_p2p.argtypes = [C.POINTER(EmbFwdTable), C.POINTER(EmbBwdTable), i32, i32, i64, i32, i32,
                                              vp, C.POINTER(vp), i32, i64, i64, i64, C.POINTER(EmbDedup), vp]
    lib.dlrm_b200_emb_bwd_update_p2p.argtypes = [C.POINTER(EmbBwdTable), i32, i32, i64, i32, i32, vp, C.POINTER(vp),
                                                 i32, i64, i64, i64, i32, f32, f32, C.POINTER(EmbDedup), vp]
    lib.dlrm_b200_enable_peer_access.argtypes = [i32, i32]
    lib.dlrm_b200_ipc_export.argtypes = [vp, C.c_char_p, C.POINTER(C.c_int64)]
    lib.dlrm_b200_ipc_open.argtypes = [C.c_char_p, i32, C.POINTER(vp)]
    lib.dlrm_b200_ipc_close.argtypes = [vp]
    lib.dlrm_b200_p2p_barrier.argtypes = [C.POINTER(vp), i32, i32, vp, vp]
    lib.dlrm_b200_p2p_allreduce_mean.argtypes = [C.POINTER(vp), i32, i32, i64, vp]
    lib.dlrm_b200_act_bwd.argtypes = [vp, vp, vp, i64, i32, f32, vp]
    lib.dlrm_b200_emb_bwd_link.argtypes = [C.POINTER(EmbBwdTable), i32, i64, i32, i32, vp, vp]
    lib.dlrm_b200_emb_bwd_update.argtypes = [C.POINTER(EmbBwdTable), i32, i32, i64, i32, i32, vp, vp,
                                             i64, i64, i32, f32, f32, C.POINTER(EmbDedup), vp]
    lib.dlrm_b200_linear_fwd.argtypes = [vp, i64, vp, i64, vp, vp, i64, i64, i64, i64, i32, i32, vp]
    lib.dlrm_b200_linear_dgrad.argtypes = [vp, i64, vp, i64, vp, i64, i32, vp, i64, i64, i64, i64, i32, vp]
    lib.dlrm_b200_linear_wgrad.argtypes = [vp, i64, vp, i64, vp, i64, vp, i64, i64, i64, i32, vp]
    lib.dlrm_b200_interact_fwd.argtypes = [vp, i64, vp, i64, i64, i32, i32, i32, vp]
    lib.dlrm_b200_interact_bwd_p2p.argtypes = [vp, i64, vp, i64, C.POINTER(vp), C.POINTER(i64), C.POINTER(i32), f32, i64,
                                               i32, i32, i32, i32, vp, vp, i64, vp]
    lib.dlrm_b200_interact_bwd.argtypes = [vp, i64, vp, i64, vp, i64, i64, i32, i32, i32, i32, vp]
    lib.dlrm_b200_loss_fwd_bwd.argtypes = [vp, vp, vp, i64, i32, f32, i32, vp, vp, vp, vp]
    lib.dlrm_b200_dense_update.argtypes = [vp, vp, vp, i64, i32, f32, f32, vp]
    lib.dlrm_b200_gemm_tc_plan_create.argtypes = [C.POINTER(GemmTcDesc), C.POINTER(vp)]
    lib.dlrm_b200_gemm_tc_plan_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32),
                                                C.POINTER(i32)]
    lib.dlrm_b200_gemm_tc_run.argtypes = [vp, vp]
    lib.dlrm_b200_emb_bwd_small_scratch_bytes.argtypes = [i64, i32, i64]
    lib.dlrm_b200_emb_bwd_small_update.argtypes = [C.POINTER(EmbBwdTable), i32, i32, i64, i32, i32, vp, C.POINTER(vp), i32,
                                                   i64, i64, i32, f32, f32, vp, i64, vp]
    lib.dlrm_b200_emb_reduce_partials.argtypes = [vp, vp, i64, i64, i32, C.POINTER(i32), C.POINTER(i32), i32, vp]
    lib.dlrm_b200_emb_bag_fwd_remote.argtypes = [C.POINTER(EmbRemoteTable), i32, i32, i64, i32, i32, vp, vp]
    lib.dlrm_b200_block_copy.argtypes = [C.POINTER(vp), C.POINTER(vp), C.POINTER(i64), i32, vp]
    lib.dlrm_b200_gen_multihot.argtypes = [C.POINTER(vp), C.POINTER(i64), C.POINTER(i32), C.POINTER(i32), i32, i32,
                                           C.c_uint64, C.c_uint64, i64, i64, vp, vp, i32, vp]
    lib.dlrm_b200_gemm_tc_plan_destroy.argtypes = [vp]
    lib.dlrm_b200_split_bf16.argtypes = [vp, i64, i64, i64, vp, vp, i64, vp]
    lib.dlrm_b200_dense_update_pack.argtypes = [C.POINTER(DenseLayer), i32, i32, f32, f32, vp]
    lib.dlrm_b200_decode_records.argtypes = [vp, i64, i32, i32, i64, vp, vp, vp, vp, vp]
    lib.dlrm_b200_gather_records.argtypes = [vp, vp, vp, vp, i64, i32, i32, i64, vp, vp, vp, vp, vp]
    lib.dlrm_b200_ingest_records.argtypes = [vp, i32, vp, i32, vp, i32, i64, i32, i32, vp, vp, vp, i64, i64, vp, vp]
    lib.dlrm_b200_host_stage_in.argtypes = [C.POINTER(HostTable), i32, C.POINTER(HostStage), i32, i64, i32, i32, vp]
    lib.dlrm_b200_host_write_back.argtypes = [C.POINTER(HostTable), i32, C.POINTER(HostStage), i32, vp]
    lib.dlrm_b200_host_release.argtypes = [C.POINTER(HostTable), i32, C.POINTER(HostStage), i32, vp]
    lib.dlrm_b200_host_cache_flush.argtypes = [C.POINTER(HostTable), i32, C.POINTER(HostStage), i32, vp]
    lib.dlrm_b200_host_register.argtypes = [vp, i64]
    lib.dlrm_b200_host_unregister.argtypes = [vp]
    lib.dlrm_b200_emb_bwd_update_lr_dev.argtypes = [C.POINTER(EmbBwdTable), i32, i32, i64, i32, i32, vp, vp,
                                                    i64, i64, i32, f32, vp, f32, C.POINTER(EmbDedup), vp]
    lib.dlrm_b200_emb_bwd_small_update_lr_dev.argtypes = [C.POINTER(EmbBwdTable), i32, i32, i64, i32, i32, vp,
                                                          C.POINTER(vp), i32, i64, i64, i32, f32, vp, f32, vp, i64, vp]
    lib.dlrm_b200_dense_update_lr_dev.argtypes = [vp, vp, vp, i64, i32, f32, vp, f32, vp]
    lib.dlrm_b200_dense_update_pack_lr_dev.argtypes = [C.POINTER(DenseLayer), i32, i32, f32, vp, f32, vp]
    lib.dlrm_b200_emb_quantize_rows.argtypes = [vp, i32, i64, i64, i32, vp, i32, i64, vp]
    for name in SYMBOLS:
        fn = getattr(lib, name)
        if name in ("dlrm_b200_head_scratch_bytes", "dlrm_b200_emb_bwd_small_scratch_bytes"):
            fn.restype = i64
        elif name != "dlrm_b200_last_error":
            fn.restype = i32


def lib():
    """Load (building first if the in-tree .so is stale or absent).  Raises on failure."""
    global _lib
    if _lib is None:
        path = _build.LIB
        if not _build.is_fresh():
            if _build.nvcc_path() is not None:
                path = _build.build()
            elif not os.path.exists(path):
                raise RuntimeError(
                    "libdlrm_b200.so is missing and nvcc is unavailable: run "
                    "`python -c 'import __graft_entry__ as g; g.build()'` first. "
                    "dlrm_b200 has no CPU or PyTorch fallback.")
        _lib = C.CDLL(path)
        _declare(_lib)
        if _lib.dlrm_b200_abi_version() != 1:
            raise RuntimeError("libdlrm_b200.so ABI mismatch")
        # experiment knob: DLRM_TUNE="name=value,name=value" (names in TUNE) applied once at load
        for kv in filter(None, os.environ.get("DLRM_TUNE", "").split(",")):
            k, v = kv.split("=")
            if _lib.dlrm_b200_set_tunable(TUNE[k.strip()], int(v)) != 0:
                raise RuntimeError("DLRM_TUNE: " + _lib.dlrm_b200_last_error().decode())
    return _lib


def check(rc, what=""):
    if rc != 0:
        raise RuntimeError(f"libdlrm_b200 {what}: " + lib().dlrm_b200_last_error().decode())


def set_tunable(name, value):
    check(lib().dlrm_b200_set_tunable(TUNE[name], int(value)), "set_tunable")


def device_info(device=0):
    sm, ma, mi = C.c_int(), C.c_int(), C.c_int()
    check(lib().dlrm_b200_device_info(device, C.byref(sm), C.byref(ma), C.byref(mi)), "device_info")
    return sm.value, ma.value, mi.value


class GemmTcPlan:
    """RAII wrapper of a wgmma GEMM plan (TMA descriptors + launch geometry)."""

    def __init__(self, **kw):
        d = GemmTcDesc()
        for k, v in kw.items():
            if not hasattr(d, k):
                raise AttributeError(k)
            setattr(d, k, v)
        self.desc = d
        self.handle = C.c_void_p()
        check(lib().dlrm_b200_gemm_tc_plan_create(C.byref(d), C.byref(self.handle)), "gemm_tc_plan_create")

    def info(self):
        a, b, c, e, m = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int()
        check(lib().dlrm_b200_gemm_tc_plan_info(self.handle, C.byref(a), C.byref(b), C.byref(c), C.byref(e),
                                                C.byref(m)))
        return dict(tile_n=a.value, stages=b.value, splits=c.value, ctas=e.value, tile_m=m.value)

    def run(self, stream):
        check(lib().dlrm_b200_gemm_tc_run(self.handle, stream), "gemm_tc_run")

    def __del__(self):
        try:
            if self.handle:
                lib().dlrm_b200_gemm_tc_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

