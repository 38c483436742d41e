"""ctypes binding of libvexb200.so (include/vexb200.h).  Fails loudly if the library is missing:
there is no Python or CPU fallback for any compute entry point."""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libvexb200.so"
HEADER = _HERE.parent / "include" / "vexb200.h"

# enums (mirrors of include/vexb200.h)
OK = 0
ERR_CUDA, ERR_INVALID, ERR_NCCL, ERR_UNSUPPORTED, ERR_NOMEM, ERR_PEER = range(1, 7)
F64, F32, I32, U32, I64, U64 = range(6)
SET, ADD, SUB, MUL, DIV, MOD, AND, OR, XOR, LSH, RSH = range(11)
SUM, SUM_KAHAN, MAX, MIN, MINMAX = range(5)
TERM_VEC, TERM_SCALAR, TERM_INDEX, TERM_DSCALAR, TERM_SPMV, TERM_CCSR, TERM_PTR = range(7)
FMT_AUTO, FMT_CSR, FMT_HELL, FMT_PATTERNS, FMT_SELL = range(5)
FMT_VALUES_F32 = 0x100          # ORed into fmt: double values stored as float, double vectors and sums
MAX_TERMS, MAX_CODE, MAX_STACK, MAX_TEMPS = 16, 64, 12, 8


def PTR(dtype: int) -> int:
    """VEXB_PTR(dtype): the type of a pointer to `dtype` elements (a user function's pointer parameter)."""
    return dtype | 0x10


_OPS = ("TERM CVT NEG LNOT ADD SUB MUL DIV MOD BAND BOR BXOR SHL SHR LT GT LE GE EQ NE LAND LOR SELECT "
        "SIN COS TAN ASIN ACOS ATAN SINH COSH TANH EXP EXP2 LOG LOG2 LOG10 SQRT RSQRT CBRT FABS FLOOR CEIL "
        "ROUND TRUNC POW ATAN2 FMOD HYPOT FMIN FMAX FMA CALL TDEF TREF LOAD").split()
OP = {name: i for i, name in enumerate(_OPS)}


class TermValue(C.Union):
    _fields_ = [("ptr", C.c_void_p), ("f64", C.c_double), ("f32", C.c_float), ("i32", C.c_int32),
                ("u32", C.c_uint32), ("i64", C.c_int64), ("u64", C.c_uint64)]


class Term(C.Structure):
    _fields_ = [("kind", C.c_uint8), ("dtype", C.c_uint8), ("pad", C.c_uint8 * 6), ("v", TermValue)]


class Instr(C.Structure):
    _fields_ = [("op", C.c_uint8), ("type", C.c_uint8), ("arg", C.c_uint16)]


class Expr(C.Structure):
    _fields_ = [("n_terms", C.c_int32), ("n_code", C.c_int32), ("term", Term * MAX_TERMS), ("code", Instr * MAX_CODE)]


class DevProps(C.Structure):
    _fields_ = [("name", C.c_char * 256), ("cc_major", C.c_int32), ("cc_minor", C.c_int32), ("sm_count", C.c_int32),
                ("max_threads_per_block", C.c_int32), ("warp_size", C.c_int32), ("pad", C.c_int32),
                ("smem_per_block_optin", C.c_size_t), ("total_mem", C.c_size_t), ("l2_bytes", C.c_size_t)]


class SpmatInfo(C.Structure):
    _fields_ = [("nrows", C.c_size_t), ("ncols", C.c_size_t), ("nnz", C.c_size_t), ("fmt", C.c_int32),
                ("val_dtype", C.c_int32), ("ell_width", C.c_size_t), ("ell_pitch", C.c_size_t),
                ("csr_tail_nnz", C.c_size_t), ("n_tiles", C.c_size_t), ("tile_nnz", C.c_size_t),
                ("device_bytes", C.c_size_t), ("ell_col_bytes", C.c_int32),
                ("ell_classes", C.c_int32), ("val_bytes", C.c_int32)]


class BspmatInfo(C.Structure):
    _fields_ = [("nrows", C.c_size_t), ("ncols", C.c_size_t), ("nnzb", C.c_size_t), ("block", C.c_int32),
                ("val_dtype", C.c_int32), ("n_slices", C.c_size_t), ("n_slots", C.c_size_t), ("device_bytes", C.c_size_t)]


class ZspmatInfo(C.Structure):
    _fields_ = [("nrows", C.c_size_t), ("ncols", C.c_size_t), ("nnz", C.c_size_t), ("val_dtype", C.c_int32),
                ("n_slices", C.c_size_t), ("n_slots", C.c_size_t), ("device_bytes", C.c_size_t)]


class UsrmatInfo(C.Structure):
    _fields_ = [("nrows", C.c_size_t), ("ncols", C.c_size_t), ("nnz", C.c_size_t), ("val_bytes", C.c_int32),
                ("n_slices", C.c_size_t), ("n_slots", C.c_size_t), ("device_bytes", C.c_size_t)]


class UsrOps(C.Structure):
    _fields_ = [("val_type", C.c_char_p), ("rhs_type", C.c_char_p), ("rhs_bytes", C.c_size_t),
                ("decl", C.c_char_p), ("product", C.c_char_p), ("append", C.c_char_p)]


class CcsrInfo(C.Structure):
    _fields_ = [("nrows", C.c_size_t), ("unique_rows", C.c_size_t), ("nnz", C.c_size_t), ("idx_bytes", C.c_int32),
                ("table_in_smem", C.c_int32), ("device_bytes", C.c_size_t)]


class DspmatInfo(C.Structure):
    _fields_ = [("nrows", C.c_size_t), ("ncols_local", C.c_size_t), ("n_ghost", C.c_size_t), ("n_send", C.c_size_t),
                ("loc_nnz", C.c_size_t), ("rem_nnz", C.c_size_t), ("loc", SpmatInfo), ("rem", SpmatInfo)]


class VexbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"vexb error {code}: {msg}")
        self.code = code


def declared_symbols() -> list[str]:
    """Every function name declared in include/vexb200.h."""
    text = HEADER.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vexb_[a-z0-9_]+)\s*\(", text)))


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
    L = C.CDLL(str(LIB_PATH))
    vp, sz, i, d = C.c_void_p, C.c_size_t, C.c_int, C.c_double
    P = C.POINTER
    sig = {
        "vexb_abi_version": ([], i),
        "vexb_last_error": ([], C.c_char_p),
        "vexb_init": ([], i), "vexb_shutdown": ([], i),
        "vexb_device_count": ([P(i)], i),
        "vexb_device_props": ([i, P(DevProps)], i),
        "vexb_set_param": ([C.c_char_p, C.c_long], i),
        "vexb_get_param": ([C.c_char_p, P(C.c_long)], i),
        "vexb_launch_count": ([P(C.c_uint64)], i),
        "vexb_stream_create": ([i, P(vp)], i), "vexb_stream_destroy": ([i, vp], i),
        "vexb_stream_sync": ([i, vp], i), "vexb_device_sync": ([i], i),
        "vexb_event_create": ([i, P(vp)], i), "vexb_event_destroy": ([i, vp], i),
        "vexb_event_record": ([i, vp, vp], i), "vexb_event_sync": ([i, vp], i),
        "vexb_stream_wait_event": ([i, vp, vp], i),
        "vexb_event_elapsed_ms": ([vp, vp, P(C.c_float)], i),
        "vexb_malloc": ([i, sz, P(vp)], i), "vexb_free": ([i, vp], i),
        "vexb_host_alloc": ([sz, P(vp)], i), "vexb_host_free": ([vp], i),
        "vexb_h2d": ([i, vp, vp, sz, vp, i], i), "vexb_d2h": ([i, vp, vp, sz, vp, i], i),
        "vexb_d2d": ([i, vp, vp, sz, vp], i), "vexb_memset": ([i, vp, i, sz, vp], i),
        "vexb_partition": ([sz, i, P(d), P(sz)], i),
        "vexb_eval": ([i, vp, vp, i, i, P(Expr), sz, sz], i),
        "vexb_eval_multi": ([i, vp, i, P(vp), i, i, P(P(Expr)), sz, sz, P(i)], i),
        "vexb_eval_path": ([i, i, P(Expr), C.c_char_p, sz], i),
        "vexb_function_register": ([C.c_char_p, i, i, P(i), C.c_char_p, P(i)], i),
        "vexb_jit_source": ([i, i, P(Expr), C.c_char_p, P(sz), i], i),
        "vexb_jit_source_multi": ([i, i, i, P(P(Expr)), C.c_char_p, P(sz), i], i),
        "vexb_jit_source_reduce": ([i, i, P(i), P(Expr), C.c_char_p, P(sz), i], i),
        "vexb_function_register_ex": ([C.c_char_p, i, i, P(i), C.c_char_p, i, P(i), C.c_char_p, P(i)], i),
        "vexb_program_header_push": ([i, C.c_char_p], i),
        "vexb_program_header_pop": ([i], i),
        "vexb_program_header_get": ([i, C.c_char_p, P(sz)], i),
        "vexb_jit_source_dev": ([i, i, i, P(Expr), C.c_char_p, P(sz), i], i),
        "vexb_jit_source_multi_dev": ([i, i, i, i, P(P(Expr)), C.c_char_p, P(sz), i], i),
        "vexb_jit_source_reduce_dev": ([i, i, i, P(i), P(Expr), C.c_char_p, P(sz), i], i),
        "vexb_reduce_workspace_bytes": ([i, P(sz)], i),
        "vexb_reduce": ([i, vp, P(Expr), i, sz, sz, i, vp, vp], i),
        "vexb_reduce_identity": ([i, vp, i, i, vp], i),
        "vexb_reduce_fetch": ([i, vp, vp, i, i, vp], i),
        "vexb_comm_unique_id": ([vp], i),
        "vexb_comm_create_rank": ([i, i, i, vp, P(vp)], i),
        "vexb_comm_create_all": ([i, P(i), P(vp)], i),
        "vexb_comm_destroy": ([vp], i),
        "vexb_comm_rank": ([vp, P(i), P(i), P(i)], i),
        "vexb_comm_allreduce": ([i, P(vp), P(vp), P(vp), i, i, i], i),
        "vexb_comm_barrier": ([i, P(vp), P(vp)], i),
        "vexb_graph_begin": ([i, vp], i), "vexb_graph_end": ([i, vp, P(vp)], i),
        "vexb_graph_launch": ([vp, vp], i), "vexb_graph_destroy": ([vp], i),
        "vexb_peer_create": ([i, i, i, P(vp), vp], i), "vexb_peer_connect": ([vp, vp], i),
        "vexb_peer_create_all": ([i, P(i), P(vp)], i), "vexb_peer_destroy": ([vp], i),
        "vexb_peer_error": ([vp, P(C.c_uint64)], i),
        "vexb_peer_allreduce": ([vp, vp, vp, i, i], i),
        "vexb_reduce_all": ([i, vp, P(Expr), i, sz, sz, i, vp, vp, vp], i),
        "vexb_strip_ghost_cols": ([sz, vp, i, vp, i, sz, sz, vp, P(sz)], i),
        "vexb_halo_plan_create": ([i, P(sz), vp, P(sz), P(vp)], i),
        "vexb_halo_plan_destroy": ([vp], i),
        "vexb_halo_plan_ref_sizes": ([vp, P(sz)], i),
        "vexb_halo_plan_ref_tables": ([vp, vp, P(sz)], i),
        "vexb_halo_plan_ref_recv": ([vp, i, vp], i),
        "vexb_halo_plan_counts": ([vp, i, P(sz), P(sz)], i),
        "vexb_halo_plan_send_cols": ([vp, i, vp], i),
        "vexb_csr_create": ([i, vp, sz, sz, vp, i, vp, i, vp, i, i, P(vp)], i),
        "vexb_csr_row_patterns": ([sz, vp, i, vp, i, vp, i, sz, P(sz), vp], i),
        "vexb_csr_sell_layout": ([sz, vp, i, C.c_long, P(sz), P(sz), vp, vp], i),
        "vexb_spmat_destroy": ([vp], i),
        "vexb_spmat_get_info": ([vp, P(SpmatInfo)], i),
        "vexb_spmat_hell_download": ([vp, vp, vp, vp, vp, vp], i),
        "vexb_spmv": ([i, vp, vp, vp, vp, d, i], i),
        "vexb_bsr_create": ([i, vp, sz, sz, i, vp, i, vp, i, vp, i, P(vp)], i),
        "vexb_bspmat_destroy": ([vp], i),
        "vexb_bspmat_get_info": ([vp, P(BspmatInfo)], i),
        "vexb_bspmv": ([i, vp, vp, vp, vp, d, i], i),
        "vexb_zsr_create": ([i, vp, sz, sz, vp, i, vp, i, vp, i, P(vp)], i),
        "vexb_zspmat_destroy": ([vp], i),
        "vexb_zspmat_get_info": ([vp, P(ZspmatInfo)], i),
        "vexb_zspmv": ([i, vp, vp, vp, vp, d, i], i),
        "vexb_usr_create": ([i, vp, sz, sz, vp, i, vp, i, vp, i, P(vp)], i),
        "vexb_usrmat_destroy": ([vp], i),
        "vexb_usrmat_get_info": ([vp, P(UsrmatInfo)], i),
        "vexb_usr_spmv": ([i, vp, vp, P(UsrOps), vp, vp, i], i),
        "vexb_jit_source_usr": ([P(UsrOps), i, C.c_char_p, P(sz), i], i),
        "vexb_ccsr_create": ([i, vp, sz, sz, vp, i, vp, i, vp, i, vp, i, P(vp)], i),
        "vexb_ccsr_destroy": ([vp], i),
        "vexb_ccsr_get_info": ([vp, P(CcsrInfo)], i),
        "vexb_ccsr_spmv": ([i, vp, vp, vp, vp, d, i], i),
        "vexb_ccsr_jit_source": ([sz, vp, vp, vp, i, i, C.c_char_p, P(sz), i], i),
        "vexb_stencil_apply": ([i, vp, i, vp, i, i, vp, sz, vp, vp, vp, d, i], i),
        "vexb_copy_peer": ([i, vp, i, vp, sz, vp], i),
        "vexb_stencil_operator_register": ([i, i, i, C.c_char_p, P(i)], i),
        "vexb_stencil_operator_source": ([i, C.c_char_p, P(sz), i], i),
        "vexb_stencil_operator_apply": ([i, vp, i, vp, sz, vp, vp, vp, d, i], i),
        "vexb_dspmat_create": ([i, vp, i, vp, sz, vp, i, vp, i, vp, i, i, P(vp)], i),
        "vexb_dspmat_destroy": ([vp], i),
        "vexb_dspmat_get_info": ([vp, P(DspmatInfo)], i),
        "vexb_dspmat_download_split": ([vp, vp, vp, vp, vp, vp, vp], i),
        "vexb_dspmat_send_buffer": ([vp], vp),
        "vexb_dspmat_ghost_buffer": ([vp], vp),
        "vexb_dspmat_pack": ([vp, vp, vp], i),
        "vexb_dspmat_mul_local": ([vp, vp, vp, vp, d, i], i),
        "vexb_dspmat_mul_remote": ([vp, vp, vp, d], i),
        "vexb_halo_exchange": ([i, P(vp), P(vp), P(vp)], i),
        "vexb_dspmat_apply": ([i, P(vp), P(vp), P(vp), P(vp), P(vp), d, i], i),
        "vexb_dspmat_halo_handle": ([vp, vp], i), "vexb_dspmat_halo_connect": ([vp, vp], i),
        "vexb_dspmat_halo_connect_local": ([i, P(vp)], i), "vexb_dspmat_halo_connected": ([vp, P(i)], i),
        "vexb_dspmat_halo_disconnect": ([vp], i),
        "vexb_dspmat_apply_dot": ([i, P(vp), P(vp), P(vp), P(vp), d, i, P(vp), P(vp), P(vp)], i),
        "vexb_peer_fault": ([P(C.c_uint64), i], i),
        "vexb_dspmat_inline_strip": ([vp, P(vp)], i),
        "vexb_dspmat_sweep_strip": ([vp, P(vp)], i),
        "vexb_spmv_multi": ([i, vp, vp, i, P(vp), P(vp), d, i], i),
        "vexb_dspmat_apply_multi": ([i, P(vp), P(vp), P(vp), i, P(vp), P(vp), d, i], i),
        "vexb_jit_pending": ([P(i)], i),
        "vexb_jit_precompile": ([i, i, P(Expr), i], i),
        "vexb_reduce_multi": ([i, vp, P(Expr), i, sz, sz, i, P(i), vp, vp, vp], i),
        "vexb_cg_update_r": ([i, vp, i, sz, vp, vp, vp, vp, vp, vp, vp], i),
        "vexb_cg_update_xp": ([i, vp, i, sz, vp, vp, vp, vp, vp, vp], i),
        "vexb_sort_workspace_bytes": ([sz, i, i, P(sz)], i),
        "vexb_sort": ([i, vp, vp, i, vp, i, sz, i, vp, sz], i),
        "vexb_sort_merge": ([i, P(sz), vp, i, vp, i, i, vp, vp], i),
        "vexb_scan_workspace_bytes": ([sz, i, P(sz)], i),
        "vexb_scan": ([i, vp, vp, vp, i, sz, i, vp, vp, sz], i),
        "vexb_scan_by_key": ([i, vp, vp, i, vp, vp, i, sz, i, vp, vp, sz], i),
        "vexb_reduce_by_key_count": ([i, vp, vp, i, vp, i, sz, vp, sz, P(sz)], i),
        "vexb_reduce_by_key_write": ([i, vp, vp, i, vp, i, sz, vp, vp, vp, sz], i),
    }
    for name, (args, res) in sig.items():
        fn = getattr(L, name)          # AttributeError here == the library does not export a declared symbol
        fn.argtypes = args
        fn.restype = res
    L._signatures = sig
    _lib = L
    return L


def check(code: int):
    if code != OK:
        raise VexbError(code, lib().vexb_last_error().decode(errors="replace"))
