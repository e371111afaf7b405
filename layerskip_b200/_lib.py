"""ctypes binding of liblsk.so — the declarations mirror include/lsk.h one to one.

There is NO fallback: if the shared library is missing the import of the engine fails loudly
(`LskLibraryError`), telling the user to build it.  Nothing here touches `oracle/`.
"""
from __future__ import annotations

import ctypes as C
import os

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LSK_LIB") or os.path.join(PKG_DIR, "liblsk.so")   # LSK_LIB: tuning builds

LSK_MAX_SPEC = 15
LSK_MAX_EOS = 8
LSK_MAX_EXITS = 32
LSK_FLAG_KEEP_LOGITS = 1
LSK_FLAG_NO_PDL = 2
LSK_FLAG_NO_GRAPH = 4
LSK_FLAG_NO_PREFILL_TC = 8
LSK_FLAG_TP_NCCL = 16
LSK_ROPE_DEFAULT, LSK_ROPE_LINEAR, LSK_ROPE_LLAMA3 = 0, 1, 2

(LSK_W_EMBED, LSK_W_FINAL_NORM, LSK_W_LM_HEAD, LSK_W_LN1, LSK_W_Q, LSK_W_K, LSK_W_V, LSK_W_O,
 LSK_W_LN2, LSK_W_GATE, LSK_W_UP, LSK_W_DOWN) = range(12)

LSK_DBG_HIDDEN, LSK_DBG_LOGITS, LSK_DBG_KROW, LSK_DBG_VROW, LSK_DBG_PROBS_DRAFT, \
    LSK_DBG_PROBS_VERIFY, LSK_DBG_RESIDUAL, LSK_DBG_ARGMAX = range(8)


class LskLibraryError(RuntimeError):
    pass


class LskError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"liblsk error {code}: {message}")
        self.code = code


class lsk_config(C.Structure):
    _fields_ = [("vocab", C.c_int32), ("hidden", C.c_int32), ("inter", C.c_int32),
                ("n_layers", C.c_int32), ("n_heads", C.c_int32), ("n_kv_heads", C.c_int32),
                ("head_dim", C.c_int32), ("rms_eps", C.c_float), ("rope_theta", C.c_float),
                ("max_ctx", C.c_int32), ("tp_rank", C.c_int32), ("tp_size", C.c_int32),
                ("attn_splits", C.c_int32), ("flags", C.c_uint32),
                ("rope_scaling", C.c_int32), ("rope_factor", C.c_float),
                ("rope_low_freq_factor", C.c_float), ("rope_high_freq_factor", C.c_float),
                ("rope_original_max_pos", C.c_int32)]


class lsk_weight_desc(C.Structure):
    _fields_ = [("role", C.c_int32), ("layer", C.c_int32), ("data", C.c_void_p),
                ("rows", C.c_int64), ("cols", C.c_int64)]


class lsk_generation(C.Structure):
    _fields_ = [("exit_layer", C.c_int32), ("max_steps", C.c_int32), ("n_eos", C.c_int32),
                ("eos_ids", C.c_int32 * LSK_MAX_EOS), ("sample", C.c_int32),
                ("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float),
                ("no_repeat_ngram_size", C.c_int32), ("seed", C.c_uint64)]


class lsk_round_out(C.Structure):
    _fields_ = [("n_drafted", C.c_int32), ("n_matches", C.c_int32), ("n_emitted", C.c_int32),
                ("kv_len", C.c_int32), ("draft_ids", C.c_int32 * (LSK_MAX_SPEC + 1)),
                ("emitted_ids", C.c_int32 * (LSK_MAX_SPEC + 1)),
                ("verified_ids", C.c_int32 * (LSK_MAX_SPEC + 1))]


class lsk_gemm_plan(C.Structure):
    _fields_ = [("ok", C.c_int32), ("nt", C.c_int32), ("tiles_per_pass", C.c_int32),
                ("n_chunks", C.c_int32), ("chunk_cols", C.c_int32), ("ring_stages", C.c_int32),
                ("stage_bytes", C.c_int32), ("grid", C.c_int32), ("block", C.c_int32),
                ("n_tiles", C.c_int32), ("smem_bytes", C.c_int64), ("smem_limit", C.c_int64)]


class lsk_attn_plan(C.Structure):
    _fields_ = [("ok", C.c_int32), ("n_splits", C.c_int32), ("ring_stages", C.c_int32), ("grid", C.c_int32),
                ("block", C.c_int32), ("row_blocks", C.c_int32), ("kv_refetched_per_row_block", C.c_int32),
                ("smem_bytes", C.c_int64), ("smem_limit", C.c_int64)]


class lsk_memory_plan(C.Structure):
    _fields_ = [("weights", C.c_int64), ("embed", C.c_int64), ("lm_head", C.c_int64), ("kv_pool", C.c_int64),
                ("scratch", C.c_int64), ("total", C.c_int64)]


class lsk_memory_uses(C.Structure):
    _fields_ = [("lm_head_tc", C.c_int32), ("sampling", C.c_int32), ("ngram_ban", C.c_int32),
                ("adaptive", C.c_int32), ("score_exits", C.c_int32), ("accept_exits", C.c_int32),
                ("packed_scoring", C.c_int32), ("tp_peer", C.c_int32), ("batch_seqs", C.c_int32)]


# name -> (restype, argtypes); every symbol include/lsk.h declares
SIGNATURES = {
    "lsk_abi_version": (C.c_int, []),
    "lsk_last_error": (C.c_char_p, []),
    "lsk_create": (C.c_int, [C.POINTER(lsk_config), C.POINTER(C.c_void_p)]),
    "lsk_destroy": (None, [C.c_void_p]),
    "lsk_comm_unique_id": (C.c_int, [C.POINTER(C.c_uint8)]),
    "lsk_comm_init": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint8)]),
    "lsk_load_weights": (C.c_int, [C.c_void_p, C.POINTER(lsk_weight_desc), C.c_int32]),
    "lsk_weights_complete": (C.c_int, [C.c_void_p]),
    "lsk_begin": (C.c_int, [C.c_void_p, C.POINTER(lsk_generation)]),
    "lsk_prefill": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32]),
    "lsk_round": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(lsk_round_out)]),
    "lsk_round_adaptive": (C.c_int, [C.c_void_p, C.c_int32, C.c_float, C.POINTER(lsk_round_out),
                                     C.POINTER(C.c_float)]),
    "lsk_prefill_batch": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32,
                                    C.POINTER(C.c_int32)]),
    "lsk_prefill_batch_seeded": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32,
                                           C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]),
    "lsk_round_batch": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                  C.POINTER(lsk_round_out)]),
    "lsk_round_batch_adaptive": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                           C.c_float, C.POINTER(lsk_round_out), C.POINTER(C.c_float)]),
    "lsk_ar_step": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "lsk_score": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32,
                            C.POINTER(C.c_float), C.POINTER(C.c_int32)]),
    "lsk_score_batch": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32,
                                  C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int32)]),
    "lsk_score_prefixed": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32,
                                     C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                     C.c_int32, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int32)]),
    "lsk_score_exits": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32), C.c_int32,
                                  C.POINTER(lsk_generation), C.POINTER(C.c_float), C.POINTER(C.c_int32),
                                  C.POINTER(C.c_float)]),
    "lsk_kv_len": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "lsk_debug_forward_rows": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32]),
    "lsk_debug_read": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int64,
                                 C.POINTER(C.c_float), C.c_int64]),
    "lsk_debug_set_page_table": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32]),
    "lsk_round_bytes": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_double)]),
    "lsk_ar_bytes": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_double)]),
    "lsk_launch_count": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64)]),
    "lsk_last_device_ms": (C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    "lsk_profile_round": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(lsk_round_out),
                                    C.POINTER(C.c_float), C.POINTER(C.c_int64),
                                    C.POINTER(C.c_float)]),
    "lsk_plan_gemm": (C.c_int, [C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                C.POINTER(lsk_gemm_plan)]),
    "lsk_plan_attention": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                     C.POINTER(lsk_attn_plan)]),
    "lsk_plan_memory": (C.c_int, [C.POINTER(lsk_config), C.c_int32, C.POINTER(lsk_memory_uses),
                                  C.POINTER(lsk_memory_plan)]),
    "lsk_memory_in_use": (C.c_int, [C.c_void_p, C.POINTER(lsk_memory_plan)]),
    "lsk_test_pack": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "lsk_test_gemm": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int32,
                                C.c_void_p, C.c_int32, C.POINTER(C.c_float)]),
    "lsk_test_attn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.c_void_p,
                                C.c_int32, C.POINTER(C.c_float)]),
    "lsk_test_attn_seqs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                     C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32,
                                     C.POINTER(C.c_int32), C.c_void_p]),
    "lsk_test_lmhead_tc": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                     C.c_float, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_int32, C.POINTER(C.c_float)]),
    "lsk_test_logprob": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    "lsk_test_accept": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                  C.POINTER(lsk_generation), C.c_void_p]),
    "lsk_test_draw": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "lsk_test_sample": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(lsk_generation),
                                  C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "lsk_test_accept_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32),
                                         C.POINTER(C.c_int32), C.POINTER(lsk_generation), C.c_int32, C.c_int32,
                                         C.c_int32, C.POINTER(lsk_round_out), C.c_void_p]),
}

_lib = None


def load() -> C.CDLL:
    """Load liblsk.so (once) and type every entry point."""
    global _lib
    if _lib is not None:
        return _lib
    # torch first: liblsk links libnccl.so.2 by soname and must bind to the NCCL build torch
    # already mapped (two different libnccl.so.2 in one process do not mix).
    import torch  # noqa: F401
    if not os.path.exists(LIB_PATH):
        raise LskLibraryError(
            f"{LIB_PATH} not found. The CUDA extension is required (there is no CPU or PyTorch "
            "fallback): build it with `python -m layerskip_b200.build`.")
    try:
        lib = C.CDLL(LIB_PATH)
    except OSError as exc:  # pragma: no cover
        raise LskLibraryError(f"cannot load {LIB_PATH}: {exc}") from exc
    for name, (restype, argtypes) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as exc:
            raise LskLibraryError(f"{LIB_PATH} does not export {name}") from exc
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def check(code: int) -> None:
    if code != 0:
        raise LskError(code, load().lsk_last_error().decode("utf-8", "replace"))
