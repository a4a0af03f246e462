"""Loads the C-ABI library (vibrato_b200/libvibrato_b200.so) and declares its entry points.

The product path runs exclusively through this library; there is no Python / CPU fallback for the
hot path.  A missing library is a hard error (`build()` compiles it with nvcc for sm_90a).
"""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("VBT_SO") or os.path.join(_HERE, "libvibrato_b200.so")  # VBT_SO: developer override
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "vibrato_b200.h")

VBT_OK = 0
ERR_NAMES = {
    1: "InvalidArgument", 2: "InvalidFormat", 3: "TryFromInt", 4: "ParseInt", 5: "BincodeDecode", 6: "BincodeEncode",
    7: "StdIo", 8: "Utf8", 9: "Unsupported", 10: "ParseFloat", 100: "Cuda", 101: "NoDevice", 102: "Internal",
}


class VibratoError(Exception):
    """Mirror of vibrato::errors::VibratoError (errors.rs:11-42); `.kind` names the variant."""

    def __init__(self, code, msg):
        self.code = code
        self.kind = ERR_NAMES.get(code, str(code))
        super().__init__(f"{self.kind}: {msg}")


def build(verbose=False):
    """Compiles the library in-tree: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo (csrc/Makefile)."""
    cmd = ["make", "-C", os.path.join(_HERE, "csrc"), "-j8"]
    if not verbose:
        cmd.append("-s")
    subprocess.check_call(cmd)
    return SO_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError(
            f"{SO_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(the tokenizer has no fallback path)")
    L = C.CDLL(SO_PATH)
    vp, cp, sz = C.c_void_p, C.c_char_p, C.c_size_t
    u64, u32, i32 = C.c_uint64, C.c_uint32, C.c_int32
    pp = C.POINTER(vp)

    def sig(name, res, args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = args

    sig("vbt_last_error", cp, [])
    sig("vbt_version", cp, [])
    sig("vbt_dict_from_bytes", i32, [vp, sz, pp])
    sig("vbt_dict_from_zstd_file", i32, [cp, pp])
    sig("vbt_dict_from_mecab", i32, [vp, sz, vp, sz, vp, sz, vp, sz, pp])
    sig("vbt_dict_from_parts", i32, [vp, sz, vp, u32, u32, vp, sz, vp, sz, pp])
    sig("vbt_dict_from_bigram", i32, [vp, sz, vp, sz, vp, sz, vp, sz, vp, sz, vp, sz, i32, pp])
    sig("vbt_scorer_accumulate", i32, [vp, sz, vp, vp, sz, C.POINTER(i32)])
    sig("vbt_mecab_generate_bigram_info", i32, [vp, sz, vp, sz, vp, sz, vp, sz, C.c_double] + [pp, C.POINTER(sz)] * 3)
    sig("vbt_dict_write", i32, [vp, pp, C.POINTER(sz)])
    sig("vbt_dict_write_zstd_file", i32, [vp, cp, i32])
    sig("vbt_bytes_free", None, [vp])
    sig("vbt_dict_set_user_lexicon_csv", i32, [vp, vp, sz])
    sig("vbt_dict_free", None, [vp])
    sig("vbt_dict_feature", i32, [vp, u32, pp, C.POINTER(sz)])
    sig("vbt_dict_word_param", i32, [vp, u32, C.POINTER(C.c_uint16), C.POINTER(C.c_uint16), C.POINTER(C.c_int16)])
    sig("vbt_dict_shape", i32, [vp] + [C.POINTER(u32)] * 5)
    sig("vbt_dict_common_prefix", i32, [vp, i32, vp, sz, vp, vp, sz, C.POINTER(sz)])
    sig("vbt_dict_audit", i32, [vp, i32, vp, sz])
    sig("vbt_dict_cate_id", i32, [vp, cp, sz, C.POINTER(i32)])
    sig("vbt_dict_map_connection_ids", i32, [vp, vp, sz, vp, sz])
    sig("vbt_dict_conn_cost", i32, [vp, C.c_uint16, C.c_uint16, C.POINTER(i32)])
    sig("vbt_dict_char_info", i32, [vp, u32, C.POINTER(u32)])
    sig("vbt_connid_counts", i32, [vp, vp, vp, C.POINTER(u32), C.POINTER(u32)])
    sig("vbt_dict_blob_size", i32, [vp, C.POINTER(u64)])
    sig("vbt_dict_pack_blob", i32, [vp, vp, u64])
    sig("vbt_tokenizer_new", i32, [vp, i32, u64, i32, pp])
    sig("vbt_tokenizer_new_from_device_blob", i32, [u64, u64, i32, u64, i32, pp])
    sig("vbt_tokenizer_new_multi", i32, [vp, i32, u64, vp, i32, pp])
    sig("vbt_tokenizer_describe", i32, [vp, vp, sz])
    sig("vbt_pin_thread_to_device", i32, [i32])
    sig("vbt_tokenizer_free", None, [vp])
    sig("vbt_tokenize_batch", i32, [vp, vp, vp, u64, pp])
    sig("vbt_result_view", i32, [vp, pp, pp, C.POINTER(u64), C.POINTER(u64)])
    sig("vbt_result_view_compact", i32, [vp, pp, pp, C.POINTER(u64), C.POINTER(u64)])
    sig("vbt_result_text", i32, [vp, pp, pp, C.POINTER(u64)])
    sig("vbt_evaluate", i32, [vp, vp, vp, sz, vp, sz, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)])
    sig("vbt_result_free", None, [vp])
    sig("vbt_tokenize_batch_device", i32, [vp, u64, u64, u64, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)])
    sig("vbt_host_alloc", i32, [sz, pp])
    sig("vbt_host_free", None, [vp])
    sig("vbt_tokenizer_set_counting", i32, [vp, i32])
    sig("vbt_tokenizer_set_stream", i32, [vp, u64])
    sig("vbt_tokenizer_set_option", i32, [vp, cp, C.c_int64])
    sig("vbt_last_stage_ms", i32, [vp, C.POINTER(C.c_float), i32, C.POINTER(i32)])
    sig("vbt_stage_names", cp, [])
    sig("vbt_last_launch_count", i32, [vp, C.POINTER(u64)])
    sig("vbt_last_counters", i32, [vp, C.POINTER(u64)])
    _lib = L
    return L


def check(rc):
    if rc != VBT_OK:
        raise VibratoError(rc, lib().vbt_last_error().decode("utf-8", "replace"))
