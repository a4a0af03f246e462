"""ctypes binding of oracle/libvibrato_oracle.so — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` legs may
import this module; the product package (vibrato_b200/) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvibrato_oracle.so")

NUM_COUNTERS = 10
COUNTER_NAMES = ["U", "C", "M", "T", "P", "W", "E", "N", "K", "walks"]
# SURVEY.md §8(d): B_alg = U + 4C + 4M + 8T + 4P + 6W + 2E + 20N + 24K
B_ALG_WEIGHTS = np.array([1, 4, 4, 8, 4, 6, 2, 20, 24, 0], dtype=np.uint64)

TOKEN_DTYPE = np.dtype(
    [("start_char", "<u4"), ("end_char", "<u4"), ("start_byte", "<u4"), ("end_byte", "<u4"),
     ("word_idx", "<u4"), ("total_cost", "<i4")]
)
assert TOKEN_DTYPE.itemsize == 24


def build(force=False):
    """Compiles the oracle with the committed Makefile (gcc only)."""
    src = os.path.join(_HERE, "vibrato_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


_libs = {}


def lib(path=None):
    """The oracle library: the committed build, or another build of the same source at `path` (a variant compiled
    with different -D flags, e.g. by tools/lattice_stats.py or the strict-ties test)."""
    so = path or _SO
    if so in _libs:
        return _libs[so]
    if path is None and not os.path.exists(_SO):
        build()
    L = C.CDLL(so)
    vp, cp, sz, u64, u32 = C.c_void_p, C.c_char_p, C.c_size_t, C.c_uint64, C.c_uint32
    L.vo_dict_from_mecab.restype = vp
    L.vo_dict_from_mecab.argtypes = [cp, sz, cp, sz, cp, sz, cp, sz, cp, sz]
    L.vo_dict_from_parts.restype = vp
    L.vo_dict_from_parts.argtypes = [cp, sz, vp, u32, u32, cp, sz, cp, sz, cp, sz]
    L.vo_dict_set_user_csv.restype = C.c_int
    L.vo_dict_set_user_csv.argtypes = [vp, cp, sz, cp, sz]
    L.vo_dict_free.argtypes = [vp]
    L.vo_dict_feature.restype = vp
    L.vo_dict_feature.argtypes = [vp, u32, C.POINTER(sz)]
    L.vo_dict_word_param.restype = C.c_int
    L.vo_dict_word_param.argtypes = [vp, u32, C.POINTER(C.c_uint16), C.POINTER(C.c_uint16), C.POINTER(C.c_int16)]
    L.vo_dict_conn_cost.restype = C.c_int32
    L.vo_dict_conn_cost.argtypes = [vp, C.c_uint16, C.c_uint16]
    L.vo_dict_num_left.restype = u32
    L.vo_dict_num_left.argtypes = [vp]
    L.vo_dict_num_right.restype = u32
    L.vo_dict_num_right.argtypes = [vp]
    L.vo_dict_num_words.restype = u32
    L.vo_dict_num_words.argtypes = [vp, C.c_int]
    L.vo_dict_char_info.restype = u32
    L.vo_dict_char_info.argtypes = [vp, u32]
    L.vo_dict_common_prefix.restype = sz
    L.vo_dict_common_prefix.argtypes = [vp, C.c_int, vp, sz, vp, vp, sz]
    L.vo_worker_new.restype = vp
    L.vo_worker_new.argtypes = [vp, C.c_int, u64, cp, sz]
    L.vo_worker_free.argtypes = [vp]
    L.vo_worker_tokenize.restype = sz
    L.vo_worker_tokenize.argtypes = [vp, cp, sz]
    L.vo_worker_tokenize_counted.restype = sz
    L.vo_worker_tokenize_counted.argtypes = [vp, cp, sz, vp]
    L.vo_worker_tokens.restype = vp
    L.vo_worker_tokens.argtypes = [vp]
    L.vo_tokenize_batch.restype = u64
    L.vo_tokenize_batch.argtypes = [vp, C.c_int, u64, vp, vp, u64, C.c_int, vp, C.POINTER(vp), vp]
    L.vo_benchmark.restype = C.c_double
    L.vo_benchmark.argtypes = [vp, C.c_int, u64, vp, vp, u64, C.c_int, C.c_int, C.POINTER(u64)]
    L.vo_free.argtypes = [vp]
    L.vo_connid_counts_batch.restype = C.c_int
    L.vo_connid_counts_batch.argtypes = [vp, C.c_int, u64, vp, vp, u64, C.c_int, vp, vp]
    L.vo_dict_map_connection_ids.restype = C.c_int
    L.vo_dict_map_connection_ids.argtypes = [vp, vp, sz, vp, sz, cp, sz]
    L.vo_dict_from_bigram.restype = vp
    L.vo_dict_from_bigram.argtypes = [cp, sz, cp, sz, cp, sz, cp, sz, cp, sz, cp, sz, cp, sz]
    L.vo_dict_from_bigram_dual.restype = vp
    L.vo_dict_from_bigram_dual.argtypes = [cp, sz, cp, sz, cp, sz, cp, sz, cp, sz, cp, sz, cp, sz]
    L.vo_scorer_accumulate.restype = C.c_int32
    L.vo_scorer_accumulate.argtypes = [vp, sz, vp, vp, sz]
    L.vo_utf8_valid.restype = C.c_int
    L.vo_utf8_valid.argtypes = [cp, sz]
    _libs[so] = L
    return L


class OracleError(Exception):
    pass


def _b(x):
    return x.encode("utf-8") if isinstance(x, str) else bytes(x)


class OracleDictionary:
    """SystemDictionaryBuilder::from_readers + Dictionary (dictionary/builder.rs:64-89)."""

    def __init__(self, lex_csv, matrix, char_def, unk_def, dual_connector=False, so=None):
        """`matrix`: matrix.def text, an int16 ndarray [num_left, num_right], or a tuple
        (bigram.right, bigram.left, bigram.cost) for from_readers_with_bigram_info (builder.rs:111-148),
        whose `dual_connector` flag picks the Raw or the Dual connector.  `so`: path of another build of the
        oracle library (lib())."""
        self._L = L = lib(so)
        err = C.create_string_buffer(512)
        lex_csv, char_def, unk_def = _b(lex_csv), _b(char_def), _b(unk_def)
        if isinstance(matrix, tuple):
            br, bl, bc = (_b(x) for x in matrix)
            build = L.vo_dict_from_bigram_dual if dual_connector else L.vo_dict_from_bigram
            h = build(lex_csv, len(lex_csv), br, len(br), bl, len(bl), bc, len(bc), char_def,
                      len(char_def), unk_def, len(unk_def), err, 512)
        elif isinstance(matrix, np.ndarray):
            m = np.ascontiguousarray(matrix, dtype=np.int16)
            num_left, num_right = m.shape  # data[left * num_right + right]
            h = L.vo_dict_from_parts(lex_csv, len(lex_csv), m.ctypes.data, num_right, num_left, char_def,
                                     len(char_def), unk_def, len(unk_def), err, 512)
        else:
            matrix = _b(matrix)
            h = L.vo_dict_from_mecab(lex_csv, len(lex_csv), matrix, len(matrix), char_def, len(char_def), unk_def,
                                     len(unk_def), err, 512)
        if not h:
            raise OracleError(err.value.decode("utf-8", "replace"))
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.vo_dict_free(self._h)
            self._h = None

    def set_user_csv(self, csv):
        err = C.create_string_buffer(512)
        if csv is None:
            rc = self._L.vo_dict_set_user_csv(self._h, None, 0, err, 512)
        else:
            csv = _b(csv)
            rc = self._L.vo_dict_set_user_csv(self._h, csv, len(csv), err, 512)
        if rc != 0:
            raise OracleError(err.value.decode("utf-8", "replace"))
        return self

    def feature(self, word_idx):
        n = C.c_size_t()
        p = self._L.vo_dict_feature(self._h, int(word_idx), C.byref(n))
        if not p:
            raise IndexError(word_idx)
        return C.string_at(p, n.value).decode("utf-8")

    def word_param(self, word_idx):
        l, r, c = C.c_uint16(), C.c_uint16(), C.c_int16()
        if self._L.vo_dict_word_param(self._h, int(word_idx), C.byref(l), C.byref(r), C.byref(c)) != 0:
            raise IndexError(word_idx)
        return l.value, r.value, c.value

    def conn_cost(self, right_id, left_id):
        return self._L.vo_dict_conn_cost(self._h, right_id, left_id)

    @property
    def num_left(self):
        return self._L.vo_dict_num_left(self._h)

    @property
    def num_right(self):
        return self._L.vo_dict_num_right(self._h)

    def num_words(self, lex_type=0):
        return self._L.vo_dict_num_words(self._h, lex_type)

    def char_info(self, cp):
        return self._L.vo_dict_char_info(self._h, cp)

    def common_prefix(self, text, lex_type=0):
        chars = np.frombuffer(text.encode("utf-32-le"), dtype=np.uint32)
        cap = 4096
        while True:  # the C side returns the full hit count; a postings list may hold more than `cap`
            ids = np.zeros(cap, dtype=np.uint32)
            ends = np.zeros(cap, dtype=np.uint32)
            n = self._L.vo_dict_common_prefix(self._h, lex_type, chars.ctypes.data, len(chars), ids.ctypes.data,
                                            ends.ctypes.data, cap)
            if n <= cap:
                return [(int(ids[i]), int(ends[i])) for i in range(n)]
            cap = n

    def worker(self, ignore_space=False, max_grouping_len=0):
        return OracleWorker(self, ignore_space, max_grouping_len)

    def tokenize_batch(self, utf8, offsets, ignore_space=False, max_grouping_len=0, n_threads=1, want_tokens=True,
                       want_counters=False):
        """Returns (tok_offsets[n+1] u64, tokens TOKEN_DTYPE[], counters u64[10] or None)."""
        L = self._L
        buf = np.frombuffer(utf8, dtype=np.uint8) if not isinstance(utf8, np.ndarray) else utf8
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(off) - 1
        tok_off = np.zeros(n + 1, dtype=np.uint64)
        toks_p = C.c_void_p()
        cnt = np.zeros(NUM_COUNTERS, dtype=np.uint64) if want_counters else None
        total = L.vo_tokenize_batch(self._h, int(ignore_space), int(max_grouping_len),
                                    buf.ctypes.data if len(buf) else None, off.ctypes.data, n, n_threads,
                                    tok_off.ctypes.data, C.byref(toks_p) if want_tokens else None,
                                    cnt.ctypes.data if want_counters else None)
        toks = None
        if want_tokens:
            nt = int(tok_off[-1])
            assert nt == total
            toks = np.empty(nt, dtype=TOKEN_DTYPE)
            if nt:
                C.memmove(toks.ctypes.data, toks_p.value, nt * TOKEN_DTYPE.itemsize)
            L.vo_free(toks_p)
        return tok_off, toks, cnt

    def connid_counts(self, utf8, offsets, ignore_space=False, max_grouping_len=0, n_threads=1):
        """init_connid_counter + update_connid_counts over the batch -> (lid_count, rid_count) uint64."""
        buf = np.frombuffer(utf8, dtype=np.uint8) if not isinstance(utf8, np.ndarray) else utf8
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        lid = np.zeros(self.num_left, dtype=np.uint64)
        rid = np.zeros(self.num_right, dtype=np.uint64)
        rc = self._L.vo_connid_counts_batch(self._h, int(ignore_space), int(max_grouping_len), buf.ctypes.data,
                                          off.ctypes.data, len(off) - 1, n_threads, lid.ctypes.data, rid.ctypes.data)
        if rc != 0:
            raise OracleError("connid counting failed")
        return lid, rid

    def map_connection_ids(self, lmap, rmap):
        """Dictionary::map_connection_ids_from_iter (dictionary.rs:245-259)."""
        lm = np.ascontiguousarray(lmap, dtype=np.uint16)
        rm = np.ascontiguousarray(rmap, dtype=np.uint16)
        err = C.create_string_buffer(512)
        if self._L.vo_dict_map_connection_ids(self._h, lm.ctypes.data, len(lm), rm.ctypes.data, len(rm), err, 512) != 0:
            raise OracleError(err.value.decode("utf-8", "replace"))
        return self

    def benchmark(self, utf8, offsets, ignore_space=False, max_grouping_len=0, n_threads=1, runs=1):
        """Timed body of benchmark/src/main.rs:53-65; returns (seconds, n_words)."""
        buf = np.frombuffer(utf8, dtype=np.uint8) if not isinstance(utf8, np.ndarray) else utf8
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        nw = C.c_uint64()
        secs = self._L.vo_benchmark(self._h, int(ignore_space), int(max_grouping_len), buf.ctypes.data,
                                  off.ctypes.data, len(off) - 1, n_threads, runs, C.byref(nw))
        return secs, nw.value


class OracleWorker:
    """Tokenizer::new(dict).ignore_space(..)?.max_grouping_len(..).new_worker() (tokenizer.rs:26-84)."""

    def __init__(self, d, ignore_space=False, max_grouping_len=0):
        err = C.create_string_buffer(512)
        self._d = d
        self._L = d._L
        self._h = self._L.vo_worker_new(d._h, int(ignore_space), int(max_grouping_len), err, 512)
        if not self._h:
            raise OracleError(err.value.decode("utf-8", "replace"))
        self._sent = b""
        self._n = 0

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.vo_worker_free(self._h)
            self._h = None

    def tokenize(self, text, counters=None):
        """reset_sentence + tokenize (worker.rs:34-55); returns list of token dicts."""
        s = _b(text)
        self._sent = s
        if counters is not None:
            n = self._L.vo_worker_tokenize_counted(self._h, s, len(s), counters.ctypes.data)
        else:
            n = self._L.vo_worker_tokenize(self._h, s, len(s))
        self._n = n
        arr = np.empty(n, dtype=TOKEN_DTYPE)
        if n:
            C.memmove(arr.ctypes.data, self._L.vo_worker_tokens(self._h), n * TOKEN_DTYPE.itemsize)
        out = []
        for t in arr:
            wi = int(t["word_idx"])
            out.append(dict(
                surface=s[int(t["start_byte"]):int(t["end_byte"])].decode("utf-8"),
                range_char=[int(t["start_char"]), int(t["end_char"])],
                range_byte=[int(t["start_byte"]), int(t["end_byte"])],
                feature=self._d.feature(wi), lex_type=wi >> 30, word_id=wi & 0x3FFFFFFF,
                total_cost=int(t["total_cost"]), word_idx=wi))
        return out


def compute_connid_probs(lid_count, rid_count):
    """ConnIdCounter::compute_probs (mapper.rs:108-146): [(id, prob)] without id 0, by descending
    probability then ascending id."""
    out = []
    for cnt in (lid_count, rid_count):
        total = float(np.sum(cnt, dtype=np.float64))
        probs = [(i, float(c) / total if total else float("nan")) for i, c in enumerate(cnt)][1:]
        probs.sort(key=lambda t: (-t[1], t[0]))
        out.append(probs)
    return out[0], out[1]


def scorer_accumulate(triples, keys1, keys2):
    """ScorerBuilder::insert x n + build + Scorer::accumulate_cost (scorer.rs:110-168, 255-267)."""
    t = np.ascontiguousarray(np.array(triples, dtype=np.int64).astype(np.uint32).reshape(-1))
    k1 = np.ascontiguousarray(keys1, dtype=np.uint32)
    k2 = np.ascontiguousarray(keys2, dtype=np.uint32)
    return lib().vo_scorer_accumulate(t.ctypes.data, len(t) // 3, k1.ctypes.data, k2.ctypes.data, len(k1))


def utf8_valid(b):
    return bool(lib().vo_utf8_valid(b, len(b)))


LEX_TYPE_NAMES = ("System", "User", "Unknown")  # LexType's Debug names (dictionary.rs:30-40)


def format_batch(od, utf8, offsets, tok_off, toks, mode):
    """The output loop of the `tokenize` CLI (tokenize/src/main.rs:83-127) over oracle tokens: returns
    (text_offsets uint64[n + 1], text bytes).  mode: "mecab" | "wakati" | "detail".  Test infrastructure."""
    buf = bytes(memoryview(np.ascontiguousarray(utf8)))
    out = bytearray()
    text_off = np.zeros(len(offsets), dtype=np.uint64)
    feat_cache, param_cache = {}, {}
    for i in range(len(offsets) - 1):
        text_off[i] = len(out)
        base = int(offsets[i])
        a, b = int(tok_off[i]), int(tok_off[i + 1])
        for k in range(a, b):
            t = toks[k]
            w = int(t["word_idx"])
            surface = buf[base + int(t["start_byte"]):base + int(t["end_byte"])]
            if mode == "wakati":
                if k != a:
                    out += b" "
                out += surface
                continue
            if w not in feat_cache:
                feat_cache[w] = od.feature(w).encode("utf-8")
            out += surface + b"\t" + feat_cache[w]
            if mode == "detail":
                if w not in param_cache:
                    param_cache[w] = od.word_param(w)
                l, r, c = param_cache[w]
                out += (f"\tlex_type={LEX_TYPE_NAMES[w >> 30]}\tleft_id={l}\tright_id={r}\tword_cost={c}"
                        f"\ttotal_cost={int(t['total_cost'])}").encode()
            out += b"\n"
        out += b"\n" if mode == "wakati" else b"EOS\n"
    text_off[len(offsets) - 1] = len(out)
    return text_off, bytes(out)


def _csv_row(row):
    """parse_csv_row of the evaluate tool (evaluate/src/main.rs:40-59): csv-core fields of one row."""
    out, cur, i, n = [], [], 0, len(row)
    quoted = False
    at_field_start = True
    while i < n:
        ch = row[i]
        if quoted:
            if ch == '"':
                if i + 1 < n and row[i + 1] == '"':
                    cur.append('"')
                    i += 1
                else:
                    quoted = False
            else:
                cur.append(ch)
        elif ch == '"' and at_field_start:
            quoted = True
        elif ch == ",":
            out.append("".join(cur))
            cur = []
            at_field_start = True
            i += 1
            continue
        else:
            cur.append(ch)
        at_field_start = False
        i += 1
    out.append("".join(cur))
    return out


def evaluate_corpus(od, corpus, feature_indices=(), max_grouping_len=0):
    """The `evaluate` tool's loop (evaluate/src/main.rs:61-138) over oracle tokens: (num_ref, num_sys, num_cor).
    corpus: text in Corpus::from_reader's format (trainer/corpus.rs:78-121).  Test infrastructure."""
    examples, tokens = [], []
    lines = corpus.split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    for line in lines:  # BufRead::lines(): "\n" or "\r\n" terminated
        if line.endswith("\r"):
            line = line[:-1]
        parts = line.split("\t")
        if len(parts) == 2:
            tokens.append((parts[0], parts[1]))
        elif parts == ["EOS"]:
            if "".join(t[0] for t in tokens):
                examples.append(tokens)
            tokens = []
        else:
            raise OracleError("InvalidFormat(rdr): Each line must be a pair of a surface and features or `EOS`")

    def key(rng, feature):
        fields = _csv_row(feature)
        if feature_indices:
            fields = [fields[i] if i < len(fields) else "*" for i in feature_indices]
        return (rng, tuple(fields))

    w = od.worker(ignore_space=False, max_grouping_len=max_grouping_len)
    num_ref = num_sys = num_cor = 0
    for ex in examples:
        refs, start = set(), 0
        for surface, feature in ex:
            refs.add(key((start, start + len(surface)), feature))
            start += len(surface)
        syss = {key(tuple(t["range_char"]), t["feature"]) for t in w.tokenize("".join(s for s, _ in ex))}
        num_ref += len(refs)
        num_sys += len(syss)
        num_cor += len(refs & syss)
    return num_ref, num_sys, num_cor
