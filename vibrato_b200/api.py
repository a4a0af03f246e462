"""Host-side mirror of vibrato's public API over the C ABI (include/vibrato_b200.h).

Names, argument meaning and error behaviour follow the reference so that its tests read the same
here (paths relative to /root/reference/vibrato/src/):

    Dictionary.read / SystemDictionaryBuilder.from_readers / reset_user_lexicon_from_reader
                                               dictionary.rs:173,209 ; dictionary/builder.rs:64
    Tokenizer(dict).ignore_space(b).max_grouping_len(n).new_worker()   tokenizer.rs:26-84
    Worker.reset_sentence / tokenize / num_tokens / token / token_iter worker.rs:34-74
    Token.surface / feature / range_char / range_byte / word_idx / lex_type /
          left_id / right_id / word_cost / total_cost                  token.rs:21-92
    generate_bigram_info                                               mecab.rs:31-181

plus the batched entry point the GPU wants: Tokenizer.tokenize_batch(list_of_str) -> BatchResult.
All tokenisation runs in the CUDA library; nothing here computes a lattice.
"""
import ctypes as C

import numpy as np

from . import _native
from ._native import VibratoError, check, lib

TOKEN_DTYPE = np.dtype(
    [("start_char", "<u4"), ("end_char", "<u4"), ("start_byte", "<u4"), ("end_byte", "<u4"),
     ("word_idx", "<u4"), ("total_cost", "<i4")]
)
LEX_TYPE_NAMES = ("System", "User", "Unknown")  # dictionary.rs:30-40 (Debug names used by tokenize -O detail)


def _buf(x):
    """bytes-like -> (ctypes address holder, length)."""
    if isinstance(x, str):
        x = x.encode("utf-8")
    if isinstance(x, np.ndarray):
        x = np.ascontiguousarray(x)
        return x, x.ctypes.data, x.nbytes
    b = bytes(x)
    return b, C.cast(C.c_char_p(b), C.c_void_p).value if b else None, len(b)


class WordIdx:
    """dictionary/word_idx.rs:5-11"""

    __slots__ = ("lex_type", "word_id")

    def __init__(self, lex_type, word_id):
        self.lex_type = lex_type
        self.word_id = word_id

    @property
    def packed(self):
        return (self.lex_type << 30) | self.word_id

    def __eq__(self, o):
        return (self.lex_type, self.word_id) == (o.lex_type, o.word_id)

    def __repr__(self):
        return f"WordIdx({LEX_TYPE_NAMES[self.lex_type]}, {self.word_id})"


class Dictionary:
    """vibrato::Dictionary (dictionary.rs:54-56)."""

    def __init__(self, handle):
        self._h = handle
        self._free = lib().vbt_dict_free  # bound now: module globals may be gone at interpreter exit

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._free(h)

    @staticmethod
    def read(data):
        """Dictionary::read (dictionary.rs:173): `data` is the zstd-decoded `.dic` stream."""
        keep, p, n = _buf(data)
        h = C.c_void_p()
        check(lib().vbt_dict_from_bytes(p, n, C.byref(h)))
        return Dictionary(h)

    @staticmethod
    def from_zstd_file(path):
        h = C.c_void_p()
        check(lib().vbt_dict_from_zstd_file(str(path).encode(), C.byref(h)))
        return Dictionary(h)

    def write(self):
        """Dictionary::write (dictionary.rs:142-150) -> bytes."""
        p, n = C.c_void_p(), C.c_size_t()
        check(lib().vbt_dict_write(self._h, C.byref(p), C.byref(n)))
        try:
            return C.string_at(p, n.value)
        finally:
            lib().vbt_bytes_free(p)

    def write_zstd_file(self, path, level=19):
        """Dictionary::write into zstd::Encoder::new(File::create(path), level) (compile/src/main.rs:98-100): the
        `system.dic.zst` that from_zstd_file and every tool's -i read.  A failed write leaves no file behind."""
        check(lib().vbt_dict_write_zstd_file(self._h, str(path).encode(), int(level)))
        return self

    def reset_user_lexicon_from_reader(self, user_lexicon):
        """Dictionary::reset_user_lexicon_from_reader (dictionary.rs:209-229); None clears it."""
        if user_lexicon is None:
            check(lib().vbt_dict_set_user_lexicon_csv(self._h, None, 0))
        else:
            keep, p, n = _buf(user_lexicon)
            check(lib().vbt_dict_set_user_lexicon_csv(self._h, p if n else C.cast(C.c_char_p(b""), C.c_void_p), n))
        return self

    def word_feature(self, word_idx):
        """Dictionary::word_feature (dictionary.rs:108-114)."""
        wi = word_idx.packed if isinstance(word_idx, WordIdx) else int(word_idx)
        p, n = C.c_void_p(), C.c_size_t()
        check(lib().vbt_dict_feature(self._h, wi, C.byref(p), C.byref(n)))
        return C.string_at(p, n.value).decode("utf-8")

    def word_param(self, word_idx):
        """Dictionary::word_param (dictionary.rs:98-104) -> (left_id, right_id, word_cost)."""
        wi = word_idx.packed if isinstance(word_idx, WordIdx) else int(word_idx)
        l, r, c = C.c_uint16(), C.c_uint16(), C.c_int16()
        check(lib().vbt_dict_word_param(self._h, wi, C.byref(l), C.byref(r), C.byref(c)))
        return l.value, r.value, c.value

    def shape(self):
        v = [C.c_uint32() for _ in range(5)]
        check(lib().vbt_dict_shape(self._h, *[C.byref(x) for x in v]))
        return dict(zip(("num_left", "num_right", "n_system", "n_user", "n_unknown"), (x.value for x in v)))

    def map_connection_ids_from_iter(self, lmap, rmap):
        """Dictionary::map_connection_ids_from_iter (dictionary.rs:245-259)."""
        lm = np.ascontiguousarray(list(lmap), dtype=np.uint16)
        rm = np.ascontiguousarray(list(rmap), dtype=np.uint16)
        check(lib().vbt_dict_map_connection_ids(self._h, lm.ctypes.data if len(lm) else None, len(lm),
                                                rm.ctypes.data if len(rm) else None, len(rm)))
        return self

    def conn_cost(self, right_id, left_id):
        c = C.c_int32()
        check(lib().vbt_dict_conn_cost(self._h, right_id, left_id, C.byref(c)))
        return c.value

    def char_info(self, code_point):
        v = C.c_uint32()
        check(lib().vbt_dict_char_info(self._h, code_point, C.byref(v)))
        return v.value

    def cate_id(self, name):
        i = C.c_int32()
        b = name.encode()
        check(lib().vbt_dict_cate_id(self._h, b, len(b), C.byref(i)))
        return None if i.value < 0 else i.value

    def common_prefix(self, text, lex_type=0):
        """Lexicon::common_prefix_iterator (lexicon.rs:33-46) on the host copy -> [(word_id, end_char)]."""
        chars = np.array([ord(c) for c in text], dtype=np.uint32)
        cap = 1 << 14
        ids = np.zeros(cap, dtype=np.uint32)
        ends = np.zeros(cap, dtype=np.uint32)
        n = C.c_size_t()
        check(lib().vbt_dict_common_prefix(self._h, lex_type, chars.ctypes.data, len(chars), ids.ctypes.data,
                                           ends.ctypes.data, cap, C.byref(n)))
        return [(int(ids[i]), int(ends[i])) for i in range(min(n.value, cap))]

    def audit(self, lex_type=0):
        """vbt_dict_audit: {keys, words, listed, longest_key, keys_not_found, words_unlisted_or_twice}."""
        out = np.zeros(6, dtype=np.uint64)
        check(lib().vbt_dict_audit(self._h, lex_type, out.ctypes.data, 6))
        return dict(zip(("keys", "words", "listed", "longest_key", "keys_not_found", "words_unlisted_or_twice"),
                        (int(x) for x in out)))

    def pack_blob(self, out=None):
        """Packed device image (host bytes) for upload / NCCL broadcast."""
        n = C.c_uint64()
        check(lib().vbt_dict_blob_size(self._h, C.byref(n)))
        if out is None:
            out = np.empty(n.value, dtype=np.uint8)
        assert out.nbytes == n.value
        check(lib().vbt_dict_pack_blob(self._h, out.ctypes.data, n.value))
        return out


class SystemDictionaryBuilder:
    """vibrato::SystemDictionaryBuilder (dictionary/builder.rs:12-89)."""

    @staticmethod
    def from_readers(system_lexicon, connector, char_prop, unk_handler):
        """from_readers(lex.csv, matrix.def, char.def, unk.def). `connector` may also be an int16
        ndarray [num_left, num_right] (MatrixConnector::new) for dictionaries too big for text."""
        k1, p1, n1 = _buf(system_lexicon)
        k3, p3, n3 = _buf(char_prop)
        k4, p4, n4 = _buf(unk_handler)
        h = C.c_void_p()
        if isinstance(connector, np.ndarray):
            m = np.ascontiguousarray(connector, dtype=np.int16)
            nl, nr = m.shape
            check(lib().vbt_dict_from_parts(p1, n1, m.ctypes.data, nr, nl, p3, n3, p4, n4, C.byref(h)))
        else:
            k2, p2, n2 = _buf(connector)
            check(lib().vbt_dict_from_mecab(p1, n1, p2, n2, p3, n3, p4, n4, C.byref(h)))
        return Dictionary(h)


    @staticmethod
    def from_readers_with_bigram_info(system_lexicon, bigram_right, bigram_left, bigram_cost, char_prop, unk_handler,
                                      dual_connector=False):
        """from_readers_with_bigram_info (builder.rs:111-148): compact connector built from bigram.* files."""
        bufs = [_buf(x) for x in (system_lexicon, bigram_right, bigram_left, bigram_cost, char_prop, unk_handler)]
        args = []
        for _, p, n in bufs:
            args += [p, n]
        h = C.c_void_p()
        check(lib().vbt_dict_from_bigram(*args, int(dual_connector), C.byref(h)))
        return Dictionary(h)


def generate_bigram_info(feature_def, right_id_def, left_id_def, model_def, cost_factor):
    """mecab::generate_bigram_info (mecab.rs:31-181): a trained MeCab model (feature.def, right-id.def, left-id.def,
    model.def, in the reference's order) -> (bigram_right, bigram_left, bigram_cost) as bytes, the sources of
    SystemDictionaryBuilder.from_readers_with_bigram_info.  right-id.def gives bigram.right, left-id.def bigram.left."""
    bufs = [_buf(x) for x in (feature_def, right_id_def, left_id_def, model_def)]
    args = []
    for _, p, n in bufs:
        args += [p, n]
    ptrs = [C.c_void_p() for _ in range(3)]
    lens = [C.c_size_t() for _ in range(3)]
    out = []
    for p, n in zip(ptrs, lens):
        out += [C.byref(p), C.byref(n)]
    check(lib().vbt_mecab_generate_bigram_info(*args, float(cost_factor), *out))
    try:
        return tuple(C.string_at(p, n.value) for p, n in zip(ptrs, lens))
    finally:
        for p in ptrs:
            lib().vbt_bytes_free(p)


def scorer_accumulate(triples, keys1, keys2):
    """Test hook: ScorerBuilder + Scorer::accumulate_cost (raw_connector/scorer.rs)."""
    t = np.ascontiguousarray(np.array(triples, dtype=np.int32).reshape(-1))
    k1 = np.ascontiguousarray(keys1, dtype=np.uint32)
    k2 = np.ascontiguousarray(keys2, dtype=np.uint32)
    c = C.c_int32()
    check(lib().vbt_scorer_accumulate(t.ctypes.data, len(t) // 3, k1.ctypes.data, k2.ctypes.data, len(k1), C.byref(c)))
    return c.value


COMPACT_TOKEN_DTYPE = np.dtype(
    [("start_byte", "<u4"), ("end_byte", "<u4"), ("word_idx", "<u4"), ("total_cost", "<i4")]
)  # vbt_token16: the tokenizer option "compact_tokens"


def expand_compact_tokens(compact, tok_offsets, utf8, byte_offsets):
    """vbt_token16 records -> full TOKEN_DTYPE records: the character range of a token is the number of characters of
    the sentence in front of its byte range (what Sentence::compile's c2b table inverts, sentence.rs:40-46)."""
    out = np.zeros(len(compact), dtype=TOKEN_DTYPE)
    for name in ("start_byte", "end_byte", "word_idx", "total_cost"):
        out[name] = compact[name]
    if len(compact) == 0:
        return out
    utf8 = np.asarray(utf8, dtype=np.uint8)
    off = np.asarray(byte_offsets, dtype=np.int64)
    lead = np.concatenate([[0], np.cumsum((utf8 & 0xC0) != 0x80, dtype=np.int64)])  # characters starting before byte i
    counts = np.diff(np.asarray(tok_offsets, dtype=np.int64))
    sent_of = np.repeat(np.arange(len(counts)), counts)
    base = off[sent_of]
    out["start_char"] = lead[base + compact["start_byte"]] - lead[base]
    out["end_char"] = lead[base + compact["end_byte"]] - lead[base]
    return out


class BatchResult:
    """Tokens of a batch: `tok_offsets[i]..tok_offsets[i+1]` index `tokens` (TOKEN_DTYPE) for sentence i.  With the
    tokenizer option compact_tokens the device returns 16-byte records (`compact`); `tokens` is then rebuilt on the
    host from them and the sentences' UTF-8."""

    def __init__(self, tokenizer, handle, sentences_utf8, byte_offsets, compact=False):
        self._tok = tokenizer
        self._h = handle
        self._free = lib().vbt_result_free
        po, pt, ns, nt = C.c_void_p(), C.c_void_p(), C.c_uint64(), C.c_uint64()
        view = lib().vbt_result_view_compact if compact else lib().vbt_result_view
        check(view(handle, C.byref(po), C.byref(pt), C.byref(ns), C.byref(nt)))
        self.n_sent, self.n_tokens = ns.value, nt.value
        self.tok_offsets = np.ctypeslib.as_array(C.cast(po, C.POINTER(C.c_uint64)), shape=(self.n_sent + 1,))
        dt = COMPACT_TOKEN_DTYPE if compact else TOKEN_DTYPE
        if self.n_tokens:
            raw = np.ctypeslib.as_array(C.cast(pt, C.POINTER(C.c_uint8)), shape=(self.n_tokens * dt.itemsize,))
            toks = raw.view(dt)
        else:
            toks = np.empty(0, dtype=dt)
        self.compact = toks if compact else None
        self.tokens = expand_compact_tokens(toks, self.tok_offsets, sentences_utf8, byte_offsets) if compact else toks
        self._utf8 = sentences_utf8
        self._off = byte_offsets

    def close(self):
        h, self._h = self._h, None
        if h:
            self.tok_offsets = self.tok_offsets.copy()
            self.tokens = self.tokens.copy()
            if self.compact is not None:
                self.compact = self.compact.copy()
            self._free(h)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._free(h)

    def num_tokens(self, i):
        return int(self.tok_offsets[i + 1] - self.tok_offsets[i])

    def text(self):
        """(text_offsets uint64[n_sent + 1], text bytes): what `tokenize` prints for the batch
        (tokenize/src/main.rs:83-127), formatted on the device; needs Tokenizer.output_mode(...) first."""
        if self._h is None:
            raise VibratoError(1, "the result was closed")
        po, pt, nb = C.c_void_p(), C.c_void_p(), C.c_uint64()
        check(lib().vbt_result_text(self._h, C.byref(po), C.byref(pt), C.byref(nb)))
        offs = np.ctypeslib.as_array(C.cast(po, C.POINTER(C.c_uint64)), shape=(self.n_sent + 1,)).copy()
        text = C.string_at(pt, nb.value) if nb.value else b""
        return offs, text

    def sentence_tokens(self, i):
        """Token views of sentence i, in order (Worker::token_iter)."""
        s = bytes(self._utf8[int(self._off[i]):int(self._off[i + 1])])
        a, b = int(self.tok_offsets[i]), int(self.tok_offsets[i + 1])
        return [Token(self._tok, s, self.tokens[k]) for k in range(a, b)]


OUTPUT_MODES = {None: 0, "none": 0, "mecab": 1, "wakati": 2, "detail": 3}  # tokenize/src/main.rs:12-29


class Tokenizer:
    """vibrato::Tokenizer (tokenizer.rs:13-84); the device engine is created on first use."""

    def __init__(self, dict_, device=0, devices=None):
        self._dict = dict_
        self._devices = None if devices is None else [int(x) for x in devices]
        self._ignore_space = False
        self._max_grouping_len = 0
        self._device = device
        self._h = None
        self._options = {}  # engine options set so far: replayed when the engine is rebuilt (ignore_space / max_grouping_len)
        self._stream = 0
        self._counting = False
        self._free = lib().vbt_tokenizer_free

    @staticmethod
    def new(dict_, device=0, devices=None):
        """`devices=[...]`: one tokenizer over several GPUs of this node (vbt_tokenizer_new_multi): the batch is split
        by bytes, the dictionary image is uploaded once and broadcast, one result comes back in input order."""
        return Tokenizer(dict_, device, devices)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._free(h)

    def _reset(self):
        """ignore_space / max_grouping_len are fixed when the engine is built: drop it; handle() rebuilds it and
        replays the options set so far.  Connection-id counts gathered by the old engine are lost with it, so
        changing these after init_connid_counter() is refused."""
        if self._h:
            if getattr(self, "_connid_active", False):
                raise VibratoError(1, "tokenizer: ignore_space / max_grouping_len cannot change while connection ids are being counted")
            self._free(self._h)
            self._h = None

    def ignore_space(self, yes):
        """tokenizer.rs:42-55: Err(InvalidArgument) when `SPACE` is undefined in char.def."""
        if yes and self._dict.cate_id("SPACE") is None:
            raise VibratoError(1, "dict: SPACE is not defined in the input dictionary (i.e., char.def).")
        self._ignore_space = bool(yes)
        self._reset()
        return self

    def max_grouping_len(self, n):
        """tokenizer.rs:67-74: 0 means unlimited."""
        self._max_grouping_len = int(n)
        self._reset()
        return self

    def dictionary(self):
        return self._dict

    def new_worker(self):
        return Worker(self)

    def handle(self):
        if self._h is None:
            h = C.c_void_p()
            if self._devices is not None:
                devs = (C.c_int32 * len(self._devices))(*self._devices)
                check(lib().vbt_tokenizer_new_multi(self._dict._h, int(self._ignore_space), self._max_grouping_len,
                                                    devs, len(self._devices), C.byref(h)))
            else:
                check(lib().vbt_tokenizer_new(self._dict._h, int(self._ignore_space), self._max_grouping_len,
                                              self._device, C.byref(h)))
            self._h = h
            # a rebuilt engine starts from defaults: put back what the caller had configured
            for name, value in self._options.items():
                check(lib().vbt_tokenizer_set_option(h, name.encode(), int(value)))
            if self._counting:
                check(lib().vbt_tokenizer_set_counting(h, 1))
            if self._stream:
                check(lib().vbt_tokenizer_set_stream(h, int(self._stream)))
        return self._h

    @staticmethod
    def pack(sentences):
        """list[str|bytes] -> (utf8 uint8[], byte_offsets uint64[n+1])"""
        blobs = [s.encode("utf-8") if isinstance(s, str) else bytes(s) for s in sentences]
        off = np.zeros(len(blobs) + 1, dtype=np.uint64)
        if blobs:
            off[1:] = np.cumsum([len(b) for b in blobs], dtype=np.uint64)
        return np.frombuffer(b"".join(blobs), dtype=np.uint8), off

    def tokenize_batch(self, sentences=None, utf8=None, byte_offsets=None):
        """reset_sentence + tokenize for every sentence of the batch on the GPU (host in, host out)."""
        if sentences is not None:
            utf8, byte_offsets = self.pack(sentences)
        utf8 = np.ascontiguousarray(utf8, dtype=np.uint8)
        byte_offsets = np.ascontiguousarray(byte_offsets, dtype=np.uint64)
        n = len(byte_offsets) - 1
        h = C.c_void_p()
        check(lib().vbt_tokenize_batch(self.handle(), utf8.ctypes.data if utf8.size else None,
                                       byte_offsets.ctypes.data, n, C.byref(h)))
        return BatchResult(self, h, utf8, byte_offsets, compact=bool(self._options.get("compact_tokens", 0)))

    def tokenize_batch_device(self, d_utf8, d_byte_offsets, n_sent, n_bytes):
        """Device-resident variant: addresses in, (d_tok_offsets, d_tokens, n_tokens) out."""
        a, b, n = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib().vbt_tokenize_batch_device(self.handle(), int(d_utf8), int(d_byte_offsets), int(n_sent),
                                              int(n_bytes), C.byref(a), C.byref(b), C.byref(n)))
        return a.value, b.value, n.value

    # connection-id statistics (worker.rs:77-103) ---------------------------------------------------
    def init_connid_counter(self):
        """Worker::init_connid_counter: zero the counters; every batch tokenised afterwards is counted."""
        self.set_option("connid_counting", 1)
        self._connid_active = True

    def connid_counts(self):
        """-> (lid_count uint64[num_left], rid_count uint64[num_right]) accumulated since init_connid_counter."""
        nl, nr = C.c_uint32(), C.c_uint32()
        check(lib().vbt_connid_counts(self.handle(), None, None, C.byref(nl), C.byref(nr)))
        lid = np.zeros(nl.value, dtype=np.uint64)
        rid = np.zeros(nr.value, dtype=np.uint64)
        check(lib().vbt_connid_counts(self.handle(), lid.ctypes.data, rid.ctypes.data, None, None))
        return lid, rid

    def compute_connid_probs(self):
        """Worker::compute_connid_probs -> ConnIdCounter::compute_probs (mapper.rs:108-146): two lists of
        (id, probability) without id 0, by descending probability then ascending id."""
        out = []
        for cnt in self.connid_counts():
            total = float(cnt.sum(dtype=np.float64))
            probs = [(i, float(c) / total if total else float("nan")) for i, c in enumerate(cnt)][1:]
            probs.sort(key=lambda t: (-t[1], t[0]))
            out.append(probs)
        return out[0], out[1]

    # measurement hooks -------------------------------------------------------------------------
    def set_counting(self, on):
        check(lib().vbt_tokenizer_set_counting(self.handle(), int(on)))
        self._counting = bool(on)

    def set_option(self, name, value):
        check(lib().vbt_tokenizer_set_option(self.handle(), name.encode(), int(value)))
        if name != "connid_counting":  # accumulated counts cannot be carried into a rebuilt engine
            self._options[name] = int(value)

    def evaluate(self, corpus, feature_indices=()):
        """The loop of the `evaluate` tool (evaluate/src/main.rs:61-138) over a `surface\\tfeature` / `EOS` corpus:
        returns num_ref / num_sys / num_cor and precision / recall / f1 (main.rs:129-131)."""
        _, p, n = _buf(corpus)
        idx = np.ascontiguousarray(list(feature_indices), dtype=np.uint64)
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib().vbt_evaluate(self._dict._h, self.handle(), p, n, idx.ctypes.data if len(idx) else None, len(idx),
                                 C.byref(a), C.byref(b), C.byref(c)))
        num_ref, num_sys, num_cor = a.value, b.value, c.value
        precision = num_cor / num_sys if num_sys else float("nan")
        recall = num_cor / num_ref if num_ref else float("nan")
        f1 = 2.0 * precision * recall / (precision + recall) if precision + recall else float("nan")
        return {"num_ref": num_ref, "num_sys": num_sys, "num_cor": num_cor, "precision": precision, "recall": recall,
                "f1": f1}

    def compact_tokens(self, yes=True):
        """Results come back as 16-byte records (vbt_token16: byte range, word_idx, total_cost) — a third less PCIe
        traffic; BatchResult rebuilds the character ranges from the sentences' UTF-8 on the host."""
        self.set_option("compact_tokens", int(bool(yes)))
        return self

    def output_mode(self, mode):
        """`tokenize -O mecab|wakati|detail` (tokenize/src/main.rs:43-45): batches tokenised afterwards also carry
        their formatted text (BatchResult.text()).  None switches the stage off."""
        if mode not in OUTPUT_MODES:
            raise VibratoError(1, "Could not parse a mode")  # tokenize/src/main.rs:26
        self.set_option("output_mode", OUTPUT_MODES[mode])
        return self

    def describe(self):
        """dict: devices, how the dictionary image travelled ("nccl <version>" / "cudaMemcpyPeer" / "single device"), ..."""
        import json
        buf = C.create_string_buffer(1024)
        check(lib().vbt_tokenizer_describe(self.handle(), buf, 1024))
        return json.loads(buf.value.decode())

    def set_stream(self, cuda_stream):
        check(lib().vbt_tokenizer_set_stream(self.handle(), int(cuda_stream)))
        self._stream = int(cuda_stream)

    def last_stage_ms(self):
        names = lib().vbt_stage_names().decode().split(",")
        ms = (C.c_float * 16)()
        n = C.c_int32()
        check(lib().vbt_last_stage_ms(self.handle(), ms, 16, C.byref(n)))
        return dict(zip(names, [float(ms[i]) for i in range(n.value)]))

    def last_launch_count(self):
        n = C.c_uint64()
        check(lib().vbt_last_launch_count(self.handle(), C.byref(n)))
        return n.value

    def last_counters(self):
        cnt = (C.c_uint64 * 10)()
        check(lib().vbt_last_counters(self.handle(), cnt))
        return np.array(list(cnt), dtype=np.uint64)


class Token:
    """vibrato::token::Token (token.rs:8-92)."""

    __slots__ = ("_tok", "_sent", "_r")

    def __init__(self, tokenizer, sentence_bytes, rec):
        self._tok = tokenizer
        self._sent = sentence_bytes
        self._r = rec

    def range_char(self):
        return range(int(self._r["start_char"]), int(self._r["end_char"]))

    def range_byte(self):
        return range(int(self._r["start_byte"]), int(self._r["end_byte"]))

    def surface(self):
        return self._sent[int(self._r["start_byte"]):int(self._r["end_byte"])].decode("utf-8")

    def word_idx(self):
        w = int(self._r["word_idx"])
        return WordIdx(w >> 30, w & 0x3FFFFFFF)

    def feature(self):
        return self._tok._dict.word_feature(int(self._r["word_idx"]))

    def lex_type(self):
        return int(self._r["word_idx"]) >> 30

    def left_id(self):
        return self._tok._dict.word_param(int(self._r["word_idx"]))[0]

    def right_id(self):
        return self._tok._dict.word_param(int(self._r["word_idx"]))[1]

    def word_cost(self):
        return self._tok._dict.word_param(int(self._r["word_idx"]))[2]

    def total_cost(self):
        return int(self._r["total_cost"])


class Worker:
    """vibrato::tokenizer::worker::Worker (worker.rs:13-74): the one-sentence loop of
    tokenize/src/main.rs:78-81 keeps working unmodified (one tiny batch per call)."""

    def __init__(self, tokenizer):
        self._tok = tokenizer
        self._sent = b""
        self._tokens = []

    def reset_sentence(self, text):
        self._sent = text.encode("utf-8") if isinstance(text, str) else bytes(text)
        self._tokens = []

    def tokenize(self):
        if not self._sent:  # worker.rs:50-52
            return
        res = self._tok.tokenize_batch([self._sent])
        self._tokens = [Token(self._tok, self._sent, r.copy()) for r in res.tokens]
        res.close()

    def num_tokens(self):
        return len(self._tokens)

    def token(self, i):
        return self._tokens[i]

    def token_iter(self):
        return iter(self._tokens)
