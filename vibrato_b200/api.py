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
LINK_DTYPE = np.dtype([("prev", "<i4"), ("flags", "<u4")])  # vbt_lattice_link
NODE_BEST = 1  # VBT_NODE_BEST
SPAN_ANY = 0xFFFFFFFF  # VBT_SPAN_ANY: a required token of any feature
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
    host from them and the sentences' UTF-8.  With Tokenizer.marginals(theta) on, `token_probs` (float32[n_tokens])
    and `path_probs` (float32[n_sent]) hold the marginal of every token and the probability of each sentence's best
    path; both are None otherwise.  With Tokenizer.lattice() on, `node_offsets[i]..node_offsets[i+1]` index `nodes`
    (TOKEN_DTYPE), `node_links` (LINK_DTYPE) and `node_probs` (float32, None without marginals): every node of sentence
    i's lattice (include/vibrato_b200.h); all four are None otherwise.  With Tokenizer.lattice(margin=D), the nodes are
    the near-best ones and `node_margins` (int64) holds each one's exact cost margin; None otherwise.  With
    Tokenizer.sampling(n, theta) on,
    `sample_offsets[i * n + j]..sample_offsets[i * n + j + 1]` index `samples` (TOKEN_DTYPE): sample j of sentence i
    (sentence_samples()); both are None otherwise.  With Tokenizer.uncertainty() on, `entropies` and `log_path_probs`
    (float64[n_sent]) hold each sentence's path entropy (nats) and best-path log-probability, and with
    boundary_probs=True `boundary_offsets[i]..boundary_offsets[i+1]` index `boundary_probs` (float32): the probability
    that a token ends at each character position 0..n of sentence i (sentence_boundary_probs()); None otherwise.  With
    Tokenizer.posterior(gamma) on, `posterior_offsets[i]..posterior_offsets[i+1]` index `posterior_tokens`
    (TOKEN_DTYPE) and `posterior_probs` (float32): sentence i's posterior-decoded path and each token's marginal
    (sentence_posterior()), and `posterior_gains` (float64[n_sent]) its total gain; all four are None otherwise."""

    def __init__(self, tokenizer, handle, sentences_utf8, byte_offsets, compact=False, marginals=False, lattice=False,
                 samples=0, margins=False, uncertainty=0, posterior=False):
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
        self.token_probs = self.path_probs = None
        if marginals:
            tp, pp = C.c_void_p(), C.c_void_p()
            check(lib().vbt_result_marginals(handle, C.byref(tp), C.byref(pp)))
            f32 = C.POINTER(C.c_float)
            self.token_probs = (np.ctypeslib.as_array(C.cast(tp, f32), shape=(self.n_tokens,)) if self.n_tokens
                                else np.empty(0, dtype=np.float32))
            self.path_probs = (np.ctypeslib.as_array(C.cast(pp, f32), shape=(self.n_sent,)) if self.n_sent
                               else np.empty(0, dtype=np.float32))
        self.node_offsets = self.nodes = self.node_links = self.node_probs = self.node_margins = None
        if lattice:
            po, pn, pl, pp, nn = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint64()
            check(lib().vbt_result_lattice(handle, C.byref(po), C.byref(pn), C.byref(pl), C.byref(pp), C.byref(nn)))
            n = nn.value
            self.node_offsets = np.ctypeslib.as_array(C.cast(po, C.POINTER(C.c_uint64)), shape=(self.n_sent + 1,))
            u8 = C.POINTER(C.c_uint8)
            self.nodes = (np.ctypeslib.as_array(C.cast(pn, u8), shape=(n * TOKEN_DTYPE.itemsize,)).view(TOKEN_DTYPE)
                          if n else np.empty(0, dtype=TOKEN_DTYPE))
            self.node_links = (np.ctypeslib.as_array(C.cast(pl, u8), shape=(n * LINK_DTYPE.itemsize,)).view(LINK_DTYPE)
                               if n else np.empty(0, dtype=LINK_DTYPE))
            if pp.value:
                self.node_probs = (np.ctypeslib.as_array(C.cast(pp, C.POINTER(C.c_float)), shape=(n,)) if n
                                   else np.empty(0, dtype=np.float32))
            if margins:
                pm = C.c_void_p()
                check(lib().vbt_result_lattice_margins(handle, C.byref(pm)))
                self.node_margins = (np.ctypeslib.as_array(C.cast(pm, C.POINTER(C.c_int64)), shape=(n,)) if n
                                     else np.empty(0, dtype=np.int64))
        self.entropies = self.log_path_probs = self.boundary_offsets = self.boundary_probs = None
        if uncertainty:
            pe, pl, po, pb = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
            check(lib().vbt_result_uncertainty(handle, C.byref(pe), C.byref(pl), C.byref(po), C.byref(pb)))
            f64 = C.POINTER(C.c_double)
            n = self.n_sent
            self.entropies = np.ctypeslib.as_array(C.cast(pe, f64), shape=(n,)) if n else np.empty(0, dtype=np.float64)
            self.log_path_probs = (np.ctypeslib.as_array(C.cast(pl, f64), shape=(n,)) if n
                                   else np.empty(0, dtype=np.float64))
            if uncertainty >= 2:
                self.boundary_offsets = np.ctypeslib.as_array(C.cast(po, C.POINTER(C.c_uint64)), shape=(n + 1,))
                npos = int(self.boundary_offsets[n])
                self.boundary_probs = (np.ctypeslib.as_array(C.cast(pb, C.POINTER(C.c_float)), shape=(npos,)) if npos
                                       else np.empty(0, dtype=np.float32))
        self.n_samples = int(samples)  # samples per sentence, 0 without sampling
        self.sample_offsets = self.samples = None
        if samples:
            po, ps, nn = C.c_void_p(), C.c_void_p(), C.c_uint64()
            check(lib().vbt_result_samples(handle, C.byref(po), C.byref(ps), C.byref(nn)))
            n = nn.value
            self.sample_offsets = np.ctypeslib.as_array(C.cast(po, C.POINTER(C.c_uint64)),
                                                        shape=(self.n_sent * self.n_samples + 1,))
            self.samples = (np.ctypeslib.as_array(C.cast(ps, C.POINTER(C.c_uint8)), shape=(n * TOKEN_DTYPE.itemsize,))
                            .view(TOKEN_DTYPE) if n else np.empty(0, dtype=TOKEN_DTYPE))
        self.posterior_offsets = self.posterior_tokens = self.posterior_probs = self.posterior_gains = None
        if posterior:
            po, pt, pp, pg, nn = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint64()
            check(lib().vbt_result_posterior(handle, C.byref(po), C.byref(pt), C.byref(pp), C.byref(pg), C.byref(nn)))
            n, ns = nn.value, self.n_sent
            self.posterior_offsets = np.ctypeslib.as_array(C.cast(po, C.POINTER(C.c_uint64)), shape=(ns + 1,))
            self.posterior_tokens = (np.ctypeslib.as_array(C.cast(pt, C.POINTER(C.c_uint8)),
                                                           shape=(n * TOKEN_DTYPE.itemsize,)).view(TOKEN_DTYPE)
                                     if n else np.empty(0, dtype=TOKEN_DTYPE))
            self.posterior_probs = (np.ctypeslib.as_array(C.cast(pp, C.POINTER(C.c_float)), shape=(n,)) if n
                                    else np.empty(0, dtype=np.float32))
            self.posterior_gains = (np.ctypeslib.as_array(C.cast(pg, C.POINTER(C.c_double)), shape=(ns,)) if ns
                                    else np.empty(0, dtype=np.float64))
        self._utf8 = sentences_utf8
        self._off = byte_offsets

    def close(self):
        h, self._h = self._h, None
        if h:
            self.tok_offsets = self.tok_offsets.copy()
            self.tokens = self.tokens.copy()
            if self.compact is not None:
                self.compact = self.compact.copy()
            if self.token_probs is not None:
                self.token_probs = self.token_probs.copy()
                self.path_probs = self.path_probs.copy()
            for name in ("node_offsets", "nodes", "node_links", "node_probs", "node_margins", "sample_offsets", "samples",
                         "entropies", "log_path_probs", "boundary_offsets", "boundary_probs", "posterior_offsets",
                         "posterior_tokens", "posterior_probs", "posterior_gains"):
                if getattr(self, name) is not None:
                    setattr(self, name, getattr(self, name).copy())
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
        # string_at takes a C int size: texts of 2 GiB and more (n samples of a large batch) are read as an array
        n = nb.value
        text = b"" if not n else C.string_at(pt, n) if n < 2 ** 31 else (C.c_char * n).from_address(pt.value).raw
        return offs, text

    def sentence_tokens(self, i):
        """Token views of sentence i, in order (Worker::token_iter)."""
        s = bytes(self._utf8[int(self._off[i]):int(self._off[i + 1])])
        a, b = int(self.tok_offsets[i]), int(self.tok_offsets[i + 1])
        tp = self.token_probs
        return [Token(self._tok, s, self.tokens[k], None if tp is None else float(tp[k])) for k in range(a, b)]

    def num_nodes(self, i):
        return int(self.node_offsets[i + 1] - self.node_offsets[i])

    def sentence_samples(self, i):
        """The n sampled segmentations of sentence i (Tokenizer.sampling), each a list of Token views; Token.prob()
        raises on them."""
        if self.samples is None:
            raise VibratoError(1, "no samples: switch sampling on with Tokenizer.sampling() before tokenising")
        s = bytes(self._utf8[int(self._off[i]):int(self._off[i + 1])])
        n, so = self.n_samples, self.sample_offsets
        return [[Token(self._tok, s, self.samples[k]) for k in range(int(so[i * n + j]), int(so[i * n + j + 1]))]
                for j in range(n)]

    def sentence_posterior(self, i):
        """Token views of sentence i's posterior-decoded path (Tokenizer.posterior), in order; Token.prob() gives
        each token's marginal."""
        if self.posterior_tokens is None:
            raise VibratoError(1, "no posterior paths: switch posterior decoding on with Tokenizer.posterior() "
                                  "before tokenising")
        s = bytes(self._utf8[int(self._off[i]):int(self._off[i + 1])])
        a, b = int(self.posterior_offsets[i]), int(self.posterior_offsets[i + 1])
        return [Token(self._tok, s, self.posterior_tokens[k], float(self.posterior_probs[k])) for k in range(a, b)]

    def sentence_boundary_probs(self, i):
        """float32[n_chars + 1]: P(a token ends at character position p) for p = 0..n of sentence i (needs
        Tokenizer.uncertainty(boundary_probs=True))."""
        if self.boundary_probs is None:
            raise VibratoError(1, "no boundary probabilities: switch them on with "
                                  "Tokenizer.uncertainty(boundary_probs=True) before tokenising")
        return self.boundary_probs[int(self.boundary_offsets[i]):int(self.boundary_offsets[i + 1])]

    def sentence_nodes(self, i):
        """LatticeNode views of sentence i's lattice, in node order (needs Tokenizer.lattice())."""
        if self.nodes is None:
            raise VibratoError(1, "no lattice: switch it on with Tokenizer.lattice() before tokenising")
        s = bytes(self._utf8[int(self._off[i]):int(self._off[i + 1])])
        a, b = int(self.node_offsets[i]), int(self.node_offsets[i + 1])
        npb, nm = self.node_probs, self.node_margins
        return [LatticeNode(self._tok, s, self.nodes[k], self.node_links[k], None if npb is None else float(npb[k]),
                            None if nm is None else int(nm[k]))
                for k in range(a, b)]


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
        self._format = None  # (node, unk, bos, eos) of output_format(), replayed after the options
        self._theta = 0.0  # marginals(), replayed before the format
        self._lattice = 0  # lattice(), replayed before the format
        self._lattice_margin = -1  # lattice(margin=D), replayed with it
        self._uncertainty = 0  # uncertainty(), replayed after the marginals
        self._sampling = (0, 0.0, 0)  # sampling() as (n, theta, seed), replayed after the marginals
        self._sample_text = False  # sampling(text=True), replayed after sampling
        self._posterior = None  # posterior()'s gamma, replayed after the marginals
        self._posterior_text = False  # posterior(text=True), replayed after it
        self._stream = 0
        self._counting = False
        self._free = lib().vbt_tokenizer_free

    @staticmethod
    def new(dict_, device=0, devices=None):
        """`devices=[...]`: one tokenizer over several GPUs of this node (vbt_tokenizer_new_multi): the batch is split
        by bytes, the dictionary image is uploaded once and broadcast, one result comes back in input order.  A device
        listed more than once runs one shard per entry on it: this runs the sharded path on one GPU and is not faster."""
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
            if self._theta:
                check(lib().vbt_tokenizer_set_marginals(h, self._theta))
            if self._lattice:
                check(lib().vbt_tokenizer_set_option(h, b"lattice", self._lattice))
            if self._lattice_margin >= 0:
                check(lib().vbt_tokenizer_set_option(h, b"lattice_margin", self._lattice_margin))
            if self._uncertainty:
                check(lib().vbt_tokenizer_set_option(h, b"uncertainty", self._uncertainty))
            if self._sampling[0]:
                check(lib().vbt_tokenizer_set_sampling(h, *self._sampling))
            if self._sample_text:
                check(lib().vbt_tokenizer_set_option(h, b"sample_text", 1))
            if self._posterior is not None:
                check(lib().vbt_tokenizer_set_posterior(h, 1, self._posterior))
            if self._posterior_text:
                check(lib().vbt_tokenizer_set_option(h, b"posterior_text", 1))
            if self._format is not None:
                self._set_format(h, self._format)
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

    @staticmethod
    def pack_bounds(boundaries):
        """list[list[int]] (per-sentence byte offsets) -> (bnd_offsets uint64[n+1], bnd uint32[])"""
        off = np.zeros(len(boundaries) + 1, dtype=np.uint64)
        if boundaries:
            off[1:] = np.cumsum([len(b) for b in boundaries], dtype=np.uint64)
        flat = [v for b in boundaries for v in b]
        return off, np.array(flat, dtype=np.uint32)

    @staticmethod
    def pack_spans(spans):
        """list[list[(start, end) | (start, end, pattern)]] (per-sentence byte offsets; pattern str or bytes) ->
        (span_offsets uint64[n+1], span_records uint32[k, 3], patterns list[bytes]).  Equal patterns share one entry;
        a span without a pattern gets VBT_SPAN_ANY."""
        off = np.zeros(len(spans) + 1, dtype=np.uint64)
        if spans:
            off[1:] = np.cumsum([len(s) for s in spans], dtype=np.uint64)
        index, patterns, rec = {}, [], []
        for sent in spans:
            for sp in sent:
                p = SPAN_ANY
                if len(sp) > 2 and sp[2] is not None:
                    b = sp[2].encode("utf-8") if isinstance(sp[2], str) else bytes(sp[2])
                    if b not in index:
                        index[b] = len(patterns)
                        patterns.append(b)
                    p = index[b]
                rec.append((sp[0], sp[1], p))
        return off, np.array(rec, dtype=np.uint32).reshape(-1, 3), patterns

    @staticmethod
    def _pattern_table(patterns):
        blobs = [p.encode("utf-8") if isinstance(p, str) else bytes(p) for p in patterns]
        off = np.zeros(len(blobs) + 1, dtype=np.uint64)
        if blobs:
            off[1:] = np.cumsum([len(b) for b in blobs], dtype=np.uint64)
        return np.frombuffer(b"".join(blobs) + b"\0", dtype=np.uint8), off

    def tokenize_batch(self, sentences=None, utf8=None, byte_offsets=None, boundaries=None, bnd_offsets=None, bnd=None,
                       spans=None, span_offsets=None, span_records=None, patterns=None):
        """reset_sentence + tokenize for every sentence of the batch on the GPU (host in, host out).

        Required boundaries (vbt_tokenize_batch_bounded): `boundaries` = one list of sentence-relative byte offsets
        per sentence, or the packed form bnd_offsets (uint64[n+1]) / bnd (uint32[]).  No token of a sentence crosses
        one of its boundaries; the library validates them.

        Required tokens (vbt_tokenize_batch_spans): `spans` = one list per sentence of (start, end) or
        (start, end, pattern) byte ranges, each of which must be exactly one token (whose feature matches the
        pattern, README "Required tokens"); or the packed form span_offsets (uint64[n+1]) / span_records
        (uint32[k, 3]: start, end, pattern index or SPAN_ANY) / patterns (list of str or bytes).  Boundaries may
        come with them."""
        if sentences is not None:
            utf8, byte_offsets = self.pack(sentences)
        if boundaries is not None:
            bnd_offsets, bnd = self.pack_bounds(boundaries)
        if spans is not None:
            span_offsets, span_records, patterns = self.pack_spans(spans)
        utf8 = np.ascontiguousarray(utf8, dtype=np.uint8)
        byte_offsets = np.ascontiguousarray(byte_offsets, dtype=np.uint64)
        n = len(byte_offsets) - 1
        h = C.c_void_p()
        if span_offsets is not None:
            span_offsets = np.ascontiguousarray(span_offsets, dtype=np.uint64)
            recs = np.ascontiguousarray(span_records if span_records is not None else np.zeros((0, 3)),
                                        dtype=np.uint32).reshape(-1, 3)
            pat, pat_off = self._pattern_table(patterns or [])
            if bnd_offsets is not None:
                bnd_offsets = np.ascontiguousarray(bnd_offsets, dtype=np.uint64)
                bnd = np.ascontiguousarray(bnd if bnd is not None else [], dtype=np.uint32)
            check(lib().vbt_tokenize_batch_spans(
                self.handle(), utf8.ctypes.data if utf8.size else None, byte_offsets.ctypes.data, n,
                bnd_offsets.ctypes.data if bnd_offsets is not None else None,
                bnd.ctypes.data if bnd_offsets is not None and bnd.size else None, span_offsets.ctypes.data,
                recs.ctypes.data if recs.size else None, pat.ctypes.data, pat_off.ctypes.data, len(pat_off) - 1,
                C.byref(h)))
        elif bnd_offsets is None:
            check(lib().vbt_tokenize_batch(self.handle(), utf8.ctypes.data if utf8.size else None,
                                           byte_offsets.ctypes.data, n, C.byref(h)))
        else:
            bnd_offsets = np.ascontiguousarray(bnd_offsets, dtype=np.uint64)
            bnd = np.ascontiguousarray(bnd if bnd is not None else [], dtype=np.uint32)
            check(lib().vbt_tokenize_batch_bounded(self.handle(), utf8.ctypes.data if utf8.size else None,
                                                   byte_offsets.ctypes.data, n, bnd_offsets.ctypes.data,
                                                   bnd.ctypes.data if bnd.size else None, C.byref(h)))
        return BatchResult(self, h, utf8, byte_offsets, compact=bool(self._options.get("compact_tokens", 0)),
                           marginals=self._theta > 0, lattice=self._lattice > 0, samples=self._sampling[0],
                           margins=self._lattice > 0 and self._lattice_margin >= 0,
                           uncertainty=self._uncertainty if self._theta > 0 else 0,
                           posterior=self._posterior is not None and self._theta > 0)

    def tokenize_batch_device(self, d_utf8, d_byte_offsets, n_sent, n_bytes, d_bnd_offsets=None, d_bnd=None, n_bnd=0,
                              d_span_offsets=None, d_spans=None, n_spans=0, patterns=None):
        """Device-resident variant: addresses in, (d_tok_offsets, d_tokens, n_tokens) out.  With d_bnd_offsets
        (uint64[n_sent+1]) and d_bnd (uint32[n_bnd]), also device addresses: required boundaries as in
        tokenize_batch.  With d_span_offsets (uint64[n_sent+1]) and d_spans (uint32[n_spans, 3]), device addresses,
        and `patterns` (a host list): required tokens as in tokenize_batch."""
        a, b, n = C.c_uint64(), C.c_uint64(), C.c_uint64()
        if d_span_offsets is not None:
            pat, pat_off = self._pattern_table(patterns or [])
            check(lib().vbt_tokenize_batch_device_spans(
                self.handle(), int(d_utf8), int(d_byte_offsets), int(n_sent), int(n_bytes), int(d_bnd_offsets or 0),
                int(d_bnd or 0), int(n_bnd), int(d_span_offsets), int(d_spans or 0), int(n_spans), pat.ctypes.data,
                pat_off.ctypes.data, len(pat_off) - 1, C.byref(a), C.byref(b), C.byref(n)))
        elif d_bnd_offsets is None:
            check(lib().vbt_tokenize_batch_device(self.handle(), int(d_utf8), int(d_byte_offsets), int(n_sent),
                                                  int(n_bytes), C.byref(a), C.byref(b), C.byref(n)))
        else:
            check(lib().vbt_tokenize_batch_device_bounded(self.handle(), int(d_utf8), int(d_byte_offsets), int(n_sent),
                                                          int(n_bytes), int(d_bnd_offsets), int(d_bnd or 0),
                                                          int(n_bnd), C.byref(a), C.byref(b), C.byref(n)))
        return a.value, b.value, n.value

    def last_device_marginals(self):
        """-> (d_token_probs, d_path_probs): device addresses (float32[n_tokens], float32[n_sent]) of the marginals of
        the last tokenize_batch_device call, valid until the next call."""
        a, b = C.c_uint64(), C.c_uint64()
        check(lib().vbt_last_device_marginals(self.handle(), C.byref(a), C.byref(b)))
        return a.value, b.value

    def last_device_uncertainty(self):
        """-> (d_entropies, d_log_path_probs, d_boundary_offsets, d_boundary_probs, n_positions): device addresses
        (float64[n_sent], float64[n_sent], uint64[n_sent + 1], float32[n_positions]; the last three 0 without
        boundary_probs) of the uncertainty of the last tokenize_batch_device call, valid until the next call."""
        v = [C.c_uint64() for _ in range(5)]
        check(lib().vbt_last_device_uncertainty(self.handle(), *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def last_device_lattice(self):
        """-> (d_node_offsets, d_nodes, d_links, d_node_probs, n_nodes): device addresses (uint64[n_sent + 1],
        vbt_token[n_nodes], vbt_lattice_link[n_nodes], float32[n_nodes] or 0 without marginals) of the lattice of the
        last tokenize_batch_device call, valid until the next call."""
        v = [C.c_uint64() for _ in range(5)]
        check(lib().vbt_last_device_lattice(self.handle(), *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def last_device_lattice_margins(self):
        """-> d_node_margins: device address (int64[n_nodes]) of the node margins of the last tokenize_batch_device
        call made with lattice(margin=D), valid until the next call."""
        v = C.c_uint64()
        check(lib().vbt_last_device_lattice_margins(self.handle(), C.byref(v)))
        return v.value

    def last_device_samples(self):
        """-> (d_sample_offsets, d_samples, n_sample_tokens): device addresses (uint64[n_sent * n + 1],
        vbt_token[n_sample_tokens]) of the samples of the last tokenize_batch_device call, valid until the next call."""
        v = [C.c_uint64() for _ in range(3)]
        check(lib().vbt_last_device_samples(self.handle(), *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def last_device_posterior(self):
        """-> (d_posterior_offsets, d_posterior_tokens, d_posterior_probs, d_posterior_gains, n_posterior_tokens):
        device addresses (uint64[n_sent + 1], vbt_token[n], float32[n], float64[n_sent]) of the posterior paths of the
        last tokenize_batch_device call, valid until the next call."""
        v = [C.c_uint64() for _ in range(5)]
        check(lib().vbt_last_device_posterior(self.handle(), *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def posterior(self, gamma=1.0, text=False):
        """Posterior decoding (maximum expected accuracy; needs marginals() on): every result then also carries each
        sentence's path whose tokens have the largest total gain (gamma + 1) * p - 1, p the token's marginal
        (BatchResult.posterior_offsets / posterior_tokens / posterior_probs / posterior_gains, sentence_posterior()).
        gamma >= 0 and finite; 1 is the centroid estimator, larger values favour recall.  None switches it off.
        text=True ("posterior_text") renders the posterior path in place of the best path in the output text.  The
        tokens and every other output do not change; the "small_batch" route steps aside.  Definition:
        include/vibrato_b200.h."""
        if not text and self._posterior_text:  # before posterior decoding may switch off, which posterior text refuses
            check(lib().vbt_tokenizer_set_option(self.handle(), b"posterior_text", 0))
            self._posterior_text = False
        on = gamma is not None
        check(lib().vbt_tokenizer_set_posterior(self.handle(), int(on), float(gamma) if on else 0.0))
        self._posterior = float(gamma) if on else None
        if text:
            check(lib().vbt_tokenizer_set_option(self.handle(), b"posterior_text", 1))
            self._posterior_text = True
        return self

    def sampling(self, n, theta=1.0, seed=0, text=False):
        """Segmentation sampling ("subword regularisation"): every result then carries n segmentations per sentence
        drawn with replacement from P(path) = exp(-theta * cost(path)) / Z, the distribution of marginals()
        (BatchResult.samples / sample_offsets, sentence_samples()).  theta > 0 and finite; with marginals on it must be
        theirs.  seed (u64) keys the draws, which depend only on (seed, sentence index, sample, step); the sentence
        index starts at sample_base() in every call.  n = 0 (or None) switches sampling off.  The tokens do not
        change; the "small_batch" route steps aside.  text=True ("sample_text") also renders each sentence's n samples,
        one after another, in place of its best path in the output text (BatchResult.text()); set it before a format.
        Definition: include/vibrato_b200.h."""
        n = 0 if n is None else int(n)
        theta, seed = float(theta), int(seed)
        if not 0 <= seed < 2 ** 64:
            raise VibratoError(1, "sampling: seed must be an unsigned 64-bit integer")
        if not 0 <= n < 2 ** 32:
            raise VibratoError(1, "sampling: n must be between 0 (off) and 1024")
        if not text and self._sample_text:  # before sampling may switch off, which sample text refuses
            check(lib().vbt_tokenizer_set_option(self.handle(), b"sample_text", 0))
            self._sample_text = False
        check(lib().vbt_tokenizer_set_sampling(self.handle(), n, theta, seed))
        self._sampling = (n, theta, seed) if n else (0, 0.0, 0)
        if text:
            check(lib().vbt_tokenizer_set_option(self.handle(), b"sample_text", 1))
            self._sample_text = True
        return self

    def sample_base(self, i):
        """The draws of sentence s of the calls that follow use the sentence index i + s (the option "sample_base",
        default 0), so that a corpus tokenised in pieces draws what one call over all of it would: set it to each
        piece's first index.  A call with i + n_sent > 2^32 is refused."""
        self.set_option("sample_base", int(i))
        return self

    def lattice(self, on=True, text=False, margin=None):
        """Lattice output: results then carry every node of each sentence's lattice (BatchResult.nodes /
        node_links / node_probs, sentence_nodes()), with its best predecessor, a best-path flag and, with marginals,
        its marginal.  text=True also renders the nodes in place of the tokens in the output text (MeCab -a).
        margin=D (an integer, 0 <= D <= 2^62; the option "lattice_margin") keeps only the nodes on paths whose cost is
        within D of the best one, plus the best path, and adds BatchResult.node_margins; None keeps every node.
        The "small_batch" route steps aside.  Definition: include/vibrato_b200.h."""
        value = (2 if text else 1) if on else 0
        m = -1 if margin is None else int(margin)
        if margin is not None and m < 0:
            raise VibratoError(1, "lattice: margin must be None or a cost margin between 0 and 2^62")
        check(lib().vbt_tokenizer_set_option(self.handle(), b"lattice_margin", m))
        self._lattice_margin = m
        check(lib().vbt_tokenizer_set_option(self.handle(), b"lattice", value))
        self._lattice = value
        return self

    def marginals(self, theta):
        """Marginal probabilities at temperature `theta` (> 0; None or 0 switches them off): P(path) is proportional
        to exp(-theta * cost(path)) over every BOS -> EOS path of the lattice, a token's marginal sums P over the
        paths through its node.  Results then carry BatchResult.token_probs / path_probs and Token.prob().  The tokens
        do not change; the "small_batch" route steps aside while they are on.  Definition: include/vibrato_b200.h."""
        theta = 0.0 if theta is None else float(theta)
        check(lib().vbt_tokenizer_set_marginals(self.handle(), theta))
        self._theta = theta
        return self

    def uncertainty(self, on=True, boundary_probs=False):
        """Segmentation uncertainty (the option "uncertainty"; needs marginals() on): results then carry each
        sentence's path entropy in nats and best-path log-probability (BatchResult.entropies / log_path_probs, float64),
        and with boundary_probs=True the probability that a token ends at each character position 0..n
        (BatchResult.boundary_offsets / boundary_probs, sentence_boundary_probs()).  on=False switches it off.  The
        tokens and every other output do not change; the "small_batch" route steps aside.  Definition:
        include/vibrato_b200.h."""
        value = (2 if boundary_probs else 1) if on else 0
        check(lib().vbt_tokenizer_set_option(self.handle(), b"uncertainty", value))
        self._uncertainty = value
        return self

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
        if name == "lattice":  # replayed with lattice()'s state, after the marginals
            self._lattice = int(value)
            return
        if name == "lattice_margin":  # replayed with lattice()'s state
            self._lattice_margin = int(value)
            return
        if name == "uncertainty":  # replayed with uncertainty()'s state, after the marginals it needs
            self._uncertainty = int(value)
            return
        if name == "sample_text":  # replayed after sampling, which it needs
            self._sample_text = bool(value)
            return
        if name == "posterior_text":  # replayed after posterior decoding, which it needs
            self._posterior_text = bool(value)
            return
        if name != "connid_counting":  # accumulated counts cannot be carried into a rebuilt engine
            self._options[name] = int(value)
        if name == "output_mode":  # a fixed mode replaces an output format
            self._format = None

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

    def output_format(self, node, unk=None, bos="", eos="EOS\n"):
        """MeCab-style output formats (`-F` / `--unk-format` / `--bos-format` / `--eos-format`), rendered on the
        device: batches tokenised afterwards carry the text in BatchResult.text().  `node` is printed per System / User
        token, `unk` per Unknown token (None: as node), `bos` / `eos` before / after every sentence.  The directives
        are listed in README.md and include/vibrato_b200.h.  Replaces output_mode(); output_format(None) switches the
        format off.  str or bytes."""
        if node is None:
            check(lib().vbt_tokenizer_set_output_format(self.handle(), None, 0, None, 0, None, 0, None, 0))
            self._format = None
            return self
        enc = lambda x: None if x is None else (x.encode("utf-8") if isinstance(x, str) else bytes(x))  # noqa: E731
        fmt = (enc(node), enc(unk), enc(bos), enc(eos))
        self._set_format(self.handle(), fmt)
        self._format = fmt
        self._options.pop("output_mode", None)
        return self

    @staticmethod
    def _set_format(h, fmt):
        args = []
        for x in fmt:
            args += [x, len(x)] if x is not None else [None, 0]
        check(lib().vbt_tokenizer_set_output_format(h, *args))

    def small_batch(self, n=64):
        """Batches of at most `n` sentences and 16 KiB tokenised afterwards run in one kernel launch (k_small_batch):
        one copy up, one launch, one copy down, one synchronisation, with the same tokens and text.  Counted runs
        keep the usual route.  0 switches the route off (the default)."""
        self.set_option("small_batch", int(n))
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

    __slots__ = ("_tok", "_sent", "_r", "_p")

    def __init__(self, tokenizer, sentence_bytes, rec, prob=None):
        self._tok = tokenizer
        self._sent = sentence_bytes
        self._r = rec
        self._p = prob

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

    def prob(self):
        """The token's marginal probability (Tokenizer.marginals)."""
        if self._p is None:
            raise VibratoError(1, "no marginals: switch them on with Tokenizer.marginals(theta) before tokenising")
        return self._p


class LatticeNode(Token):
    """One node of a sentence's lattice (Tokenizer.lattice): Token's accessors (start_char is the node's start_word,
    total_cost its min_cost), plus its best predecessor, best-path flag, marginal and, in a near-best lattice, margin."""

    __slots__ = ("_link", "_margin")

    def __init__(self, tokenizer, sentence_bytes, rec, link, prob=None, margin=None):
        super().__init__(tokenizer, sentence_bytes, rec, prob)
        self._link = link
        self._margin = margin

    def margin(self):
        """The node's exact cost margin over the best path (Tokenizer.lattice(margin=D))."""
        if self._margin is None:
            raise VibratoError(1, "no margins: pass margin= to Tokenizer.lattice() before tokenising")
        return self._margin

    def prev(self):
        """Index of the best predecessor in the sentence's node list, or None for BOS and, in a near-best lattice,
        for a predecessor that was not kept (link prev -2)."""
        p = int(self._link["prev"])
        return None if p < 0 else p

    def is_best(self):
        return bool(int(self._link["flags"]) & NODE_BEST)


class Worker:
    """vibrato::tokenizer::worker::Worker (worker.rs:13-74): the one-sentence loop of
    tokenize/src/main.rs:78-81 keeps working unmodified (one tiny batch per call)."""

    def __init__(self, tokenizer):
        self._tok = tokenizer
        self._sent = b""
        self._bounds = None
        self._spans = None
        self._tokens = []
        self._nodes = []
        self._samples = []
        self._unc = None  # (entropy, log_path_prob, boundary probabilities or None) with Tokenizer.uncertainty()
        self._post = []  # the posterior path's tokens with Tokenizer.posterior()

    def reset_sentence(self, text, boundaries=None, spans=None):
        """boundaries: required token boundaries, byte offsets into the sentence; spans: required tokens, (start, end)
        or (start, end, pattern) byte ranges (see Tokenizer.tokenize_batch)."""
        self._sent = text.encode("utf-8") if isinstance(text, str) else bytes(text)
        self._bounds = None if boundaries is None else list(boundaries)
        self._spans = None if spans is None else list(spans)
        self._tokens = []
        self._nodes = []
        self._samples = []
        self._unc = None
        self._post = []

    def tokenize(self):
        if not self._sent:  # worker.rs:50-52
            self._samples = [[] for _ in range(self._tok._sampling[0])]
            level = self._tok._uncertainty if self._tok._theta > 0 else 0
            if level:  # the one empty path: no uncertainty, and it ends where it starts
                self._unc = (0.0, 0.0, np.ones(1, dtype=np.float32) if level >= 2 else None)
            return
        res = self._tok.tokenize_batch([self._sent], boundaries=None if self._bounds is None else [self._bounds],
                                       spans=None if self._spans is None else [self._spans])
        tp = res.token_probs
        self._tokens = [Token(self._tok, self._sent, r.copy(), None if tp is None else float(tp[k]))
                        for k, r in enumerate(res.tokens)]
        self._nodes = res.sentence_nodes(0) if res.nodes is not None else []
        for nd in self._nodes:
            nd._r, nd._link = nd._r.copy(), nd._link.copy()
        self._samples = res.sentence_samples(0) if res.samples is not None else []
        for sample in self._samples:
            for t in sample:
                t._r = t._r.copy()
        if res.entropies is not None:
            self._unc = (float(res.entropies[0]), float(res.log_path_probs[0]),
                         None if res.boundary_probs is None else res.sentence_boundary_probs(0).copy())
        self._post = res.sentence_posterior(0) if res.posterior_tokens is not None else []
        for t in self._post:
            t._r = t._r.copy()
        res.close()

    def num_tokens(self):
        return len(self._tokens)

    def token(self, i):
        return self._tokens[i]

    def token_iter(self):
        return iter(self._tokens)

    def num_nodes(self):
        """Nodes of the sentence's lattice (Tokenizer.lattice())."""
        return len(self._nodes)

    def node(self, i):
        return self._nodes[i]

    def node_iter(self):
        return iter(self._nodes)

    def _uncertainty(self, k):
        if self._unc is None:
            raise VibratoError(1, "no uncertainty: switch it on with Tokenizer.uncertainty() and tokenize first")
        return self._unc[k]

    def entropy(self):
        """The sentence's path entropy in nats (Tokenizer.uncertainty())."""
        return self._uncertainty(0)

    def log_path_prob(self):
        """ln P(best path) of the sentence (Tokenizer.uncertainty())."""
        return self._uncertainty(1)

    def boundary_probs(self):
        """float32[n_chars + 1]: P(a token ends at character position p), p = 0..n (Tokenizer.uncertainty(
        boundary_probs=True))."""
        b = self._uncertainty(2)
        if b is None:
            raise VibratoError(1, "no boundary probabilities: switch them on with "
                                  "Tokenizer.uncertainty(boundary_probs=True) before tokenising")
        return b

    def _posterior_on(self):
        if self._tok._posterior is None or not self._tok._theta:
            raise VibratoError(1, "no posterior path: switch posterior decoding on with Tokenizer.posterior() "
                                  "before tokenising")

    def num_posterior_tokens(self):
        """Tokens of the sentence's posterior-decoded path (Tokenizer.posterior())."""
        self._posterior_on()
        return len(self._post)

    def posterior_token(self, i):
        """Token i of the sentence's posterior-decoded path; its prob() is the token's marginal."""
        self._posterior_on()
        return self._post[i]

    def sample_tokens(self, j):
        """The tokens of sample j of the sentence (Tokenizer.sampling())."""
        if not self._tok._sampling[0]:
            raise VibratoError(1, "no samples: switch sampling on with Tokenizer.sampling() before tokenising")
        return self._samples[j]
