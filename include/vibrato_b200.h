/*
 * vibrato_b200.h — C ABI of the H100-native batched Viterbi tokenizer.
 *
 * The reference (daac-tools/vibrato, Rust) has no FFI; its seam is the public Rust API consumed by
 * the `tokenize` and `benchmark` crates (SURVEY.md §8b).  Each entry point below names the Rust
 * item it stands behind (paths relative to /root/reference/vibrato/src/); INTEGRATION.md shows the
 * Rust shim (`extern "C"` block + Dictionary/Tokenizer/Worker/Token wrappers) that binds them.
 *
 * Conventions: every function returns an int32 status (VBT_OK = 0; 1..8 and 10 mirror the VibratoError
 * variants of errors.rs:11-42); out-parameters come last; handles are opaque and released with the
 * matching *_free; vbt_last_error() returns the calling thread's last message (UTF-8, NUL-ended).
 * No torch / CUDA types appear in any signature: device memory is passed as plain addresses.
 *
 * There is NO CPU fallback: functions that run the hot path fail with VBT_ERR_NO_DEVICE /
 * VBT_ERR_CUDA when no usable GPU is present.
 *
 * Threads: a vbt_dict may be shared by readers once built; a vbt_tokenizer owns one workspace and one
 * stream, like a vibrato Worker (tokenizer/worker.rs:14-24), so it serves one caller at a time — create one
 * tokenizer per host thread (they may share the dictionary).  A vbt_result stays valid after its tokenizer is
 * freed.  Inputs are untrusted: dictionary streams, source files and byte offsets are validated, never assumed.
 */
#ifndef VIBRATO_B200_H
#define VIBRATO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
    VBT_OK = 0,
    VBT_ERR_INVALID_ARGUMENT = 1, /* VibratoError::InvalidArgument */
    VBT_ERR_INVALID_FORMAT = 2,   /* VibratoError::InvalidFormat   */
    VBT_ERR_TRY_FROM_INT = 3,     /* VibratoError::TryFromInt      */
    VBT_ERR_PARSE_INT = 4,        /* VibratoError::ParseInt        */
    VBT_ERR_DECODE = 5,           /* VibratoError::BincodeDecode   */
    VBT_ERR_ENCODE = 6,           /* VibratoError::BincodeEncode   */
    VBT_ERR_IO = 7,               /* VibratoError::StdIo           */
    VBT_ERR_UTF8 = 8,             /* VibratoError::Utf8            */
    VBT_ERR_UNSUPPORTED = 9,      /* reserved: a recognised input this build cannot run */
    VBT_ERR_PARSE_FLOAT = 10,     /* VibratoError::ParseFloat      */
    VBT_ERR_CUDA = 100,
    VBT_ERR_NO_DEVICE = 101,
    VBT_ERR_INTERNAL = 102
};

typedef struct vbt_dict vbt_dict;           /* vibrato::Dictionary            (dictionary.rs:54-56) */
typedef struct vbt_tokenizer vbt_tokenizer; /* vibrato::Tokenizer             (tokenizer.rs:13-18)  */
typedef struct vbt_result vbt_result;       /* the top_nodes of a batch of Workers (worker.rs:13-19) */

/* One resultant token: what vibrato::token::Token exposes (token.rs:21-92), sentence-relative.
 * left_id / right_id / word_cost are functions of word_idx: vbt_dict_word_param(). */
typedef struct vbt_token {
    uint32_t start_char; /* Token::range_char().start                     token.rs:21-24 */
    uint32_t end_char;   /* Token::range_char().end                                      */
    uint32_t start_byte; /* Token::range_byte().start                     token.rs:28-32 */
    uint32_t end_byte;   /* Token::range_byte().end                                      */
    uint32_t word_idx;   /* Token::word_idx(): lex_type << 30 | word_id   token.rs:43-46; LexType 0 System,
                            1 User, 2 Unknown (dictionary.rs:30-40) */
    int32_t total_cost;  /* Token::total_cost()                           token.rs:89-92 */
} vbt_token;

/* Opt-in compact record (tokenizer option "compact_tokens" = 1): a third less to bring back over PCIe.  The character
 * range (Token::range_char, token.rs:21-24) is not carried: it is the number of characters of the caller's own UTF-8
 * in front of start_byte / end_byte (sentence.rs:40-46 builds the same table), which the host mirrors rebuild lazily. */
typedef struct vbt_token16 {
    uint32_t start_byte; /* Token::range_byte().start                     token.rs:28-32 */
    uint32_t end_byte;   /* Token::range_byte().end                                      */
    uint32_t word_idx;   /* Token::word_idx()                             token.rs:43-46 */
    int32_t total_cost;  /* Token::total_cost()                           token.rs:89-92 */
} vbt_token16;

/* Lattice output (option "lattice"): per lattice node, next to its vbt_token record. */
typedef struct vbt_lattice_link {
    int32_t prev;   /* the node's best predecessor (Node::min_idx, u16-truncated as the backtrack reads it) as an index
                       into the sentence's own node list; -1 for BOS */
    uint32_t flags; /* VBT_NODE_BEST: the node is on the best path; every other bit is 0 */
} vbt_lattice_link;
#define VBT_NODE_BEST 1u

#define VBT_WORD_ID(word_idx) ((word_idx) & 0x3FFFFFFFu)
#define VBT_LEX_TYPE(word_idx) ((word_idx) >> 30)

const char *vbt_last_error(void);
/* Library version string, e.g. "vibrato_b200 0.1.0 (sm_90a)". */
const char *vbt_version(void);

/* ---- Dictionary (host) -------------------------------------------------------------------- */

/* Dictionary::read (dictionary.rs:173-197): `dic` is the zstd-DECODED "VibratoTokenizer 0.5\n" stream. */
int32_t vbt_dict_from_bytes(const uint8_t *dic, size_t n, vbt_dict **out);
/* zstd::Decoder::new(File::open(path)) + Dictionary::read, as tokenize/src/main.rs:59-60 does. */
int32_t vbt_dict_from_zstd_file(const char *path, vbt_dict **out);
/* SystemDictionaryBuilder::from_readers (dictionary/builder.rs:64-89): MeCab-format sources. */
int32_t vbt_dict_from_mecab(const char *lex_csv, size_t lex_len, const char *matrix_def, size_t matrix_len,
                            const char *char_def, size_t char_len, const char *unk_def, size_t unk_len,
                            vbt_dict **out);
/* Same with the connection matrix given densely, matrix[left * num_right + right]
 * (MatrixConnector::new, matrix_connector.rs:18-24). */
int32_t vbt_dict_from_parts(const char *lex_csv, size_t lex_len, const int16_t *matrix, uint32_t num_right,
                            uint32_t num_left, const char *char_def, size_t char_len, const char *unk_def,
                            size_t unk_len, vbt_dict **out);
/* SystemDictionaryBuilder::from_readers_with_bigram_info (dictionary/builder.rs:111-148): the connection
 * costs come from bigram.right / bigram.left / bigram.cost through a RawConnector
 * (connector/raw_connector.rs), or with dual_connector != 0 through a DualConnector
 * (connector/dual_connector.rs:155-213; needs >= 8 feature templates, else VBT_ERR_INVALID_ARGUMENT). */
int32_t vbt_dict_from_bigram(const char *lex_csv, size_t lex_len, const char *bigram_right, size_t right_len,
                             const char *bigram_left, size_t left_len, const char *bigram_cost, size_t cost_len,
                             const char *char_def, size_t char_len, const char *unk_def, size_t unk_len,
                             int32_t dual_connector, vbt_dict **out);
/* Test hook for the reference's scorer vectors: ScorerBuilder::insert x n + build + Scorer::accumulate_cost
 * (raw_connector/scorer.rs:110-168, 255-267); triples = n x (key1, key2, cost). */
int32_t vbt_scorer_accumulate(const int32_t *triples, size_t n_triples, const uint32_t *keys1, const uint32_t *keys2,
                              size_t n_keys, int32_t *cost);
/* mecab::generate_bigram_info (mecab.rs:31-181): converts a trained MeCab model (feature.def, right-id.def,
 * left-id.def, model.def; note the reference's argument order) into the bigram.right / bigram.left / bigram.cost
 * files that vbt_dict_from_bigram reads.  right-id.def supplies bigram.right and left-id.def bigram.left.  A model.def
 * weight w becomes the cost -(w * cost_factor) truncated toward zero and saturated to i32 (NaN gives 0); zero costs
 * are dropped.  A weight f64::from_str rejects fails with VBT_ERR_PARSE_FLOAT.  The three buffers are released with
 * vbt_bytes_free; on error nothing is allocated. */
int32_t vbt_mecab_generate_bigram_info(const char *feature_def, size_t feature_len, const char *right_id_def,
                                       size_t right_id_len, const char *left_id_def, size_t left_id_len,
                                       const char *model_def, size_t model_len, double cost_factor,
                                       uint8_t **bigram_right, size_t *right_n, uint8_t **bigram_left,
                                       size_t *left_n, uint8_t **bigram_cost, size_t *cost_n);
/* Dictionary::write (dictionary.rs:142-150). *out is released with vbt_bytes_free. */
int32_t vbt_dict_write(const vbt_dict *d, uint8_t **out, size_t *n);
/* zstd::Encoder::new(File::create(path), level) + Dictionary::write + finish (compile/src/main.rs:98-100): the
 * `system.dic.zst` every tool reads with -i.  One zstd frame whose header carries the content size; only the
 * decompressed bytes are specified (they equal vbt_dict_write's), not the compressed ones.  Needs libzstd.so.1 at run
 * time.  VBT_ERR_IO when the library is missing, the file cannot be created or a write fails; a partly written file
 * is removed. */
int32_t vbt_dict_write_zstd_file(const vbt_dict *d, const char *path, int32_t level);
void vbt_bytes_free(uint8_t *p);
/* Dictionary::reset_user_lexicon_from_reader (dictionary.rs:209-229); csv == NULL clears it. */
int32_t vbt_dict_set_user_lexicon_csv(vbt_dict *d, const char *csv, size_t n);
void vbt_dict_free(vbt_dict *d);

/* Dictionary::word_feature (dictionary.rs:108-114); *p points into the dictionary. */
int32_t vbt_dict_feature(const vbt_dict *d, uint32_t word_idx, const char **p, size_t *len);
/* Dictionary::word_param (dictionary.rs:98-104) -> Token::{left_id,right_id,word_cost} (token.rs:64-85). */
int32_t vbt_dict_word_param(const vbt_dict *d, uint32_t word_idx, uint16_t *left_id, uint16_t *right_id,
                            int16_t *word_cost);
/* Connector::{num_left,num_right} (connector.rs:12-18), lexicon sizes (lex_type 0/1/2). */
int32_t vbt_dict_shape(const vbt_dict *d, uint32_t *num_left, uint32_t *num_right, uint32_t *n_system,
                       uint32_t *n_user, uint32_t *n_unknown);
/* Audit of a lexicon as loaded (lex_type 0 system / 1 user), for dictionaries whose byte layout no reference test
 * pins (tools/validate_dic.py): walks every key of the WordMap's trie (map.rs:33-42, trie.rs:49-56) and looks it up
 * again through the common-prefix search.  out[0] keys, out[1] words (Lexicon::params, lexicon.rs:24-29), out[2]
 * word ids named by the postings of those keys (posting.rs:18-21), out[3] longest key in characters, out[4] keys the
 * search does not find again, out[5] word ids named by no key or by more than one.  A sound lexicon has
 * out[1] == out[2] and out[4] == out[5] == 0. */
int32_t vbt_dict_audit(const vbt_dict *d, int32_t lex_type, uint64_t *out, size_t n_out);
/* Lexicon::common_prefix_iterator (lexicon.rs:33-46) on the host copy: (word_id, end_char) pairs in
 * the order the tokenizer sees them.  *n_out receives the full count even when it exceeds cap. */
int32_t vbt_dict_common_prefix(const vbt_dict *d, int32_t lex_type, const uint32_t *chars, size_t n_chars,
                               uint32_t *word_ids, uint32_t *end_chars, size_t cap, size_t *n_out);

/* Dictionary::map_connection_ids_from_iter (dictionary.rs:245-259): lmap / rmap list the OLD left / right ids in
 * their NEW order (the i-th item, 1-origin, becomes id i; id 0 is reserved), exactly what the `.lmap` / `.rmap`
 * files of the reference's `reorder` tool hold (map/src/main.rs:30-74). */
int32_t vbt_dict_map_connection_ids(vbt_dict *d, const uint16_t *lmap, size_t n_lmap, const uint16_t *rmap,
                                    size_t n_rmap);
/* ConnectorCost::cost (matrix_connector.rs:121-124) and CharProperty::char_info (character.rs:112-116, the
 * packed CharInfo of character.rs:10-24) on the host copy. */
int32_t vbt_dict_conn_cost(const vbt_dict *d, uint16_t right_id, uint16_t left_id, int32_t *cost);
int32_t vbt_dict_char_info(const vbt_dict *d, uint32_t code_point, uint32_t *char_info);
/* CharProperty::cate_id (character.rs:119-124): *id = -1 when the category is not defined. */
int32_t vbt_dict_cate_id(const vbt_dict *d, const char *name, size_t len, int32_t *id);

/* The packed device image of the dictionary (see vibrato_b200/csrc/device_blob.hpp).  Rank 0 packs
 * and uploads it; other ranks receive the same bytes over NCCL and hand the device address to
 * vbt_tokenizer_new_from_device_blob. */
int32_t vbt_dict_blob_size(const vbt_dict *d, uint64_t *n_bytes);
int32_t vbt_dict_pack_blob(const vbt_dict *d, uint8_t *host_dst, uint64_t n_bytes);

/* ---- Tokenizer (device) ------------------------------------------------------------------- */

/* Tokenizer::new(dict).ignore_space(ignore_space)?.max_grouping_len(max_grouping_len)
 * (tokenizer.rs:26-74): uploads the dictionary image to `device` (a CUDA ordinal).
 * Fails with VBT_ERR_INVALID_ARGUMENT when ignore_space is set and char.def has no SPACE
 * category (tokenizer.rs:44-49).  max_grouping_len == 0 means unlimited (tokenizer.rs:67-74). */
int32_t vbt_tokenizer_new(const vbt_dict *d, int32_t ignore_space, uint64_t max_grouping_len, int32_t device,
                          vbt_tokenizer **out);
/* Same, over a dictionary image that already sits in `device`'s memory at d_blob (n_bytes long;
 * e.g. the receive buffer of an NCCL broadcast).  The tokenizer does not take ownership. */
int32_t vbt_tokenizer_new_from_device_blob(uint64_t d_blob, uint64_t n_bytes, int32_t ignore_space,
                                           uint64_t max_grouping_len, int32_t device, vbt_tokenizer **out);
/* One tokenizer over `n_devices` GPUs of this node (SURVEY.md §8(b)-3/4, §8(e); no reference counterpart: a vibrato
 * Worker is one CPU thread, worker.rs:13-31 — the contract is BASELINE.json's north_star).  The dictionary image is
 * uploaded once, to devices[0], and broadcast to the others (ncclBroadcast when libnccl.so.2 can be loaded, peer
 * copies otherwise).  vbt_tokenize_batch cuts the batch into contiguous shards of about equal bytes, runs one
 * engine per device on its own host thread (pinned to the GPU's NUMA node) and returns ONE result in input order,
 * identical to a single-device one, the text of the output stage ("output_mode") included: each device formats its
 * shard.  vbt_tokenize_batch_device expects its input on devices[0] and gathers the token records back to it over
 * NVLink (ncclSend / ncclRecv).  Not available on such a tokenizer: a caller-owned stream.  A device listed more than
 * once runs one shard per entry on it (peer copies in place of NCCL): this runs the sharded path on one GPU and is
 * not faster. */
int32_t vbt_tokenizer_new_multi(const vbt_dict *d, int32_t ignore_space, uint64_t max_grouping_len,
                                const int32_t *devices, int32_t n_devices, vbt_tokenizer **out);
/* JSON description of how the tokenizer is laid out: {"devices": [...], "dictionary_transport": "nccl 22703" |
 * "cudaMemcpyPeer" | "single device", "token_gather": ..., "numa_pinned": [...]}.  A single-device tokenizer also
 * names the Viterbi kernel that did the work in its last call: "last_viterbi": "k_viterbi" (round 1; every counted
 * run) | "k_viterbi2" (with lower-bound pruning) | "k_viterbi2_unpruned" (viterbi_kernel 2, the Raw and Dual
 * connectors, or a batch holding a sentence of more than 16 000 characters) | "k_small_batch" (the whole call in one
 * kernel, see the option "small_batch") | "none" (no call yet, or no sentence).  Every tokenizer also counts the
 * attempts its last call ran again, by reason (summed over the shards of a multi-device one): "last_reruns": {"pool":
 * the candidate pool outgrew its estimate, "slots": more characters per byte than estimated, "text": a chunk's output
 * text outgrew its buffer}; the options "pool_estimate_permille" and "chars_estimate_permille" set those estimates. */
int32_t vbt_tokenizer_describe(const vbt_tokenizer *t, char *buf, size_t cap);
/* Restricts the calling thread to the CPUs of the NUMA node `device` hangs off (host-side copies of a rank then
 * stay on its socket); never widens the process's own affinity mask. */
int32_t vbt_pin_thread_to_device(int32_t device);
void vbt_tokenizer_free(vbt_tokenizer *t);

/* for each sentence: Worker::reset_sentence + Worker::tokenize (worker.rs:34-55), batched.
 * Sentence i is utf8[byte_offsets[i] .. byte_offsets[i+1]) and must be valid UTF-8 (else
 * VBT_ERR_UTF8, the failure `stdin.lines()` reports at tokenize/src/main.rs:79).  HOST pointers:
 * the call copies the input to the device, runs the kernels and copies the tokens back.
 * An empty sentence yields zero tokens (worker.rs:50-52). */
int32_t vbt_tokenize_batch(vbt_tokenizer *t, const char *utf8, const uint64_t *byte_offsets, uint64_t n_sent,
                           vbt_result **out);
/* As vbt_tokenize_batch, with required token boundaries (no reference counterpart; MeCab's partial analysis, -p,
 * answers the same need).  Sentence i's required boundaries are bnd[bnd_offsets[i] .. bnd_offsets[i+1]): byte offsets
 * into the sentence, sentence-relative like vbt_token.start_byte.
 * Guarantee: no token t of sentence i has t.start_byte < b < t.end_byte for any of its boundaries b.  Apart from that
 * the result is the minimum-cost path of the constrained lattice, chosen and tie-broken as vbt_tokenize_batch does.
 * Definition, in character positions: for a start position sw let lim(sw) be the first boundary after sw (or the
 * sentence's length).  (1) A lexicon word (system or user) that ends after lim(sw) is no candidate and does not
 * count as a match for the unknown-word rule; (2) in gen_unk_words (dictionary/unknown.rs:69-116) the groupable
 * length g becomes min(g, lim(sw) - sw) everywhere, so a boundary ends a character group; (3) the space skip of
 * ignore_space is unchanged: a boundary inside a skipped run of spaces holds trivially; (4) nothing else changes, so
 * the one-character unknown word keeps a path wherever unk.def has entries for the category.  A sentence without
 * boundaries, or with only 0 and its length, gives exactly the tokens of vbt_tokenize_batch, and a batch whose lists
 * are all empty runs the kernels of vbt_tokenize_batch.
 * Input rules: each list is non-decreasing (duplicates count once), every value is <= the sentence's byte length and
 * a value below it sits on a UTF-8 lead byte; bnd_offsets is non-decreasing.  Anything else fails the call with
 * VBT_ERR_INVALID_ARGUMENT; the errors of vbt_tokenize_batch (VBT_ERR_UTF8, bad byte_offsets) take precedence.
 * Works on single- and multi-device tokenizers, on every host route ("chunk_sentences", "small_batch") and with
 * "compact_tokens", "output_mode", output formats and "connid_counting" (which then counts the constrained
 * lattices).  With the measurement hook "counting" on the call fails with VBT_ERR_INVALID_ARGUMENT: its counters
 * describe the unconstrained walk. */
int32_t vbt_tokenize_batch_bounded(vbt_tokenizer *t, const char *utf8, const uint64_t *byte_offsets, uint64_t n_sent,
                                   const uint64_t *bnd_offsets, const uint32_t *bnd, vbt_result **out);
/* Required tokens (MeCab's partial analysis, -p, with feature patterns): a span [start_byte, end_byte) of a sentence
 * that must be exactly one token, optionally one whose feature matches a pattern.  Byte offsets are
 * sentence-relative; pattern is VBT_SPAN_ANY or an index into the call's pattern table. */
#define VBT_SPAN_ANY 0xFFFFFFFFu
typedef struct vbt_span {
    uint32_t start_byte, end_byte, pattern;
} vbt_span;
/* As vbt_tokenize_batch_bounded, with required tokens.  Sentence i's spans are spans[span_offsets[i] ..
 * span_offsets[i+1]); bnd_offsets / bnd may both be null (no explicit boundary), and span_offsets may not.  Pattern k
 * is the bytes patterns[pattern_offsets[k] .. pattern_offsets[k+1]) (n_patterns of them; both pointers may be null
 * when n_patterns is 0).
 * Definition, in character positions, for a span [a, b): (1) a and b are required boundaries, exactly as in
 * vbt_tokenize_batch_bounded; (2) no lattice node ends strictly inside the span; (3) where a word starts at a, its
 * candidates are the user-, then the system-lexicon words of surface [a, b) whose feature matches the pattern, in
 * lattice order; without any, one unknown word over [a, b) per unk.def entry of the category of character a that
 * matches (all of the category's entries when none matches), whatever max_grouping_len and the category's
 * invoke / group / length say; (4) a pattern is split into fields like a feature (csv); a word matches when each
 * pattern field that is not exactly "*" equals the word's field of the same index byte for byte, and a field the
 * word lacks never matches; an empty pattern matches every word; (5) the space skip of ignore_space is unchanged;
 * (6) nothing else changes.  Guarantee: each span is exactly one token, no token starts or ends inside it, and when
 * some lexicon word of its surface matches the pattern, the token is one of them.  The token keeps its word's own
 * feature (MeCab would print the pattern).
 * Input rules, checked on the device: within a sentence spans are sorted and do not overlap (adjacent is allowed);
 * start < end <= the sentence's byte length, both on a UTF-8 lead byte or at the end; pattern is VBT_SPAN_ANY or
 * below n_patterns; no explicit boundary lies strictly inside a span; with ignore_space no span starts at a SPACE
 * character; span_offsets is non-decreasing.  Anything else fails with VBT_ERR_INVALID_ARGUMENT, after the errors of
 * vbt_tokenize_batch_bounded.  Patterns are compiled on the host: at most 16 constrained fields and field indices up
 * to 255 (VBT_ERR_INVALID_ARGUMENT naming the pattern and byte position).  A batch whose span lists are all empty is
 * the bounded (or the plain) call.  Works on single- and multi-device tokenizers, on the whole-batch and chunked host
 * routes ("small_batch" steps aside), with marginals, the lattice, sampling, output modes and formats,
 * "compact_tokens" and "connid_counting"; "counting" refuses it. */
int32_t vbt_tokenize_batch_spans(vbt_tokenizer *t, const char *utf8, const uint64_t *byte_offsets, uint64_t n_sent,
                                 const uint64_t *bnd_offsets, const uint32_t *bnd, const uint64_t *span_offsets,
                                 const vbt_span *spans, const char *patterns, const uint64_t *pattern_offsets,
                                 uint64_t n_patterns, vbt_result **out);
/* Worker::num_tokens / token(i) / token_iter (worker.rs:59-74) for the whole batch:
 * tokens of sentence i are toks[tok_offsets[i] .. tok_offsets[i+1]), in sentence order. */
int32_t vbt_result_view(const vbt_result *r, const uint64_t **tok_offsets, const vbt_token **toks,
                        uint64_t *n_sent, uint64_t *n_tokens);
/* The same for a batch tokenised with the option "compact_tokens" = 1 (vbt_result_view refuses such a result and this
 * call refuses a full one).  With that option vbt_tokenize_batch_device's d_tokens are vbt_token16 records too. */
int32_t vbt_result_view_compact(const vbt_result *r, const uint64_t **tok_offsets, const vbt_token16 **toks,
                                uint64_t *n_sent, uint64_t *n_tokens);
/* The output loop of `tokenize` (tokenize/src/main.rs:83-127) for the whole batch, formatted on the device when the
 * tokenizer option "output_mode" was 1 (mecab: `surface\tfeature\n`.. `EOS\n`), 2 (wakati: surfaces joined by ' ',
 * `\n`) or 3 (detail: mecab + lex_type/left_id/right_id/word_cost/total_cost) during vbt_tokenize_batch: sentence i's
 * lines are text[text_offsets[i] .. text_offsets[i+1]).  Available on every host route: whole batches, the chunked
 * pipeline of large batches and multi-device tokenizers, with the same bytes on each.  VBT_ERR_INVALID_ARGUMENT when
 * the option was off.  vbt_tokenize_batch_device produces tokens only, on single- and multi-device tokenizers. */
int32_t vbt_result_text(const vbt_result *r, const uint64_t **text_offsets, const char **text, uint64_t *n_bytes);
/* The loop of the `evaluate` tool (evaluate/src/main.rs:61-138): corpus = `surface\tfeature` lines with `EOS`
 * between sentences (Corpus::from_reader, trainer/corpus.rs:78-121); every sentence (its surfaces concatenated) is
 * tokenised in one batch and compared with the corpus as sets of (char range, features[feature_indices]) — all
 * features when n_indices == 0, "*" for a missing index.  Precision = num_cor / num_sys, recall = num_cor / num_ref.
 * `d` must be the dictionary `t` was created from. */
int32_t vbt_evaluate(const vbt_dict *d, vbt_tokenizer *t, const char *corpus, size_t len, const uint64_t *feature_indices,
                     size_t n_indices, uint64_t *num_ref, uint64_t *num_sys, uint64_t *num_cor);
void vbt_result_free(vbt_result *r);

/* Device-resident variant: d_utf8 / d_byte_offsets are DEVICE addresses of the same two arrays
 * (n_bytes = byte_offsets[n_sent]); results stay in device memory owned by the tokenizer and are
 * valid until its next call: *d_tok_offsets -> uint64[n_sent+1], *d_tokens -> vbt_token[*n_tokens]. */
int32_t vbt_tokenize_batch_device(vbt_tokenizer *t, uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent,
                                  uint64_t n_bytes, uint64_t *d_tok_offsets, uint64_t *d_tokens,
                                  uint64_t *n_tokens);
/* As vbt_tokenize_batch_device with the required boundaries of vbt_tokenize_batch_bounded; d_bnd_offsets
 * (uint64[n_sent+1]) and d_bnd (uint32[n_bnd]) are DEVICE addresses, and every offset must be <= n_bnd.  A
 * multi-device tokenizer copies the two arrays to the host to cut them into shards. */
int32_t vbt_tokenize_batch_device_bounded(vbt_tokenizer *t, uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent,
                                          uint64_t n_bytes, uint64_t d_bnd_offsets, uint64_t d_bnd, uint64_t n_bnd,
                                          uint64_t *d_tok_offsets, uint64_t *d_tokens, uint64_t *n_tokens);

/* As vbt_tokenize_batch_device with the required tokens of vbt_tokenize_batch_spans: d_bnd_offsets / d_bnd (may be 0:
 * no explicit boundary), d_span_offsets (uint64[n_sent+1]) and d_spans (vbt_span[n_spans]) are DEVICE addresses, every
 * offset must be <= its array's length; the patterns stay in HOST memory. */
int32_t vbt_tokenize_batch_device_spans(vbt_tokenizer *t, uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent,
                                        uint64_t n_bytes, uint64_t d_bnd_offsets, uint64_t d_bnd, uint64_t n_bnd,
                                        uint64_t d_span_offsets, uint64_t d_spans, uint64_t n_spans,
                                        const char *patterns, const uint64_t *pattern_offsets, uint64_t n_patterns,
                                        uint64_t *d_tok_offsets, uint64_t *d_tokens, uint64_t *n_tokens);

/* Pinned host memory for callers that want full-speed host<->device copies. */
int32_t vbt_host_alloc(size_t n_bytes, void **out);
void vbt_host_free(void *p);

/* Measurement hooks (bench.py): per-stage device time of the last batch in milliseconds, in the
 * order reported by vbt_stage_names(); number of kernels the last batch launched; and the
 * algorithmic-byte counters U,C,M,T,P,W,E,N,K of SURVEY.md §8(d) measured on the device. */
/* Turns the device-side counters on or off (off by default: they cost an extra walk per position). */
int32_t vbt_tokenizer_set_counting(vbt_tokenizer *t, int32_t on);
/* Tuning knobs (results never change): "lanes_per_sentence" = 4|8|16|32 lanes of a warp per sentence in the
 * Viterbi kernel (default 16), "sort_by_length" = 0|1 (default 0: process sentences in input order),
 * "chunk_sentences" = sentences per chunk of the pipelined host path (default 262144, 0 = off),
 * "dual_stream" = 0|1 (default 0: chunks share one compute stream), "counting" = 0|1,
 * "connid_counting" = 0|1 (see vbt_connid_counts), "output_mode" = 0|1|2|3 (see vbt_result_text; default 0),
 * "small_batch" = N in 0..65536 (default 0 = off): a vbt_tokenize_batch call of at most N sentences and 16 KiB of
 * input, without "counting" or "connid_counting", runs every stage, the text of "output_mode" included, in ONE
 * kernel launch (k_small_batch) with one copy each way and one synchronisation; tokens and text are the same as on
 * the usual route.  vbt_last_launch_count then gives 1 and vbt_last_stage_ms books the whole kernel under
 * "viterbi".  A batch whose candidates or text outgrow the route's fixed scratch runs again on the usual route
 * (describe() names the route that ran).  vbt_tokenize_batch_device and the shards of a multi-device tokenizer
 * keep the usual route.
 * Output options (results change as documented with them): "compact_tokens", "lattice" (see vbt_result_lattice),
 * "sample_text" = 0|1 (default 0; 1: the output text renders the samples, see vbt_tokenizer_set_sampling) and
 * "sample_base" = i in 0..2^32 (default 0: the sentence index at which the calls' draws start, see the same) and
 * "posterior_text" = 0|1 (default 0; 1: the output text renders the posterior path, see vbt_tokenizer_set_posterior). */
int32_t vbt_tokenizer_set_option(vbt_tokenizer *t, const char *name, int64_t value);
/* MeCab-style output formats, rendered on the device in place of the option "output_mode": batches tokenised
 * afterwards carry the text of the format in vbt_result_text, on every host route (whole batch, chunked pipeline,
 * "small_batch", multi-device).  `node` is printed per System / User token, `unk` per Unknown token (NULL: the same
 * as node), `bos` before and `eos` after every sentence (NULL: "" and "EOS\n").  Strings are taken by length, not
 * NUL-terminated.  Directives ("prev" = the previous token of the sentence, or BOS with cost 0 and end byte 0):
 *   %m surface, %M bytes from prev's end to this token's end (skipped spaces + surface), %pS the skipped spaces
 *   only, %H the feature string, %f[N1,N2,..] feature fields joined by TAB, %F<c>[N1,..] joined by the byte or
 *   escape <c> (fields split as the evaluate tool splits them, quotes removed; a field whose text begins with '*',
 *   or that the feature does not have, is left out with its separator), %c / %pw word cost, %pc total cost,
 *   %pn total cost - prev's, %pC total cost - prev's - word cost (both wrapping i32), %ps / %pe start / end byte,
 *   %pl surface bytes, %pL end byte - prev's end byte, %phl / %phr left / right id, %s 0 for System / User and 1 for
 *   Unknown, %S / %L the sentence and its byte length, %% a '%'.  Escapes: \0 \a \b \t \n \v \f \r \s (space)
 *   \\.  bos / eos take only literals, escapes, %%, %S and %L.  An unknown or malformed directive or escape, a
 *   MeCab directive without a value on the best path (%h %t %P %pP %pA %pB %pi %pb %pp), more than 16 distinct field
 *   indices or one above 255 give VBT_ERR_INVALID_ARGUMENT with the directive and its byte position in
 *   vbt_last_error().  A format that references fields builds a table of them on each device (once per call of this
 *   function).  Setting "output_mode" replaces the format; node == NULL switches it off.  Excludes
 *   "compact_tokens". */
int32_t vbt_tokenizer_set_output_format(vbt_tokenizer *t, const char *node, size_t node_len, const char *unk,
                                        size_t unk_len, const char *bos, size_t bos_len, const char *eos,
                                        size_t eos_len);
/* Worker::init_connid_counter / update_connid_counts / compute_connid_probs (worker.rs:77-103): switch
 * the option "connid_counting" on (this zeroes the counters), tokenise the corpus, then read the edge
 * counts of every lattice (Lattice::add_connid_counts, lattice.rs:170-183) in the dictionary's own ids:
 * lid_count[num_left], rid_count[num_right].  Pass NULL arrays to query the sizes only. */
int32_t vbt_connid_counts(vbt_tokenizer *t, uint64_t *lid_count, uint64_t *rid_count, uint32_t *num_left,
                          uint32_t *num_right);
/* Marginal probabilities, computed on the device by forward-backward over each sentence's lattice: the nodes the
 * tokenizer inserts (ignore_space, max_grouping_len, the user lexicon and required boundaries included) plus BOS and
 * EOS.  Node k of row ends[p] has an edge to every candidate c starting at p, of cost conn(k.right, c.left) +
 * word_cost(c), and every node of the last row an edge to EOS of cost conn(k.right, 0) (conn: the dictionary's
 * connector value, the matrix i16 or the Raw / Dual i32 sum).  A path's cost is the exact (unwrapped) sum of its
 * edges; P(path) = exp(-theta * cost) / Z over all BOS -> EOS paths.  A token's marginal is the sum of P over the
 * paths through its lattice node; a sentence's path_prob = exp(-theta * min cost) / Z, the probability of one
 * minimum-cost path (1 for an empty sentence).  Nodes without a path to EOS have probability 0.
 * Where the tokenizer's own i32 path costs wrap (very long sentences, extreme Raw / Dual dictionaries) the tokens
 * keep the reference's arithmetic while the probabilities stay the exact-cost ones above.  Whether this theta has
 * the scale of MeCab's -theta is not verified.
 * theta > 0 switches them on, 0 off; negative, NaN or infinite: VBT_ERR_INVALID_ARGUMENT.  While on, batches take
 * two more kernel launches (booked under the "viterbi" stage) and the "small_batch" route steps aside.  The
 * probabilities are bit-identical across routes, chunking, sentence order and K3 variants. */
int32_t vbt_tokenizer_set_marginals(vbt_tokenizer *t, double theta);
/* token_prob[n_tokens] (at the tokens' own indices) and path_prob[n_sent] of a result tokenised with marginals on;
 * owned by the result.  VBT_ERR_INVALID_ARGUMENT for a result made without them. */
int32_t vbt_result_marginals(const vbt_result *r, const float **token_prob, const float **path_prob);
/* Device addresses (float32) of the marginals of the last vbt_tokenize_batch_device{,_bounded} call, valid until the
 * next call; VBT_ERR_INVALID_ARGUMENT when it ran without marginals. */
int32_t vbt_last_device_marginals(const vbt_tokenizer *t, uint64_t *d_token_prob, uint64_t *d_path_prob);
/* Segmentation uncertainty, the option "uncertainty" of vbt_tokenizer_set_option: 0 off (default); 1 every result
 * also carries entropy and log_path_prob per sentence; 2 also the boundary probabilities of every character position.
 * Lattice, edges, exact int64 path costs, theta and P(path) are those of the marginals above (over the constrained
 * lattice in bounded and span calls); â / b̂ / â(EOS) / R(EOS) as in the marginals' forward-backward pass.
 *   entropy[s] (float64, nats) = -sum over paths of P ln P = ln Z + theta * E[cost], computed as
 *   â(EOS) + theta * E[delta]: every edge k -> c (c = EOS included, with R(EOS) in place of R(c)) has the slack
 *   delta = R(k) + cost(k -> c) - R(c) >= 0 against the prefix minima R, which telescopes along a path to
 *   cost - R(EOS); E[delta] = sum over edges of P(edge) delta(edge).  Both terms are sums of non-negative values.
 *   An empty sentence, or one without a path, gives 0.
 *   log_path_prob[s] (float64) = -â(EOS) = ln(exp(-theta * min cost) / Z) <= 0, the log form of path_prob (which
 *   underflows to 0 past about 103 nats); path_prob[s] == float32(exp(log_path_prob[s])) to 1 float32 ulp.  An empty
 *   sentence gives 0, one without a path -inf.
 *   Boundary probabilities (level 2): boundary_offsets[n_sent + 1] (the slot offsets) index boundary_prob (float32);
 *   sentence s owns n_chars + 1 entries, one per character position p = 0..n.  Entry p = P(some token of the path
 *   ends at p) = the sum of the marginals of the nodes of ends[p], summed in float64 in row order and rounded once;
 *   1 at p = 0 (BOS).  A sentence without a path has all entries 0, an empty sentence one entry, 1.  So a required
 *   boundary or span end has an entry within 2 ulps of 1, every position strictly inside a span 0, positions the sweep
 *   skips 0, and the sum over p >= 1 is the expected number of tokens.
 * Every sum runs in a fixed order: all three arrays are bit-identical across routes, chunk sizes, sentence orders, K3
 * variants and device counts.  A non-zero value while marginals are off, switching marginals off while it is on, or a
 * value outside 0..2: VBT_ERR_INVALID_ARGUMENT.  Level 1 runs the marginals' backward pass in an instantiation that
 * also sums P * delta; level 2 adds one kernel launch (both booked under "viterbi").  The "small_batch" route steps
 * aside while it is on.  Multi-device tokenizers give the bytes of one device. */
/* entropy[n_sent], log_path_prob[n_sent] and, at level 2, boundary_offsets[n_sent + 1] into boundary_prob (NULL at
 * level 1) of a result made with "uncertainty"; owned by the result.  VBT_ERR_INVALID_ARGUMENT for a result made
 * without it. */
int32_t vbt_result_uncertainty(const vbt_result *r, const double **entropy, const double **log_path_prob,
                               const uint64_t **boundary_offsets, const float **boundary_prob);
/* Device addresses of the same arrays of the last vbt_tokenize_batch_device* call (boundary arrays 0 and n_positions 0
 * at level 1), valid until the next call; VBT_ERR_INVALID_ARGUMENT when it ran without the option. */
int32_t vbt_last_device_uncertainty(const vbt_tokenizer *t, uint64_t *d_entropy, uint64_t *d_log_path_prob,
                                    uint64_t *d_boundary_offsets, uint64_t *d_boundary_prob, uint64_t *n_positions);
/* Lattice output, the option "lattice" of vbt_tokenizer_set_option: 0 off (default); 1 every result also carries
 * every node of each sentence's lattice; 2 the same, and the output text ("output_mode" 1-3 or a format) renders the
 * nodes in place of the tokens, like MeCab's -a (BOS / EOS formats still print once per sentence).  Multi-device
 * tokenizers give the bytes of one device.
 *   Nodes: the entries of the reference's Lattice::ends once build_lattice has finished, without BOS and EOS; exactly
 *   the nodes the tokenizer inserts (ignore_space, max_grouping_len, the user lexicon and required boundaries
 *   included), dead ends and nodes ending inside a trailing space run included.  An empty sentence has none.
 *   Order: by end character position, then in insertion order (Lattice::ends[e]).  This is not MeCab's start order.
 *   Record: a vbt_token record, always 24 bytes (also under "compact_tokens"), with start_char = the node's start_word,
 *   total_cost = Node::min_cost (the tokenizer's wrapping i32), and a vbt_lattice_link.
 *   Guarantee: the nodes with VBT_NODE_BEST set, in node order, equal the sentence's token records byte for byte.
 *   With marginals on, node_prob[k] is the node's marginal (vbt_tokenizer_set_marginals); on the best path it equals
 *   token_prob bit for bit.
 * While on, batches take three more kernel launches and a scan (booked under "viterbi"), "small_batch" steps aside,
 * and with 2 a format may not print the "prev" directives %M %pS %pn %pC %pL (setting either order fails).
 *
 * Near-best lattice, the option "lattice_margin" = D (0 <= D <= 2^62; -1 = off, the default; it changes nothing while
 * "lattice" is 0).  Edges and exact int64 path costs are those of the marginals.  For a node n, F(n) is the least cost
 * of a path from BOS to n (the edge into n included), G(n) the least cost from n to EOS (the edges after n; undefined
 * without such a path), best the least cost of the sentence, and margin(n) = F(n) + G(n) - best >= 0 (0 on every
 * minimum-cost path).  The lattice group then keeps:
 *   Nodes: every node with a path to EOS and margin(n) <= D, and every node flagged VBT_NODE_BEST (where the
 *   tokenizer's i32 costs wrap, a best-path node can have margin > 0: it is kept, so the guarantee above holds).  An
 *   empty sentence, or one without a path, keeps none.  Without i32 wrap the kept set is the union of the nodes of
 *   every BOS -> EOS path of cost <= best + D; with D = 2^62 it is every node that has a path to EOS.
 *   Order and record: as above, restricted to the kept nodes.
 *   Link: prev is the index, in the kept list, of the node the full lattice's link names; -1 for BOS, -2 when that
 *   node was not kept (only where i32 costs wrap or a row holds more than 65 536 entries).  flags as above.
 *   node_margin[k]: the node's exact margin (vbt_result_lattice_margins).  node_prob is unchanged in meaning.
 * Margins are integers: the kept set is the same on every route, chunk size, sentence order and device count.  With the
 * margin on, batches take two or three more kernel launches (booked under "viterbi"). */
/* node_offsets[n_sent + 1] into nodes / links / node_prob (NULL without marginals) of a result made with the lattice;
 * owned by the result.  VBT_ERR_INVALID_ARGUMENT for a result made without it. */
int32_t vbt_result_lattice(const vbt_result *r, const uint64_t **node_offsets, const vbt_token **nodes,
                           const vbt_lattice_link **links, const float **node_prob, uint64_t *n_nodes);
/* Device addresses of the lattice of the last vbt_tokenize_batch_device{,_bounded} call (d_node_prob 0 without
 * marginals), valid until the next call; VBT_ERR_INVALID_ARGUMENT when it ran without the lattice. */
int32_t vbt_last_device_lattice(const vbt_tokenizer *t, uint64_t *d_node_offsets, uint64_t *d_nodes, uint64_t *d_links,
                                uint64_t *d_node_prob, uint64_t *n_nodes);
/* node_margin[n_nodes] (int64, indexed like nodes) of a result made with the lattice and "lattice_margin" >= 0; owned by
 * the result.  VBT_ERR_INVALID_ARGUMENT for a result made without them. */
int32_t vbt_result_lattice_margins(const vbt_result *r, const int64_t **node_margin);
/* Device address of the node margins of the last vbt_tokenize_batch_device* call, valid until the next call;
 * VBT_ERR_INVALID_ARGUMENT when it ran without the lattice or without "lattice_margin". */
int32_t vbt_last_device_lattice_margins(const vbt_tokenizer *t, uint64_t *d_node_margin);
/* Segmentation sampling ("subword regularisation"): n paths per sentence drawn independently, with replacement, from
 * P(path) = exp(-theta * cost(path)) / Z over the lattice, edges and exact int64 path costs of the marginals above.
 * Forward-filtering backward-sampling on the device: a walk starts at EOS and repeats until BOS.  At the current
 * node c (EOS: left id 0, word cost 0) the candidates are the entries k = 0..K-1 of the row c starts at, in row
 * order: x_k = R(k) + conn(right(k), left(c)) + wcost(c) (R the exact least cost from BOS), r = min x_k,
 * t_k = a(k) - theta * (x_k - r) (a the forward log weight of the marginals), m = max t_k, w_k = exp(t_k - m).  The
 * walk takes the first k whose running sum w_0 + ... + w_k (float64, in row order) exceeds u * S, S the whole sum,
 * and the last k with w_k > 0 if rounding leaves none.  u = ((x0 >> 5) * 2^26 + (x1 >> 6)) * 2^-53 from the first
 * two words of Philox4x32-10 (standard constants) at counter (t, j, i, 0) and key (seed & 0xFFFFFFFF, seed >> 32):
 * t the draw step (0 at EOS), j the sample, i = sample_base + the sentence's index in the call (the option
 * "sample_base", default 0).  Routes (chunking, devices, the sentence order) do not change i, so the same call with
 * the same seed gives the same bytes everywhere; callers who split a corpus over several calls set "sample_base" to
 * each call's first index and draw what one call over the whole corpus would.  A call with sample_base + n_sent > 2^32
 * fails.
 *   Records: each sampled token is a 24-byte vbt_token record, also under "compact_tokens"; start_char, bytes, word_idx
 *   as for tokens, total_cost the sampled path's prefix cost through the token in the tokenizer's wrapping i32
 *   arithmetic.  A sample whose nodes are the best path's has records byte-identical to the sentence's tokens.
 *   An empty sentence, or one without a path, gets n empty samples; nodes without a path to EOS are never sampled.
 * n = 1..1024 switches it on and 0 off; theta must be > 0 and finite; a call with n_sent * n >= 2^32 fails.
 * Marginals and sampling share one forward pass: setting either while the other is on with a different theta is
 * VBT_ERR_INVALID_ARGUMENT.  Tokens, marginals, the lattice and the output text do not change.  While on, batches
 * take three more kernel launches and a scan (the forward pass alone when marginals are off; booked under
 * "viterbi") with one host wait for the sample total, and "small_batch" steps aside.
 * Sample text, the option "sample_text" = 1 (default 0), needs sampling on: with an output mode or format set, the
 * output text renders each sentence's n samples, in order j = 0 .. n-1, in place of its best path.  Each sample is
 * rendered exactly as a sentence whose tokens are its records (BOS format, a node / unk rendering per record, EOS
 * format; -O mecab / wakati / detail likewise), so a sample whose records equal the sentence's tokens renders to the
 * bytes of the sentence's text without sample text, and an empty sample renders as an empty sentence does ("\n" in
 * wakati, "EOS\n" in mecab).  text_offsets keep n_sent + 1 entries: the text of sentence i is its n renderings one
 * after another.  %pc and detail's total_cost print the record's total_cost (the sampled path's prefix cost); the
 * "prev" directives %M %pS %pn %pC %pL take the previous record of the same sample (BOS for its first); %S and %L
 * the sentence.  %pP and %pb have no value: a format that prints them and sample text refuse each other in either
 * order, naming the directive and its byte position.  Sample text and "lattice" = 2 exclude each other, and
 * switching sampling off while sample text is on fails (switch it off first).  Every host route renders it (whole
 * batch, chunked pipeline, multi-device, bounded calls); vbt_tokenize_batch_device stays token-only.  Tokens,
 * samples, marginals and the lattice do not change. */
int32_t vbt_tokenizer_set_sampling(vbt_tokenizer *t, uint32_t n, double theta, uint64_t seed);
/* sample_offsets[n_sent * n + 1] into samples: sample j of sentence i is samples[sample_offsets[i * n + j] ..
 * sample_offsets[i * n + j + 1]); owned by the result.  VBT_ERR_INVALID_ARGUMENT for a result made without sampling. */
int32_t vbt_result_samples(const vbt_result *r, const uint64_t **sample_offsets, const vbt_token **samples,
                           uint64_t *n_sample_tokens);
/* Device addresses of the samples of the last vbt_tokenize_batch_device{,_bounded} call, valid until the next call;
 * VBT_ERR_INVALID_ARGUMENT when it ran without sampling. */
int32_t vbt_last_device_samples(const vbt_tokenizer *t, uint64_t *d_sample_offsets, uint64_t *d_samples,
                                uint64_t *n_sample_tokens);
/* Posterior decoding (maximum expected accuracy, gamma-centroid): per sentence the path whose tokens have the largest
 * total gain, chosen from the marginals above, which must be on.  Lattice, edges and theta are those of the marginals
 * (the constrained lattice in bounded and span calls).  A node is valid when it has a path to EOS (from the integer
 * graph, not from p).  For a valid node, p(n) is the float32 value vbt_result_lattice publishes as its node_prob,
 * exp(â + b̂ - â(EOS)), and gain(n) = (g1 * p(n)) - 1 in float64 with g1 = gamma + 1 computed once and each operation
 * rounded to nearest (no fused multiply-add).  Equivalently a token earns p - 1/(gamma + 1); gamma = 1 is the
 * centroid estimator, larger gammas favour recall, smaller ones precision.
 *   Sweep over character positions: V(0) = 0 (BOS); for q = 1..n in order, over the entries e of ends[q] in row order,
 *   with s(e) the position e starts at: if e is valid and V(s(e)) > -inf, x(e) = V(s(e)) + gain(e), one add.  V(q) is
 *   the largest x, A(q) the first entry in row order that attains it (V(q) = -inf and no A(q) without one).  The path
 *   is A(EOS's row), A(s(that node)), ... back to BOS; predecessors are chosen by position, never through the
 *   u16-truncated min_idx.
 *   posterior_offsets[n_sent + 1] index posterior_tokens: 24-byte vbt_token records (also under "compact_tokens") with
 *   start_char = the node's start_word, bytes and word_idx as for tokens, and total_cost the posterior path's prefix
 *   cost through the token in the tokenizer's wrapping i32 arithmetic; posterior_probs[k] = p of token k (float32);
 *   posterior_gains[n_sent] (float64) = V at EOS: 0 for an empty sentence, -inf for one without a path (both without
 *   tokens).
 * Guarantees: the tokens are a BOS -> EOS path of the (constrained) lattice; posterior_gains[s] is the left fold
 * ((0 + gain_1) + gain_2) + ... over the chosen path, and so at least that fold over every path, the best path's
 * included; where the chosen nodes are the best path's, the records equal the sentence's tokens byte for byte and
 * posterior_probs equals token_prob bit for bit; max is exact and every node takes one add in a fixed order, so all
 * four arrays are bit-identical across routes, chunk sizes, sentence orders, K3 variants and device counts.  Tokens,
 * marginals, the lattice, the samples, the uncertainty and the text (unless "posterior_text" is on) do not change.
 * on != 0 switches it on with gamma (>= 0, finite), 0 off.  VBT_ERR_INVALID_ARGUMENT: a negative or non-finite gamma,
 * switching it on while marginals are off, switching marginals off while it is on, switching it off while
 * "posterior_text" is on.  While on, batches take two more kernel launches and a scan (booked under "viterbi"), the
 * marginals' forward pass keeps each node's left id and word cost, and "small_batch" steps aside.
 * Posterior text, the option "posterior_text" = 1 (default 0), needs posterior decoding on: with an output mode or
 * format set, the output text renders each sentence's posterior path in place of its best path, through the same
 * renderer (%pP prints the token's p, %pc and detail's total_cost its prefix cost, the "prev" directives take the
 * previous posterior token).  It excludes "lattice" = 2 and "sample_text" in either order; %pb stays an error.  Every
 * host route renders it; vbt_tokenize_batch_device stays token-only. */
int32_t vbt_tokenizer_set_posterior(vbt_tokenizer *t, int32_t on, double gamma);
/* posterior_offsets[n_sent + 1] into posterior_tokens / posterior_probs, and posterior_gains[n_sent], of a result made
 * with posterior decoding; owned by the result.  VBT_ERR_INVALID_ARGUMENT for a result made without it. */
int32_t vbt_result_posterior(const vbt_result *r, const uint64_t **posterior_offsets, const vbt_token **posterior_tokens,
                             const float **posterior_probs, const double **posterior_gains, uint64_t *n_posterior_tokens);
/* Device addresses of the same arrays of the last vbt_tokenize_batch_device* call, valid until the next call;
 * VBT_ERR_INVALID_ARGUMENT when it ran without posterior decoding. */
int32_t vbt_last_device_posterior(const vbt_tokenizer *t, uint64_t *d_posterior_offsets, uint64_t *d_posterior_tokens,
                                  uint64_t *d_posterior_probs, uint64_t *d_posterior_gains, uint64_t *n_posterior_tokens);
/* Launch the kernels on a caller-owned CUDA stream (a cudaStream_t passed as an integer; 0 restores
 * the tokenizer's own stream), so callers can bracket batches with their own events. */
int32_t vbt_tokenizer_set_stream(vbt_tokenizer *t, uint64_t stream);
int32_t vbt_last_stage_ms(const vbt_tokenizer *t, float *ms, int32_t cap, int32_t *n_stages);
const char *vbt_stage_names(void);
int32_t vbt_last_launch_count(const vbt_tokenizer *t, uint64_t *n_launches);
/* cnt10 = U,C,M,T,P,W,E,N,K,walks of the last batch run with counting on. */
int32_t vbt_last_counters(const vbt_tokenizer *t, uint64_t *cnt10);

#ifdef __cplusplus
}
#endif
#endif
