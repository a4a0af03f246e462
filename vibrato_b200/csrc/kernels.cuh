// Device-side views and kernel declarations of the batched Viterbi tokenizer (sm_90a).
//
// Flattened "slot" space: sentence s with n_s characters owns slots [slot_off[s], slot_off[s]+n_s];
// the last one is a sentinel standing for character position n_s (the `ends[len]` row of
// vibrato's Lattice, tokenizer/lattice.rs:38-43).  All per-character arrays are indexed by slot.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "format.hpp"

namespace vbt {

struct DictView {
    const uint32_t* chr2inf;
    uint32_t chr2inf_len;
    const uint32_t* sys_table;
    uint32_t sys_table_len;
    const uint4* sys_nodes;  // {base, check, postings index of the key ending here or kNone, its word count}
    uint32_t sys_num_nodes;
    const uint4* sys_post;  // per key {len,0,0,0} then len candidate records {left|right<<16, cost word, word_idx, 0}
    const uint32_t* usr_table;  // nullptr when there is no user lexicon
    uint32_t usr_table_len;
    const uint4* usr_nodes;
    uint32_t usr_num_nodes;
    const uint4* usr_post;
    const uint32_t* unk_off;
    const uint2* unk_ent;  // {left | right << 16, cost}
    const int16_t* matrix;  // connector_kind 0 (MatrixConnector); the reduced matrix of connector_kind 2
    uint32_t num_right;     // row length of the reduced matrix (connector_kind 2)
    uint32_t conn_stride_left, conn_stride_right;  // connector_kind 0: cost = matrix[left * sl + right * sr]
    uint32_t opaque_zero;    // always 0; a value the compiler cannot fold (k_viterbi2 uses it to order its loads)
    uint32_t matrix_window;  // connector_kind 0: 1 = the matrix does not cross a 4 GiB address boundary (k_viterbi2)
    // connector_kind 1 (RawConnector, connector/raw_connector.rs + raw_connector/scorer.rs)
    uint32_t connector_kind;
    const uint32_t* right_feats;  // [num_right][feat_T]
    const uint32_t* left_feats;   // [num_left][feat_T]
    uint32_t feat_T;
    const uint32_t* sc_bases;
    const uint32_t* sc_checks;
    const int32_t* sc_costs;
    uint32_t n_bases, n_checks;
    // connector_kind 2 (DualConnector, connector/dual_connector.rs): connection id -> column / row of `matrix`,
    // plus the raw fields above with feat_T == 8
    const uint16_t* right_conn;
    const uint16_t* left_conn;
    // output stage: per lexicon type (0 system, 1 user, 2 unknown) features and dictionary-id parameters by word id
    const uint32_t* feat_off[3];
    const uint8_t* feat[3];
    const uint2* params[3];  // {left | right << 16, word_cost (i16, sign-extended in the low half)}
    uint32_t n_words[3];
    uint32_t space_mask;         // 1 << cate_id("SPACE") when ignore_space, else 0 (tokenizer.rs:16,42-55)
    unsigned long long max_grouping;  // ~0ull when unlimited (tokenizer.rs:17,67-74)
};

enum : uint32_t {
    kFlagUtf8Error = 1u,
    kFlagPoolOverflow = 2u,
    kFlagBadOffsets = 4u,  // byte_off decreases or leaves the input buffer
    // some sentence is so long that path costs may leave +-2^30: k_viterbi2 then runs without its lower-bound
    // pruning, whose arithmetic assumes that no i32 addition wraps
    kFlagLongSentence = 8u,
    // the batch has more characters than the per-character kernels were launched for (the engine sizes those
    // launches from a learned characters-per-byte ratio): later kernels stand down, the engine re-runs the batch
    kFlagSlotsOverflow = 16u,
    // the batch's output text is larger than the text buffer (sized from a learned text-per-byte ratio in the
    // chunked host pipeline): k_format_write wrote nothing, the engine re-runs the batch with a larger buffer
    kFlagTextOverflow = 32u,
    // a required boundary list is out of order, past its sentence's end or inside a multi-byte character, or the
    // boundary offsets themselves are out of order or past n_bnd (k_mark_bounds)
    kFlagBadBoundary = 64u,
    // a required token list is out of order, overlapping, empty-spanned, past its sentence's end, off a UTF-8 lead
    // byte, names no pattern, holds an explicit boundary or (ignore_space) starts at a space, or its offsets are out of
    // order or past n (k_mark_spans)
    kFlagBadSpan = 128u,
};
constexpr uint32_t kFlagsStandDown = kFlagBadOffsets | kFlagSlotsOverflow;
constexpr uint32_t kPruneMaxChars = 16000;  // (chars + 1) nodes x 65 535 per node < 2^30

enum : uint32_t { kInfoTrailing = 1u };  // tokenizer.rs:128-130: the input ends with skipped spaces
constexpr uint32_t kInfoSpecial = 0x80000000u;  // Batch::info[slot].y: info_ex[slot] holds a skip or a flag

constexpr uint32_t kInvalidCode = 0xFFFFFFFFu;
constexpr uint32_t kNone = 0xFFFFFFFFu;

// Counter slots (SURVEY.md §8d) inside Batch::counters
enum { kCntU = 0, kCntC, kCntM, kCntT, kCntP, kCntW, kCntE, kCntN, kCntK, kCntWalks, kNumCounters };

struct Batch {
    // input
    const uint8_t* utf8;
    const unsigned long long* byte_off;  // n_sent + 1
    unsigned long long total_bytes;      // size of the buffer behind utf8: no offset may exceed it
    uint32_t n_sent;
    uint32_t launch_slots;  // slots the per-character launches (K2, the row-offset scan) cover
    // per sentence
    uint32_t* n_slots;   // chars + 1 (scan input)
    uint32_t* slot_off;  // n_sent + 1
    const uint32_t* order;  // sentence processing order of K3 (longest first), or nullptr
    uint4* eos;          // {best prev entry, start_node (sentence-relative), cost, 0}
    uint32_t* n_tok;
    unsigned long long* tok_off;  // n_sent + 1
    // per slot
    uint32_t* code_sys;
    uint32_t* code_usr;
    uint32_t* cinfo;
    uint32_t* groupable;  // 0 marks the sentinel slot
    uint32_t* byte_pos;   // byte offset of the character inside its sentence (c2b, sentence.rs:40-46)
    uint2* info;          // {seg_ptr (first segment in `seg`), cand_cnt | kInfoSpecial}
    uint2* info_ex;       // {skip (start_word - start_node), flags}; written only where info.y has kInfoSpecial
    uint32_t* ends_cnt;   // upper bound of nodes ending here (+1 for BOS at the first slot)
    uint2* ends_meta;     // {exclusive scan of ends_cnt = row offset, next free entry of the row (absolute index)}
    // candidate pool and lattice rows
    // The pool holds per start position the segments of its candidates (kernels.cu, before SegOut): 8 bytes per
    // postings list or unknown-word span, which stand for the records {left | right << 16, word_cost (i16, low half)
    // | lower bound of the connection cost into `left` (i16, high half; see device_blob.hpp), word_idx, end_slot}.
    uint2* seg;
    uint32_t seg_cap;   // segments behind `seg`
    uint32_t cand_cap;  // candidates (= lattice nodes) the rows and the per-node arrays hold, BOS entries aside
    int2* ends_hot;       // lattice rows (CSR over end slot): {min_cost, right_id} — all the DP re-reads
    uint4* ends_cold;     // {start_node slot, best prev entry, word_idx, min_cost} — written once, read by the backtrack
    // output
    void* tokens;  // vbt_token[] (24 bytes each), or vbt_token16[] when compact != 0
    uint32_t compact;  // 1: 16-byte records {start_byte, end_byte, word_idx, total_cost} (character ranges left to the host)
    // bookkeeping
    unsigned long long* pool_ctr;  // candidates of the batch
    unsigned long long* seg_ctr;   // segments of the batch (the pool's allocation counter)
    uint32_t* flags;
    unsigned long long* counters;  // kNumCounters, or nullptr when counting is off
    // ConnIdCounter (mapper.rs:87-104) over internal ids, or nullptr: lid_count[num_left], rid_count[num_right]
    unsigned long long* lid_count;
    unsigned long long* rid_count;
    // Required boundaries (bounded batches only; bnd_dist == nullptr otherwise).  Sentence s's boundaries are the
    // sentence-relative byte offsets bnd[bnd_off[s] .. bnd_off[s+1]); k_mark_bounds turns them into bnd_dist[slot] =
    // (character position of the first boundary after this one, or the sentence's length) - this position, the
    // lim(sw) - sw that k_candidates<true> obeys.
    const unsigned long long* bnd_off;  // n_sent + 1
    const uint32_t* bnd;
    unsigned long long n_bnd;  // entries behind bnd: no offset may exceed it
    uint32_t* bnd_dist;        // per slot, written by k_mark_bounds
};

// Output stage: what `tokenize` prints per sentence (tokenize/src/main.rs:83-127), produced on the device;
// kOutFormat: a MeCab-style format program (format.hpp).
enum : uint32_t { kOutNone = 0, kOutMecab = 1, kOutWakati = 2, kOutDetail = 3, kOutFormat = 4 };
struct FormatArgs {
    const uint8_t* utf8;
    const unsigned long long* byte_off;  // n_sent + 1
    uint32_t n_sent;
    const unsigned long long* tok_off;   // n_sent + 1, indices into `tokens`
    const uint2* tokens;                 // vbt_token as 3 x uint2
    unsigned long long* sent_len;        // n_sent + 1: bytes of each sentence's text, terminator included
    unsigned long long* text_off;        // n_sent + 1: exclusive scan of sent_len, where each sentence's text starts
    uint8_t* text;
    unsigned long long text_cap;         // bytes behind `text`: a larger total sets kFlagTextOverflow instead
    uint32_t* flags;                     // the batch's flags: the stage stands down after an input error or overflow
    unsigned long long* text_total;      // receives text_off[n_sent] (also when it does not fit)
    uint32_t mode;
    // kOutFormat: the compiled program (device memory; every block stages it in shared memory) and the field table
    // of the fields it references.  Words are numbered system, user, unknown in turn (word_global).
    const FormatProgram* prog;
    const uint32_t* ft_keep;  // per word: bit k set = field prog->fields[k] is printed (present, not '*')
    const uint32_t* ft_off;   // per word and k (n_fields per word), + 1: where the field's unquoted text starts
    const uint8_t* ft_bytes;
    // the batch's token marginals (at the token indices of tok_off) when the program prints %pP, else nullptr (this
    // selects the kernels' %pP instantiation; k_small_batch, which never runs with marginals, ignores it)
    const float* token_prob;
};
// links != nullptr (lattice text whose program prints %pb; f.tokens are then the nodes): the %pb instantiation.
void launch_format_len(const DictView& d, const FormatArgs& f, cudaStream_t st, const int2* links = nullptr);
void launch_format_write(const DictView& d, const FormatArgs& f, cudaStream_t st, const int2* links = nullptr);
// Sample text ("sample_text" = 1): the n samples of every sentence rendered in order, each as a sentence whose tokens
// are the walk's records.  f.tok_off / f.tokens are the samples' offsets (n_sent * n + 1) and records; f.sent_len and
// f.text_off have n_sent * n + 1 entries, one per walk s * n + j; the write pass also stores sent_text_off[s] =
// f.text_off[s * n] for s = 0 .. n_sent (not for an empty batch).  The program may not print %pP or %pb.
void launch_format_len_samples(const DictView& d, const FormatArgs& f, uint32_t n, cudaStream_t st);
void launch_format_write_samples(const DictView& d, const FormatArgs& f, uint32_t n, unsigned long long* sent_text_off,
                                 cudaStream_t st);

// Field table of a format program, built once per format and device from the feature strings of the image.
struct FieldTableArgs {
    uint8_t slot_of[kFmtMaxFieldIndex + 1];  // field index -> position k in fields[], 0xFF when not referenced
    uint8_t fields[kFmtMaxFields];
    uint32_t n_fields;
    uint32_t n_words;  // all three lexicons
    uint32_t* lens;    // n_words * n_fields + 1: bytes of each printed field (pass 1)
    uint32_t* keep;    // n_words
    const uint32_t* off;  // exclusive scan of lens (pass 2)
    uint8_t* bytes;
};
void launch_field_table_len(const DictView& d, const FieldTableArgs& a, cudaStream_t st);
void launch_field_table_write(const DictView& d, const FieldTableArgs& a, cudaStream_t st);

// State of the single-pass scans of k_front and k_backtrack: scan_tiles(n_sent, kFrontTile) +
// scan_tiles(n_sent, kBackTileSmall) words of `state` and two ticket counters, all zero before the batch.
struct TileScan {
    unsigned long long* state;
    uint32_t* ticket;
};
constexpr uint32_t kFrontTile = 32, kBackTile = 256, kBackTileSmall = 32;  // sentences per tile
inline uint32_t scan_tiles(uint32_t n_sent, uint32_t tile) { return (n_sent + tile - 1) / tile; }
// count_chars, the slot-offset scan and decode: n_slots, slot_off (n_sent + 1 entries) and every per-slot array.
void launch_front(const DictView& d, const Batch& b, const TileScan& ts, cudaStream_t st);
// Bounded batches (b.bnd_dist != nullptr): writes bnd_dist from the boundary lists after launch_front and
// validates them (kFlagBadBoundary).
void launch_mark_bounds(const Batch& b, cudaStream_t st);
// Required tokens (vbt_tokenize_batch_spans): sentence s's spans are the records rec[off[s] .. off[s+1]), each
// {start byte, end byte, pattern} relative to the sentence, the pattern VBT_SPAN_ANY (kSpanAny) or an index into the
// compiled pattern table.  Pattern p constrains the fields pf[pat_off[p] .. pat_off[p+1]), each {feature field index,
// first byte in pat_bytes, byte length}, sorted by field index: a word matches when each of those fields of its
// feature (csv_fields) equals the bytes.  Passed to k_mark_spans and k_candidates_spans as a separate argument, so
// the Batch of every other kernel stays as it was.  A span batch is a bounded batch (b.bnd_dist, b.bnd_off set).
constexpr uint32_t kSpanAny = 0xFFFFFFFFu;
constexpr uint32_t kSpanInside = 0xFFFFFFFFu;  // SpanArgs::tag[slot].x of a position strictly inside a span
struct SpanArgs {
    const unsigned long long* off;  // n_sent + 1
    const uint3* rec;
    unsigned long long n;           // records behind rec: no offset may exceed it
    const uint32_t* pat_off;        // n_pat + 1
    const uint3* pf;
    const uint8_t* pat_bytes;
    uint32_t n_pat;
    uint32_t space_mask;            // DictView::space_mask: a span may not start at a skipped space
    // per slot, written by k_mark_spans: {0, 0} outside spans, {kSpanInside, 0} strictly inside one, {end - start in
    // characters, pattern} at a span's start
    uint2* tag;
};
// Span batches: marks the boundary lists and the span ends into bnd_dist, writes sp.tag and validates both
// (kFlagBadBoundary, kFlagBadSpan); in place of launch_mark_bounds.
void launch_mark_spans(const Batch& b, const SpanArgs& sp, cudaStream_t st);
// b.bnd_dist != nullptr selects the bounded instantiation of k_candidates: no candidate crosses a marked boundary.
// sp != nullptr (a span batch) selects k_candidates_spans: the bounded candidates, none strictly inside a span, and at
// a span's start only the words of the span's surface that match its pattern (or its unknown words).
void launch_candidates(const DictView& d, const Batch& b, uint32_t max_slots, cudaStream_t st, const SpanArgs* sp = nullptr);
// Counted runs only: per-slot {M | walks << 24, T, P, W} of SURVEY.md §8(d), summed by K3 over visited positions.
void launch_candidate_stats(const DictView& d, const Batch& b, uint32_t max_slots, uint4* stats, cudaStream_t st);
// lanes_per_sentence in {4, 8, 16, 32}: how many lanes of a warp cooperate on one sentence.
// stats != nullptr or b.lid_count != nullptr selects the counting instantiation.
// kernel: 0 = k_viterbi (round 1), 1 = k_viterbi2 (predecessors staged in shared memory, lower-bound pruning),
// 2 = k_viterbi2 without pruning.  Counted runs always use k_viterbi.  Returns the number of kernels launched and
// stores in *route which Viterbi kernel the batch takes.
enum ViterbiRoute : uint32_t {
    kRouteNone = 0,        // empty batch: no Viterbi kernel
    kRouteV1,              // k_viterbi
    kRouteV2,              // k_viterbi2 with pruning
    kRouteV2Unpruned,      // k_viterbi2 without pruning (kernel 2, the Raw / Dual connectors, or the pruned one's twin)
    kRouteSmallBatch,      // k_small_batch: the whole batch in one kernel (launch_small_batch)
    kRouteV2PrunedOrTwin,  // the pruned k_viterbi2 and its twin are both launched: kFlagLongSentence picks one
};
// The kernel that did the work, once the batch's flags are known on the host.
inline ViterbiRoute resolve_viterbi_route(uint32_t launched, uint32_t batch_flags) {
    if (launched == kRouteV2PrunedOrTwin) return (batch_flags & kFlagLongSentence) ? kRouteV2Unpruned : kRouteV2;
    return ViterbiRoute(launched);
}
int launch_viterbi(const DictView& d, const Batch& b, const uint4* stats, int lanes_per_sentence, int kernel,
                   cudaStream_t st, uint32_t* route);

// Marginal probabilities: forward-backward over the lattice K3 left in ends_hot / ends_meta, between K3 and K4
// (K4 overwrites ends_meta).  Per lattice entry n, with R(n) the exact (64-bit) minimum cost from BOS to n:
//   ab[n].x = â(n) = log alpha(n) + theta R(n),   ab[n].y = b̂(n) = log beta(n) + theta (R(EOS) - R(n)),
// so prob(n) = exp(â(n) + b̂(n) - â(EOS)) and path_prob = exp(-â(EOS)).  Every term of the log-sum-exps is
// â - theta * (an exact non-negative integer excess), so the values stay within [-inf, log #paths].  Each node sums
// its terms in one lane in a fixed order (predecessors in row order, candidates in candidate order): the results do
// not depend on the route, the chunking or the sentence order.  The forward pass numbers the candidates' lattice
// entries itself, in the order every K3 variant inserts them (position order, then candidate order).
struct MargArgs {
    double theta;            // > 0
    uint32_t* fill;          // per slot: the row's next free entry while the forward pass numbers the nodes
    uint32_t* ncand;         // per slot: the candidates of a position the sweep visits, 0 elsewhere
    // per candidate of a visited position: its lattice entry; a sentence's are numbered in position order from its
    // first row offset (ends_meta[first slot].x), so the array is as long as the lattice rows
    uint32_t* cand_entry;
    long long* R;            // per lattice entry
    double2* ab;             // per lattice entry: {â, b̂}
    long long* r_eos;        // per sentence: R(EOS)
    double* a_eos;           // per sentence: â(EOS)
    float* path_prob;        // per sentence: exp(-â(EOS)); 1 for an empty sentence
    float* token_prob;       // per token, at the token's index (tok_off)
    // per lattice entry: {left id | word cost (i16) << 16} as the candidate carried them, written by the sampling
    // instantiation of k_marg_forward only (lw != nullptr selects it); BOS's entry is not written
    uint32_t* lw;
};
// Segmentation uncertainty (option "uncertainty"), over the edges, exact path costs and theta of the marginals.  Per
// edge k -> c (c = EOS included, with R(EOS) = r_eos and b̂(EOS) = 0) the slack delta = R(k) + cost(k -> c) - R(c) >= 0
// telescopes along a path to cost - r_eos, so the path entropy is H = â(EOS) + theta * sum_edges P(edge) delta(edge),
// P(k -> c) = exp(â(k) + b̂(c) - theta delta - â(EOS)): two sums of non-negative terms.  The uncertainty instantiation
// of k_marg_backward folds P delta into a float64 per lane (a lane owns the same entries on every route) and reduces
// the warp in a fixed order.  k_boundary_probs writes, per slot, the sum of the marginals of the row's entries
// (float64, in row order, one lane per row, rounded once): P(a token of the path ends at that position).
struct UncertaintyArgs {
    double* entropy;               // per sentence: H (nats); 0 for an empty sentence or one without a path
    double* log_path_prob;         // per sentence: -â(EOS); 0 for an empty sentence, -inf without a path
    unsigned long long* pos_off;   // n_sent + 1: the slot offsets widened, or nullptr (no boundary probabilities)
    float* boundary_prob;          // per slot; 1 at a sentence's first slot (BOS) when it has a path
};
// The instantiations of k_marg_forward: R only (the near-best lattice alone), the log-sum-exp, and the log-sum-exp
// that also writes MargArgs::lw (samples and posterior paths); and of k_marg_backward: plain or uncertainty.
enum FwdKind { kFwdNone, kFwdR, kFwdLse, kFwdLseLw };
enum BwdKind { kBwdNone, kBwdPlain, kBwdUnc };
struct MarginArgs;
// k_marg_forward of kind fwd, k_marg_backward of kind bwd, k_boundary_probs when u.boundary_prob != nullptr, then
// k_margin_backward when g != nullptr; each kind but None is one launch.  u is read by kBwdUnc and k_boundary_probs.
void launch_marginals(const DictView& d, const Batch& b, const MargArgs& m, FwdKind fwd, BwdKind bwd,
                      const UncertaintyArgs& u, const MarginArgs* g, cudaStream_t st);
// backtrack_count, the token-offset scan and backtrack_write: n_tok, tok_off (n_sent + 1 entries) and the token
// records; with m (marginals) also MargArgs::token_prob of every token.
void launch_backtrack(const Batch& b, const MargArgs* m, const TileScan& ts, cudaStream_t st);

// Lattice output: every node K3 inserted (the entries of ends[1..=len] without BOS and EOS), after K3 and the
// marginal kernels and before K4 (which overwrites ends_meta).  A sentence's nodes are listed by end position, and
// within a row in insertion order.  Each node gets a vbt_token record (start_char = its start_word, total_cost = its
// min_cost) and a link {prev, flags}: prev = the sentence-relative node index of the predecessor ends_cold names
// (the u16-truncated min_idx, as the backtrack follows it), -1 for BOS; flags bit 0 (kNodeBest) = on the best path.
enum : uint32_t { kNodeBest = 1u };
struct LatticeArgs {
    uint32_t* row_base;           // per slot: sentence-relative node index of the row's first node (BOS left out)
    uint32_t* n_nodes;            // per sentence (scan input)
    unsigned long long* node_off; // n_sent + 1: exclusive scan of n_nodes
    uint2* nodes;                 // vbt_token as 3 x uint2, always 24 bytes
    int2* links;                  // {prev, flags}
    float* node_prob;             // per node, or nullptr without marginals (then MargArgs is not read)
};

// Near-best lattice (option "lattice_margin" = D >= 0): the lattice output keeps the nodes n with a path to EOS and
// margin(n) = R(n) + G(n) - R(EOS) <= D, and every node of the best path.  G(n) is the least exact (64-bit) cost from
// n to EOS over the edges after it; margins are exact integers, so the kept set does not depend on the route, the
// chunking or the sentence order.  Links name the predecessor's index in the kept list, -2 when it was not kept.
struct MarginArgs {
    long long D;               // 0 .. 2^62
    long long* G;              // per lattice entry; LLONG_MAX = no path to EOS
    uint32_t* keep;            // per lattice entry: the sentence-relative index in the kept list, or kNone
    long long* node_margin;    // per kept node
};
// k_margin_backward (launch_marginals): G of every lattice entry, from the R of any forward pass.
// A warp per sentence; g == nullptr: the full lattice, else the near-best one.
// k_lattice_count: row_base and l.n_nodes; k_lattice_count_margin: g->keep and l.n_nodes (the kept count).  The scan
// of n_nodes then gives l.node_off.
void launch_lattice_count(const Batch& b, const LatticeArgs& l, const MargArgs& m, const MarginArgs* g, cudaStream_t st);
// k_lattice_write<MARGIN>, after the scan: the (kept) nodes' records, links, with g also g->node_margin, and with
// l.node_prob prob = exp(â + b̂ - â(EOS)) as k_backtrack<true> computes it.
void launch_lattice_write(const Batch& b, const LatticeArgs& l, const MargArgs& m, const MarginArgs* g, cudaStream_t st);

// Segmentation sampling: n paths per sentence drawn with replacement from P(path) = exp(-theta cost) / Z, by
// forward-filtering backward-sampling over what k_marg_forward left (R, â and MargArgs::lw), after it and before K4.
// A walk starts at EOS; at node c (EOS: left id 0, word cost 0) its predecessors are the entries k = 0..K-1 of the
// row c starts at, in row order, with x_k = R(k) + conn(right(k), left(c)) + wcost(c), r = min x_k = R(c),
// t_k = â(k) - theta (x_k - r), m = max t_k and w_k = exp(t_k - m).  The walk takes the first k whose running sum
// (float64, in row order) exceeds u * S, S the whole sum (the last k with w_k > 0 if rounding leaves none), where
// u = ((x0 >> 5) 2^26 + (x1 >> 6)) 2^-53 of Philox4x32-10 at counter (t, j, i, 0) and key (seed lo, seed hi):
// t the draw step (0 at EOS), j the sample, i = sent_base + the sentence's index in the batch.  One lane per walk
// (sentence, sample), launched in b.order; a walk's records are 24-byte vbt_token records built as the backtrack
// builds them, with total_cost the sampled path's prefix cost in the tokenizer's wrapping i32 arithmetic.
struct SampleArgs {
    uint32_t n;                     // samples per sentence, 1..1024
    unsigned long long seed;
    unsigned long long sent_base;   // the caller's index of the batch's (chunk's, shard's) first sentence
    uint32_t* cnt;                  // per walk s * n + j (+ 1 for the scan): its tokens
    int32_t* total;                 // per walk: the path's total cost (wrapping i32)
    unsigned long long* off;        // n_sent * n + 1: exclusive scan of cnt
    uint2* out;                     // vbt_token as 3 x uint2
};
// k_sample_count: cnt and total of every walk (an empty sentence, one without a path or a re-run batch: 0).
void launch_sample_count(const DictView& d, const Batch& b, const MargArgs& m, const SampleArgs& s, cudaStream_t st);
// k_sample_write: the same walks again, writing each walk's records at off[walk] from its last token back.
void launch_sample_write(const DictView& d, const Batch& b, const MargArgs& m, const SampleArgs& s, cudaStream_t st);

// Posterior decoding (set_posterior): per sentence the path whose tokens have the largest total gain, over the lattice,
// edges and marginals of k_marg_forward / k_marg_backward, after them and before K4.  A node's p is the float32
// exp(â + b̂ - â(EOS)) that k_lattice_write publishes, its gain (g1 p) - 1 in float64 with g1 = gamma + 1 and no FMA.
// Sweep: V(BOS) = 0; for q = 1 .. EOS's row in order, over the entries e of row q in row order, x(e) = V(s(e)) + gain(e)
// (one round-to-nearest add) where V(s(e)) > -inf, s(e) the row e starts at; V(q) = max x, A(q) = the first entry that
// attains it (-inf / none without one).  The path is A(EOS's row), A(s(that entry)), ... back to BOS.  A node is valid
// when it has a path to EOS; every entry of a row has the same successors, so validity belongs to the row, and a row
// off every path to EOS never feeds V of a row on one: the sweep need not test it.  max is exact and each x is one add
// in a fixed order, so every output is independent of the route, the chunking and the sentence order.
struct PosteriorArgs {
    double g1;                 // gamma + 1, computed on the host
    double* V;                 // per slot: V(q) (scratch)
    uint32_t* A;               // per slot: A(q) (scratch)
    uint32_t* cnt;             // per sentence (+ 1 for the scan): the path's tokens
    int32_t* total;            // per sentence: the path's total cost (wrapping i32)
    unsigned long long* off;   // n_sent + 1: exclusive scan of cnt
    uint2* out;                // vbt_token as 3 x uint2, always 24 bytes; total_cost = the prefix cost (wrapping i32)
    float* prob;               // per token: its p
    double* gain;              // per sentence: V at EOS; 0 for an empty sentence, -inf without a path
};
// k_posterior_sweep (a warp per sentence in b.order): V, A, gain, cnt and total (0 for every sentence of a re-run batch).
// Needs MargArgs::lw (the sampling instantiation of k_marg_forward) for the prefix costs.
void launch_posterior_sweep(const DictView& d, const Batch& b, const MargArgs& m, const PosteriorArgs& p, cudaStream_t st);
// k_posterior_write (a thread per sentence), after the scan of cnt: the records and probabilities from the last back.
void launch_posterior_write(const DictView& d, const Batch& b, const MargArgs& m, const PosteriorArgs& p, cudaStream_t st);

// What k_small_batch reports besides its outputs: the batch flags and the totals of its scans.
struct SmallBatchOut {
    uint32_t flags;
    uint32_t total_slots;
    unsigned long long n_tokens;
    unsigned long long text_bytes;  // 0 unless f.mode != kOutNone
    unsigned long long reserved;
};
// Every stage from count_chars to backtrack_write, and the output stage when f.mode != kOutNone, for a whole batch
// in ONE launch of one thread block.  Inputs as for the separate kernels except: b.flags and f.flags are ignored
// (the kernel keeps the flags in shared memory and reports them in *out), b.order / counters / lid_count must be
// null, b.launch_slots, b.pool_ctr and b.seg_ctr are unused, and the per-slot arrays must hold n_bytes + n_sent + 1
// entries (the hard bound), so only the candidate pool (b.seg_cap segments, b.cand_cap candidates; ends_hot / ends_cold
// need cand_cap + n_sent + 1 entries) and the text (f.text_cap) can overflow: kFlagPoolOverflow / kFlagTextOverflow,
// the outputs are then void.
// f.tok_off / f.tokens must equal b.tok_off / b.tokens; f.sent_len needs n_sent entries, f.text_off n_sent + 1.
// A bounded batch (b.bnd_dist != nullptr, per-slot like the other arrays) is marked and validated inside the block.
void launch_small_batch(const DictView& d, const Batch& b, const FormatArgs& f, SmallBatchOut* out, cudaStream_t st);

}  // namespace vbt
