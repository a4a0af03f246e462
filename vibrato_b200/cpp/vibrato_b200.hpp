// Header-only C++17 mirror of vibrato's public API over the C ABI (include/vibrato_b200.h).
//
//   vibrato::Dictionary::read / reset_user_lexicon_from_reader / map_connection_ids_from_iter   dictionary.rs:173,209,245
//   SystemDictionaryBuilder::from_readers / from_readers_with_bigram_info   dictionary/builder.rs:64,111
//   ConnIdCounter::compute_probs   dictionary/mapper.rs:108-146
//   mecab::generate_bigram_info   mecab.rs:31-181
//   vibrato::Tokenizer::new / ignore_space / max_grouping_len / new_worker   tokenizer.rs:26-84
//   vibrato::tokenizer::worker::Worker::reset_sentence / tokenize / num_tokens / token   worker.rs:34-74
//   vibrato::token::Token accessors   token.rs:21-92
// plus Tokenizer::tokenize_batch for whole batches (what the GPU wants).
// (paths relative to /root/reference/vibrato/src/)
#pragma once

#include <algorithm>
#include <cstdint>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <string_view>
#include <utility>
#include <vector>

#include "../../include/vibrato_b200.h"

namespace vibrato_b200 {

struct VibratoError : std::runtime_error {  // errors.rs:11-42
    int32_t code;
    VibratoError(int32_t c, const std::string& m) : std::runtime_error(m), code(c) {}
};

inline void check(int32_t rc) {
    if (rc != VBT_OK) throw VibratoError(rc, vbt_last_error());
}

enum class LexType : uint8_t { System = 0, User = 1, Unknown = 2 };  // dictionary.rs:30-40
inline const char* lex_type_name(LexType t) {
    return t == LexType::System ? "System" : t == LexType::User ? "User" : "Unknown";
}

struct WordIdx {  // word_idx.rs:5-11
    LexType lex_type;
    uint32_t word_id;
    uint32_t packed() const { return (uint32_t(lex_type) << 30) | word_id; }
};

class Dictionary {
   public:
    static Dictionary read(const std::vector<uint8_t>& decoded) {  // dictionary.rs:173
        vbt_dict* h = nullptr;
        check(vbt_dict_from_bytes(decoded.data(), decoded.size(), &h));
        return Dictionary(h);
    }
    static Dictionary read_zstd_file(const std::string& path) {  // tokenize/src/main.rs:59-60
        vbt_dict* h = nullptr;
        check(vbt_dict_from_zstd_file(path.c_str(), &h));
        return Dictionary(h);
    }
    static Dictionary from_readers(std::string_view lex, std::string_view matrix, std::string_view chr,
                                   std::string_view unk) {  // builder.rs:64-89
        vbt_dict* h = nullptr;
        check(vbt_dict_from_mecab(lex.data(), lex.size(), matrix.data(), matrix.size(), chr.data(), chr.size(),
                                  unk.data(), unk.size(), &h));
        return Dictionary(h);
    }
    static Dictionary from_readers_with_bigram_info(std::string_view lex, std::string_view bigram_right,
                                                    std::string_view bigram_left, std::string_view bigram_cost,
                                                    std::string_view chr, std::string_view unk,
                                                    bool dual_connector) {  // builder.rs:111-148
        vbt_dict* h = nullptr;
        check(vbt_dict_from_bigram(lex.data(), lex.size(), bigram_right.data(), bigram_right.size(), bigram_left.data(),
                                   bigram_left.size(), bigram_cost.data(), bigram_cost.size(), chr.data(), chr.size(),
                                   unk.data(), unk.size(), dual_connector ? 1 : 0, &h));
        return Dictionary(h);
    }
    // Dictionary::write into zstd::Encoder::new(File::create(path), level) (compile/src/main.rs:98-100)
    void write_zstd_file(const std::string& path, int32_t level = 19) const {
        check(vbt_dict_write_zstd_file(h_.get(), path.c_str(), level));
    }
    Dictionary reset_user_lexicon_from_reader(const std::string* csv) && {  // dictionary.rs:209; consumes self
        check(vbt_dict_set_user_lexicon_csv(h_.get(), csv ? csv->data() : nullptr, csv ? csv->size() : 0));
        return std::move(*this);
    }
    Dictionary map_connection_ids_from_iter(const std::vector<uint16_t>& lmap,
                                            const std::vector<uint16_t>& rmap) && {  // dictionary.rs:245-259
        check(vbt_dict_map_connection_ids(h_.get(), lmap.data(), lmap.size(), rmap.data(), rmap.size()));
        return std::move(*this);
    }
    std::string_view word_feature(WordIdx w) const {  // dictionary.rs:108
        const char* p = nullptr;
        size_t n = 0;
        check(vbt_dict_feature(h_.get(), w.packed(), &p, &n));
        return {p, n};
    }
    void word_param(WordIdx w, uint16_t& l, uint16_t& r, int16_t& c) const {
        check(vbt_dict_word_param(h_.get(), w.packed(), &l, &r, &c));
    }
    bool has_category(std::string_view name) const {
        int32_t id = -1;
        check(vbt_dict_cate_id(h_.get(), name.data(), name.size(), &id));
        return id >= 0;
    }
    const vbt_dict* raw() const { return h_.get(); }

   private:
    explicit Dictionary(vbt_dict* h) : h_(h, &vbt_dict_free) {}
    std::unique_ptr<vbt_dict, void (*)(vbt_dict*)> h_;
};

namespace mecab {

// The three files mecab::generate_bigram_info writes (bigram.right, bigram.left, bigram.cost), the sources of
// Dictionary::from_readers_with_bigram_info
struct BigramInfo {
    std::string right, left, cost;
};

// mecab::generate_bigram_info (mecab.rs:31-181): a trained MeCab model -> bigram.* files.  The reference's argument
// order: right-id.def supplies bigram.right, left-id.def bigram.left.
inline BigramInfo generate_bigram_info(std::string_view feature_def, std::string_view right_id_def,
                                       std::string_view left_id_def, std::string_view model_def, double cost_factor) {
    uint8_t* p[3] = {};
    size_t n[3] = {};
    check(vbt_mecab_generate_bigram_info(feature_def.data(), feature_def.size(), right_id_def.data(), right_id_def.size(),
                                         left_id_def.data(), left_id_def.size(), model_def.data(), model_def.size(),
                                         cost_factor, &p[0], &n[0], &p[1], &n[1], &p[2], &n[2]));
    using Bytes = std::unique_ptr<uint8_t, void (*)(uint8_t*)>;
    Bytes own[3] = {{p[0], &vbt_bytes_free}, {p[1], &vbt_bytes_free}, {p[2], &vbt_bytes_free}};
    auto text = [&](int i) { return std::string(reinterpret_cast<const char*>(own[i].get()), n[i]); };
    return {text(0), text(1), text(2)};
}

}  // namespace mecab

class BatchResult {
   public:
    explicit BatchResult(vbt_result* r) : r_(r, &vbt_result_free) {
        check(vbt_result_view(r, &off_, &toks_, &n_sent_, &n_tokens_));
    }
    uint64_t n_sent() const { return n_sent_; }
    uint64_t n_tokens() const { return n_tokens_; }
    const uint64_t* tok_offsets() const { return off_; }
    const vbt_token* tokens() const { return toks_; }
    // What `tokenize` prints for the batch (tokenize/src/main.rs:83-127), formatted on the device; needs
    // Tokenizer::output_mode(...) before the batch.  text_offsets()[i] is where sentence i's lines start.
    std::string_view text(const uint64_t** text_offsets = nullptr) const {
        const char* p = nullptr;
        uint64_t n = 0;
        check(vbt_result_text(r_.get(), text_offsets, &p, &n));
        return {p, size_t(n)};
    }
    // Marginal probabilities (Tokenizer::marginals before the batch): float per token, at the tokens' indices, and
    // the best path's probability per sentence.  Throws on a result made without them.
    const float* token_probs() const {
        const float* tp = nullptr;
        check(vbt_result_marginals(r_.get(), &tp, nullptr));
        return tp;
    }
    const float* path_probs() const {
        const float* pp = nullptr;
        check(vbt_result_marginals(r_.get(), nullptr, &pp));
        return pp;
    }
    // Lattice output (Tokenizer::lattice before the batch, see vbt_result_lattice): node_offsets()[i] ..
    // node_offsets()[i + 1] index sentence i's nodes, links and (with marginals, else nullptr) node probabilities.
    // Throws on a result made without the lattice.
    struct Lattice {
        const uint64_t* node_offsets = nullptr;
        const vbt_token* nodes = nullptr;
        const vbt_lattice_link* links = nullptr;
        const float* node_probs = nullptr;
        uint64_t n_nodes = 0;
    };
    Lattice lattice() const {
        Lattice l;
        check(vbt_result_lattice(r_.get(), &l.node_offsets, &l.nodes, &l.links, &l.node_probs, &l.n_nodes));
        return l;
    }
    // The near-best lattice's node margins (Tokenizer::lattice with a margin), indexed like lattice().nodes.  Throws
    // on a result made without them.
    const int64_t* lattice_margins() const {
        const int64_t* m = nullptr;
        check(vbt_result_lattice_margins(r_.get(), &m));
        return m;
    }
    // Segmentation uncertainty (Tokenizer::uncertainty before the batch, see vbt_result_uncertainty): entropy and
    // log_path_prob per sentence; with boundary probabilities, sentence i's positions 0..n are
    // boundary_prob[boundary_offsets[i] .. boundary_offsets[i + 1]) (both nullptr without them).  Throws on a result
    // made without the option.
    struct Uncertainty {
        const double* entropy = nullptr;
        const double* log_path_prob = nullptr;
        const uint64_t* boundary_offsets = nullptr;
        const float* boundary_prob = nullptr;
    };
    Uncertainty uncertainty() const {
        Uncertainty u;
        check(vbt_result_uncertainty(r_.get(), &u.entropy, &u.log_path_prob, &u.boundary_offsets, &u.boundary_prob));
        return u;
    }
    // Segmentation sampling (Tokenizer::sampling before the batch, see vbt_tokenizer_set_sampling): sample j of
    // sentence i is samples[sample_offsets[i * n + j] .. sample_offsets[i * n + j + 1]).  Throws on a result made
    // without sampling.
    struct Samples {
        const uint64_t* sample_offsets = nullptr;
        const vbt_token* samples = nullptr;
        uint64_t n_sample_tokens = 0;
    };
    Samples samples() const {
        Samples s;
        check(vbt_result_samples(r_.get(), &s.sample_offsets, &s.samples, &s.n_sample_tokens));
        return s;
    }
    // Posterior decoding (Tokenizer::posterior before the batch, see vbt_tokenizer_set_posterior): sentence i's path is
    // tokens[offsets[i] .. offsets[i + 1]) with probs at the same indices, and gains[i] its total gain.  Throws on a
    // result made without it.
    struct Posterior {
        const uint64_t* offsets = nullptr;
        const vbt_token* tokens = nullptr;
        const float* probs = nullptr;
        const double* gains = nullptr;
        uint64_t n_tokens = 0;
    };
    Posterior posterior() const {
        Posterior p;
        check(vbt_result_posterior(r_.get(), &p.offsets, &p.tokens, &p.probs, &p.gains, &p.n_tokens));
        return p;
    }

   private:
    std::unique_ptr<vbt_result, void (*)(vbt_result*)> r_;
    const uint64_t* off_ = nullptr;
    const vbt_token* toks_ = nullptr;
    uint64_t n_sent_ = 0, n_tokens_ = 0;
};

// ConnIdProbs (mapper.rs:84): (id, occurrence probability) pairs
using ConnIdProbs = std::vector<std::pair<uint32_t, double>>;

// ConnIdCounter::compute_probs (mapper.rs:108-146) for one side: each count over the sum, id 0 dropped, by descending
// probability then ascending id.  With a zero sum every probability is NaN, no two compare, and the order is by id.
inline ConnIdProbs compute_connid_probs(const std::vector<uint64_t>& counts) {
    uint64_t sum = 0;
    for (uint64_t c : counts) sum += c;
    ConnIdProbs probs;
    for (uint32_t i = 1; i < counts.size(); ++i) probs.emplace_back(i, double(counts[i]) / double(sum));
    std::sort(probs.begin(), probs.end(), [](const auto& a, const auto& b) {
        if (a.second > b.second) return true;
        if (a.second < b.second) return false;
        return a.first < b.first;  // equal, or incomparable (NaN)
    });
    return probs;
}

class Worker;

class Tokenizer {
   public:
    explicit Tokenizer(Dictionary dict, int device = 0) : dict_(std::move(dict)), device_(device) {}  // tokenizer.rs:26
    Tokenizer ignore_space(bool yes) && {  // tokenizer.rs:42-55
        if (yes && !dict_.has_category("SPACE"))
            throw VibratoError(VBT_ERR_INVALID_ARGUMENT, "dict: SPACE is not defined in the input dictionary (i.e., char.def).");
        ignore_space_ = yes;
        return std::move(*this);
    }
    Tokenizer max_grouping_len(size_t n) && {  // tokenizer.rs:67-74
        max_grouping_len_ = n;
        return std::move(*this);
    }
    // Not in the reference: spread every batch over these GPUs of the node (vbt_tokenizer_new_multi); same calls,
    // same results.
    Tokenizer devices(std::vector<int32_t> devs) && {
        devices_ = std::move(devs);
        return std::move(*this);
    }
    const Dictionary& dictionary() const { return dict_; }
    Worker new_worker() const;
    // The loop of the `evaluate` tool (evaluate/src/main.rs:61-138): counts over a `surface\tfeature` / `EOS` corpus
    struct EvalCounts {
        uint64_t num_ref = 0, num_sys = 0, num_cor = 0;
    };
    EvalCounts evaluate(std::string_view corpus, const std::vector<uint64_t>& feature_indices) const {
        EvalCounts c;
        check(vbt_evaluate(dict_.raw(), handle(), corpus.data(), corpus.size(), feature_indices.data(),
                           feature_indices.size(), &c.num_ref, &c.num_sys, &c.num_cor));
        return c;
    }
    // OutputMode of the `tokenize` CLI (tokenize/src/main.rs:12-29): "mecab", "wakati", "detail"; "" = off
    void output_mode(std::string_view mode) const {
        const int64_t m = mode.empty() ? 0 : mode == "mecab" ? 1 : mode == "wakati" ? 2 : mode == "detail" ? 3 : -1;
        if (m < 0) throw VibratoError(VBT_ERR_INVALID_ARGUMENT, "Could not parse a mode");
        check(vbt_tokenizer_set_option(handle(), "output_mode", m));
    }
    // MeCab-style output formats (node / unk / BOS / EOS format strings, see vbt_tokenizer_set_output_format),
    // rendered on the device in place of output_mode(): BatchResult::text().  A null node switches the format off; a
    // null unk prints Unknown tokens with node; null bos / eos print "" / "EOS\n".
    void output_format(const std::string_view* node, const std::string_view* unk = nullptr,
                       const std::string_view* bos = nullptr, const std::string_view* eos = nullptr) const {
        // data() of an empty view may be null, which would read as "not given"
        auto p = [](const std::string_view* s) -> const char* { return !s ? nullptr : s->empty() ? "" : s->data(); };
        auto n = [](const std::string_view* s) { return s ? s->size() : size_t(0); };
        check(vbt_tokenizer_set_output_format(handle(), p(node), n(node), p(unk), n(unk), p(bos), n(bos), p(eos), n(eos)));
    }
    // Batches of at most n sentences and 16 KiB run in one kernel launch (k_small_batch), with the same tokens and
    // text; counted runs keep the usual route.  0 = off (the default).
    void small_batch(uint32_t n = 64) const { check(vbt_tokenizer_set_option(handle(), "small_batch", int64_t(n))); }
    // Marginal probabilities at temperature theta > 0 (0 = off; see vbt_tokenizer_set_marginals): BatchResult::
    // token_probs / path_probs, Token::prob().  Set it before an output format that prints %pP.
    void marginals(double theta) const {
        check(vbt_tokenizer_set_marginals(handle(), theta));
        marginals_ = theta > 0;
    }
    // Device addresses {token_prob, path_prob} (float) of the last tokenize_batch_device call, valid until the next.
    std::pair<uint64_t, uint64_t> last_device_marginals() const {
        uint64_t tp = 0, pp = 0;
        check(vbt_last_device_marginals(handle(), &tp, &pp));
        return {tp, pp};
    }
    bool has_marginals() const { return marginals_; }
    // Segmentation uncertainty (the option "uncertainty", see vbt_result_uncertainty; needs marginals):
    // BatchResult::uncertainty(); boundary_probs = true also carries each character position's boundary probability.
    void uncertainty(bool on = true, bool boundary_probs = false) const {
        const int level = on ? (boundary_probs ? 2 : 1) : 0;
        check(vbt_tokenizer_set_option(handle(), "uncertainty", level));
        uncertainty_ = level;
    }
    int uncertainty_level() const { return marginals_ ? uncertainty_ : 0; }
    // Device addresses of the last tokenize_batch_device call's uncertainty (the boundary arrays 0 at level 1).
    struct DeviceUncertainty {
        uint64_t entropy = 0, log_path_prob = 0, boundary_offsets = 0, boundary_prob = 0, n_positions = 0;
    };
    DeviceUncertainty last_device_uncertainty() const {
        DeviceUncertainty d;
        check(vbt_last_device_uncertainty(handle(), &d.entropy, &d.log_path_prob, &d.boundary_offsets, &d.boundary_prob,
                                          &d.n_positions));
        return d;
    }
    // Lattice output (the option "lattice", see vbt_result_lattice): BatchResult::lattice(); text = true also renders
    // the nodes in place of the tokens in the output text (MeCab -a).  Set text before a format that prints %pb.
    // margin = D (0 .. 2^62; the option "lattice_margin") keeps only the nodes within cost D of the best path, plus the
    // best path, with BatchResult::lattice_margins(); -1 keeps every node.
    void lattice(bool on = true, bool text = false, int64_t margin = -1) const {
        check(vbt_tokenizer_set_option(handle(), "lattice_margin", margin));
        check(vbt_tokenizer_set_option(handle(), "lattice", on ? (text ? 2 : 1) : 0));
        lattice_ = on;
        margin_ = margin >= 0;
    }
    bool has_lattice() const { return lattice_; }
    bool has_lattice_margins() const { return lattice_ && margin_; }
    // Device addresses of the last tokenize_batch_device call's lattice (node_prob 0 without marginals).
    struct DeviceLattice {
        uint64_t node_offsets = 0, nodes = 0, links = 0, node_probs = 0, n_nodes = 0;
    };
    DeviceLattice last_device_lattice() const {
        DeviceLattice d;
        check(vbt_last_device_lattice(handle(), &d.node_offsets, &d.nodes, &d.links, &d.node_probs, &d.n_nodes));
        return d;
    }
    // Segmentation sampling (see vbt_tokenizer_set_sampling): n (1..1024, 0 = off) paths per sentence drawn from
    // P(path) at temperature theta, keyed by seed: BatchResult::samples().  theta must equal the marginals' when both
    // are on.  text = true also renders the samples in place of the best path in the output text (the option
    // "sample_text"): n renderings per sentence, one after another.  Set text before a format is set.
    void sampling(uint32_t n, double theta, uint64_t seed = 0, bool text = false) const {
        if (!text) check(vbt_tokenizer_set_option(handle(), "sample_text", 0));  // before sampling may switch off
        check(vbt_tokenizer_set_sampling(handle(), n, theta, seed));
        if (text) check(vbt_tokenizer_set_option(handle(), "sample_text", 1));
        samples_ = n;
    }
    uint32_t samples_per_sentence() const { return samples_; }
    // The draws of the next calls' sentence s use the sentence index i + s (the option "sample_base"), so that a
    // corpus tokenised over several calls draws what one call over all of it would.  i + n_sent <= 2^32.
    void sample_base(uint64_t i) const { check(vbt_tokenizer_set_option(handle(), "sample_base", int64_t(i))); }
    // Device addresses of the last tokenize_batch_device call's samples.
    struct DeviceSamples {
        uint64_t sample_offsets = 0, samples = 0, n_sample_tokens = 0;
    };
    DeviceSamples last_device_samples() const {
        DeviceSamples d;
        check(vbt_last_device_samples(handle(), &d.sample_offsets, &d.samples, &d.n_sample_tokens));
        return d;
    }
    // Posterior decoding (see vbt_tokenizer_set_posterior; needs marginals): BatchResult::posterior(), each sentence's
    // path of the largest total gain at weight gamma >= 0.  text = true also renders it in place of the best path in
    // the output text (the option "posterior_text").  on = false switches both off.
    void posterior(bool on, double gamma = 1.0, bool text = false) const {
        if (!text) check(vbt_tokenizer_set_option(handle(), "posterior_text", 0));  // before posterior may switch off
        check(vbt_tokenizer_set_posterior(handle(), on ? 1 : 0, gamma));
        if (text) check(vbt_tokenizer_set_option(handle(), "posterior_text", 1));
    }
    // Device addresses of the last tokenize_batch_device call's posterior paths.
    struct DevicePosterior {
        uint64_t offsets = 0, tokens = 0, probs = 0, gains = 0, n_tokens = 0;
    };
    DevicePosterior last_device_posterior() const {
        DevicePosterior d;
        check(vbt_last_device_posterior(handle(), &d.offsets, &d.tokens, &d.probs, &d.gains, &d.n_tokens));
        return d;
    }
    // Worker::init_connid_counter / update_connid_counts / compute_connid_probs (worker.rs:77-103): after
    // init_connid_counter() every batch is counted, an empty sentence counting nothing
    void init_connid_counter() const { check(vbt_tokenizer_set_option(handle(), "connid_counting", 1)); }
    std::pair<ConnIdProbs, ConnIdProbs> compute_connid_probs() const {
        uint32_t nl = 0, nr = 0;
        check(vbt_connid_counts(handle(), nullptr, nullptr, &nl, &nr));
        std::vector<uint64_t> lid(nl), rid(nr);
        check(vbt_connid_counts(handle(), lid.data(), rid.data(), nullptr, nullptr));
        return {vibrato_b200::compute_connid_probs(lid), vibrato_b200::compute_connid_probs(rid)};
    }

    BatchResult tokenize_batch(const char* utf8, const uint64_t* byte_offsets, uint64_t n_sent) const {
        vbt_result* r = nullptr;
        check(vbt_tokenize_batch(handle(), utf8, byte_offsets, n_sent, &r));
        return BatchResult(r);
    }
    // With required boundaries: sentence i's are the byte offsets bnd[bnd_offsets[i] .. bnd_offsets[i+1]).
    BatchResult tokenize_batch(const char* utf8, const uint64_t* byte_offsets, uint64_t n_sent, const uint64_t* bnd_offsets,
                               const uint32_t* bnd) const {
        vbt_result* r = nullptr;
        check(vbt_tokenize_batch_bounded(handle(), utf8, byte_offsets, n_sent, bnd_offsets, bnd, &r));
        return BatchResult(r);
    }
    // With required tokens (vbt_tokenize_batch_spans): sentence i's spans are spans[span_offsets[i] .. span_offsets[i+1]),
    // pattern k the bytes patterns[pattern_offsets[k] .. pattern_offsets[k+1]); bnd_offsets / bnd may be null.
    BatchResult tokenize_batch(const char* utf8, const uint64_t* byte_offsets, uint64_t n_sent, const uint64_t* bnd_offsets,
                               const uint32_t* bnd, const uint64_t* span_offsets, const vbt_span* spans,
                               const char* patterns, const uint64_t* pattern_offsets, uint64_t n_patterns) const {
        vbt_result* r = nullptr;
        check(vbt_tokenize_batch_spans(handle(), utf8, byte_offsets, n_sent, bnd_offsets, bnd, span_offsets, spans, patterns,
                                       pattern_offsets, n_patterns, &r));
        return BatchResult(r);
    }
    // Device-resident batches (device addresses in, device addresses of the results out; see vibrato_b200.h).
    void tokenize_batch_device(uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent, uint64_t n_bytes,
                               uint64_t& d_tok_offsets, uint64_t& d_tokens, uint64_t& n_tokens) const {
        check(vbt_tokenize_batch_device(handle(), d_utf8, d_byte_offsets, n_sent, n_bytes, &d_tok_offsets, &d_tokens,
                                        &n_tokens));
    }
    void tokenize_batch_device(uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent, uint64_t n_bytes,
                               uint64_t d_bnd_offsets, uint64_t d_bnd, uint64_t n_bnd, uint64_t& d_tok_offsets,
                               uint64_t& d_tokens, uint64_t& n_tokens) const {
        check(vbt_tokenize_batch_device_bounded(handle(), d_utf8, d_byte_offsets, n_sent, n_bytes, d_bnd_offsets, d_bnd,
                                                n_bnd, &d_tok_offsets, &d_tokens, &n_tokens));
    }
    // With required tokens: d_span_offsets / d_spans are device addresses, the patterns host memory.
    void tokenize_batch_device(uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent, uint64_t n_bytes,
                               uint64_t d_bnd_offsets, uint64_t d_bnd, uint64_t n_bnd, uint64_t d_span_offsets,
                               uint64_t d_spans, uint64_t n_spans, const char* patterns, const uint64_t* pattern_offsets,
                               uint64_t n_patterns, uint64_t& d_tok_offsets, uint64_t& d_tokens, uint64_t& n_tokens) const {
        check(vbt_tokenize_batch_device_spans(handle(), d_utf8, d_byte_offsets, n_sent, n_bytes, d_bnd_offsets, d_bnd, n_bnd,
                                              d_span_offsets, d_spans, n_spans, patterns, pattern_offsets, n_patterns,
                                              &d_tok_offsets, &d_tokens, &n_tokens));
    }

   private:
    vbt_tokenizer* handle() const {
        if (!h_) {
            vbt_tokenizer* h = nullptr;
            if (devices_.empty())
                check(vbt_tokenizer_new(dict_.raw(), ignore_space_ ? 1 : 0, max_grouping_len_, device_, &h));
            else
                check(vbt_tokenizer_new_multi(dict_.raw(), ignore_space_ ? 1 : 0, max_grouping_len_, devices_.data(),
                                              int32_t(devices_.size()), &h));
            h_.reset(h, &vbt_tokenizer_free);
        }
        return h_.get();
    }
    Dictionary dict_;
    int device_;
    std::vector<int32_t> devices_;
    bool ignore_space_ = false;
    uint64_t max_grouping_len_ = 0;
    mutable bool marginals_ = false;
    mutable bool lattice_ = false;
    mutable bool margin_ = false;  // lattice(..., margin >= 0)
    mutable int uncertainty_ = 0;  // uncertainty(): 0, 1 or 2
    mutable uint32_t samples_ = 0;
    mutable std::shared_ptr<vbt_tokenizer> h_;
};

class Token {  // token.rs:8-92
   public:
    // prob: the token's marginal probability, or NaN when the tokenizer computes none
    Token(const Tokenizer* t, std::string_view sentence, vbt_token rec, float prob = std::numeric_limits<float>::quiet_NaN())
        : t_(t), s_(sentence), r_(rec), p_(prob) {}
    std::pair<size_t, size_t> range_char() const { return {r_.start_char, r_.end_char}; }
    std::pair<size_t, size_t> range_byte() const { return {r_.start_byte, r_.end_byte}; }
    std::string_view surface() const { return s_.substr(r_.start_byte, r_.end_byte - r_.start_byte); }
    WordIdx word_idx() const { return {LexType(r_.word_idx >> 30), r_.word_idx & 0x3FFFFFFFu}; }
    LexType lex_type() const { return word_idx().lex_type; }
    std::string_view feature() const { return t_->dictionary().word_feature(word_idx()); }
    uint16_t left_id() const { return param().l; }
    uint16_t right_id() const { return param().r; }
    int16_t word_cost() const { return param().c; }
    int32_t total_cost() const { return r_.total_cost; }
    float prob() const {  // Tokenizer::marginals
        if (p_ != p_)
            throw VibratoError(VBT_ERR_INVALID_ARGUMENT, "no marginals: switch them on with Tokenizer::marginals before tokenising");
        return p_;
    }

   private:
    struct P {
        uint16_t l, r;
        int16_t c;
    };
    P param() const {
        P p{};
        t_->dictionary().word_param(word_idx(), p.l, p.r, p.c);
        return p;
    }
    const Tokenizer* t_;
    std::string_view s_;
    vbt_token r_;
    float p_;
};

// One node of a sentence's lattice (Tokenizer::lattice): Token's accessors (start_char = start_word, total_cost =
// min_cost), plus its best predecessor, best-path flag, marginal and, in a near-best lattice, margin.
class LatticeNode : public Token {
   public:
    LatticeNode(const Tokenizer* t, std::string_view sentence, vbt_token rec, vbt_lattice_link link,
                float prob = std::numeric_limits<float>::quiet_NaN(), int64_t margin = -1)
        : Token(t, sentence, rec, prob), link_(link), margin_(margin) {}
    // index in the sentence's node list, -1 for BOS, -2 for a predecessor a near-best lattice did not keep
    int32_t prev() const { return link_.prev; }
    bool is_best() const { return (link_.flags & VBT_NODE_BEST) != 0; }
    // the exact cost margin over the best path (Tokenizer::lattice with a margin); throws without one
    int64_t margin() const {
        if (margin_ < 0) throw VibratoError(VBT_ERR_INVALID_ARGUMENT, "no margins: pass a margin to Tokenizer::lattice before tokenising");
        return margin_;
    }

   private:
    vbt_lattice_link link_;
    int64_t margin_;
};

class Worker {  // worker.rs:13-74
   public:
    explicit Worker(const Tokenizer* t) : t_(t) {}
    void reset_sentence(std::string_view s) {
        sent_.assign(s);
        bnd_.clear();
        bounded_ = false;
        spans_.clear();
        patterns_.clear();
        pat_off_.assign(1, 0);
        toks_.clear();
        nodes_.clear();
        links_.clear();
        nprobs_.clear();
        samples_.clear();
    }
    // With required boundaries (byte offsets into s; see Tokenizer::tokenize_batch).
    void reset_sentence(std::string_view s, std::vector<uint32_t> boundaries) {
        reset_sentence(s);
        bnd_ = std::move(boundaries);
        bounded_ = true;
    }
    // With required tokens as well: spans (byte ranges into s) whose pattern indexes `patterns` or is VBT_SPAN_ANY.
    void reset_sentence(std::string_view s, std::vector<uint32_t> boundaries, std::vector<vbt_span> spans,
                        const std::vector<std::string>& patterns) {
        reset_sentence(s, std::move(boundaries));
        spans_ = std::move(spans);
        for (const std::string& p : patterns) {
            patterns_ += p;
            pat_off_.push_back(patterns_.size());
        }
    }
    void tokenize() {
        samples_.assign(t_->samples_per_sentence(), {});
        const int level = t_->uncertainty_level();
        has_unc_ = level != 0;
        bprobs_.clear();
        if (sent_.empty()) {  // worker.rs:50-52; the one empty path has no uncertainty and ends where it starts
            entropy_ = log_path_prob_ = 0.0;
            if (level >= 2) bprobs_.assign(1, 1.f);
            return;
        }
        uint64_t off[2] = {0, sent_.size()};
        uint64_t boff[2] = {0, bnd_.size()};
        uint64_t soff[2] = {0, spans_.size()};
        BatchResult r = !spans_.empty() ? t_->tokenize_batch(sent_.data(), off, 1, boff, bnd_.data(), soff, spans_.data(),
                                                             patterns_.data(), pat_off_.data(), pat_off_.size() - 1)
                        : bounded_      ? t_->tokenize_batch(sent_.data(), off, 1, boff, bnd_.data())
                                        : t_->tokenize_batch(sent_.data(), off, 1);
        toks_.assign(r.tokens(), r.tokens() + r.n_tokens());
        probs_.clear();
        if (t_->has_marginals() && r.n_tokens()) probs_.assign(r.token_probs(), r.token_probs() + r.n_tokens());
        nodes_.clear();
        links_.clear();
        nprobs_.clear();
        margins_.clear();
        if (t_->has_lattice()) {
            const BatchResult::Lattice l = r.lattice();
            nodes_.assign(l.nodes, l.nodes + l.n_nodes);
            links_.assign(l.links, l.links + l.n_nodes);
            if (l.node_probs) nprobs_.assign(l.node_probs, l.node_probs + l.n_nodes);
            if (t_->has_lattice_margins() && l.n_nodes) {
                const int64_t* m = r.lattice_margins();
                margins_.assign(m, m + l.n_nodes);
            }
        }
        if (has_unc_) {
            const BatchResult::Uncertainty u = r.uncertainty();
            entropy_ = u.entropy[0];
            log_path_prob_ = u.log_path_prob[0];
            if (u.boundary_prob) bprobs_.assign(u.boundary_prob + u.boundary_offsets[0], u.boundary_prob + u.boundary_offsets[1]);
        }
        if (!samples_.empty()) {
            const BatchResult::Samples s = r.samples();
            for (size_t j = 0; j < samples_.size(); ++j) samples_[j].assign(s.samples + s.sample_offsets[j], s.samples + s.sample_offsets[j + 1]);
        }
    }
    // Tokenizer::sampling: the tokens of sample j of the sentence (Token::prob() throws on them).
    size_t num_sample_tokens(size_t j) const { return samples_.at(j).size(); }
    Token sample_token(size_t j, size_t i) const { return Token(t_, sent_, samples_.at(j)[i]); }
    size_t num_nodes() const { return nodes_.size(); }
    LatticeNode node(size_t i) const {
        return LatticeNode(t_, sent_, nodes_[i], links_[i], nprobs_.empty() ? std::numeric_limits<float>::quiet_NaN() : nprobs_[i],
                           margins_.empty() ? -1 : margins_[i]);
    }
    // Tokenizer::uncertainty: the sentence's path entropy (nats), ln P(best path) and, with boundary probabilities,
    // P(a token ends at position p) for p = 0..n; each throws without the option.
    double entropy() const {
        need_uncertainty();
        return entropy_;
    }
    double log_path_prob() const {
        need_uncertainty();
        return log_path_prob_;
    }
    const std::vector<float>& boundary_probs() const {
        need_uncertainty();
        if (t_->uncertainty_level() < 2)
            throw VibratoError(VBT_ERR_INVALID_ARGUMENT, "no boundary probabilities: pass boundary_probs to Tokenizer::uncertainty");
        return bprobs_;
    }
    size_t num_tokens() const { return toks_.size(); }
    Token token(size_t i) const {
        return probs_.empty() ? Token(t_, sent_, toks_[i]) : Token(t_, sent_, toks_[i], probs_[i]);
    }

   private:
    void need_uncertainty() const {
        if (!has_unc_) throw VibratoError(VBT_ERR_INVALID_ARGUMENT, "no uncertainty: switch it on with Tokenizer::uncertainty and tokenize first");
    }
    const Tokenizer* t_;
    std::string sent_;
    std::vector<uint32_t> bnd_;
    bool bounded_ = false;
    std::vector<vbt_span> spans_;
    std::string patterns_;
    std::vector<uint64_t> pat_off_{0};
    std::vector<vbt_token> toks_;
    std::vector<float> probs_;
    std::vector<vbt_token> nodes_;  // Tokenizer::lattice
    std::vector<vbt_lattice_link> links_;
    std::vector<float> nprobs_;
    std::vector<int64_t> margins_;  // Tokenizer::lattice with a margin
    bool has_unc_ = false;          // Tokenizer::uncertainty
    double entropy_ = 0.0, log_path_prob_ = 0.0;
    std::vector<float> bprobs_;
    std::vector<std::vector<vbt_token>> samples_;  // Tokenizer::sampling
};

inline Worker Tokenizer::new_worker() const { return Worker(this); }

}  // namespace vibrato_b200
