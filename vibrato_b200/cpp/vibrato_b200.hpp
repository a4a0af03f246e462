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
    mutable std::shared_ptr<vbt_tokenizer> h_;
};

class Token {  // token.rs:8-92
   public:
    Token(const Tokenizer* t, std::string_view sentence, vbt_token rec) : t_(t), s_(sentence), r_(rec) {}
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
};

class Worker {  // worker.rs:13-74
   public:
    explicit Worker(const Tokenizer* t) : t_(t) {}
    void reset_sentence(std::string_view s) {
        sent_.assign(s);
        toks_.clear();
    }
    void tokenize() {
        if (sent_.empty()) return;  // worker.rs:50-52
        uint64_t off[2] = {0, sent_.size()};
        BatchResult r = t_->tokenize_batch(sent_.data(), off, 1);
        toks_.assign(r.tokens(), r.tokens() + r.n_tokens());
    }
    size_t num_tokens() const { return toks_.size(); }
    Token token(size_t i) const { return Token(t_, sent_, toks_[i]); }

   private:
    const Tokenizer* t_;
    std::string sent_;
    std::vector<vbt_token> toks_;
};

inline Worker Tokenizer::new_worker() const { return Worker(this); }

}  // namespace vibrato_b200
