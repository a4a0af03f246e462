// extern "C" surface of libvibrato_b200.so (include/vibrato_b200.h).
#include "../../include/vibrato_b200.h"

#include <array>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "device_blob.hpp"
#include "engine.hpp"
#include "evaluate.hpp"
#include "host_dict.hpp"

struct vbt_dict {
    vbt::Dictionary d;
    // packed device image, built on first request and dropped once handed out (it can be ~0.5 GB)
    mutable std::vector<uint8_t> image;
    mutable uint64_t image_size = 0;
    const std::vector<uint8_t>& packed() const {
        if (image.empty()) {
            vbt::pack_device_blob(d, image);
            image_size = image.size();
        }
        return image;
    }
    void drop_image() const {
        std::vector<uint8_t>().swap(image);
    }
};
struct vbt_tokenizer {
    std::shared_ptr<vbt::Engine> e;
};
struct vbt_result {
    std::shared_ptr<vbt::Engine> owner;  // keeps the engine (and its pinned pool) alive past vbt_tokenizer_free
    vbt::HostResult* r;
};

namespace {
thread_local std::string g_err;

template <typename F>
int32_t guarded(F&& f) {
    try {
        f();
        g_err.clear();
        return VBT_OK;
    } catch (const vbt::Error& e) {
        g_err = e.what();
        return int32_t(e.code);
    } catch (const std::bad_alloc&) {
        g_err = "out of host memory";
        return VBT_ERR_INTERNAL;
    } catch (const std::exception& e) {
        g_err = e.what();
        return VBT_ERR_INTERNAL;
    }
}

void need(const void* p, const char* what) {
    if (!p) throw vbt::Error(vbt::kInvalidArgument, std::string(what) + " must not be NULL");
}
}  // namespace

extern "C" {

const char* vbt_last_error(void) { return g_err.c_str(); }
const char* vbt_version(void) { return "vibrato_b200 0.1.0 (sm_90a)"; }

int32_t vbt_dict_from_bytes(const uint8_t* dic, size_t n, vbt_dict** out) {
    return guarded([&] {
        need(dic, "dic");
        need(out, "out");
        *out = new vbt_dict{vbt::Dictionary::read(dic, n), {}, 0};
    });
}

int32_t vbt_dict_from_zstd_file(const char* path, vbt_dict** out) {
    return guarded([&] {
        need(path, "path");
        need(out, "out");
        std::vector<uint8_t> raw = vbt::zstd_decompress_file(path);
        *out = new vbt_dict{vbt::Dictionary::read(raw.data(), raw.size()), {}, 0};
    });
}

int32_t vbt_dict_from_mecab(const char* lex_csv, size_t lex_len, const char* matrix_def, size_t matrix_len,
                            const char* char_def, size_t char_len, const char* unk_def, size_t unk_len,
                            vbt_dict** out) {
    return guarded([&] {
        need(out, "out");
        *out = new vbt_dict{vbt::Dictionary::from_mecab({lex_csv, lex_len}, {matrix_def, matrix_len},
                                                       {char_def, char_len}, {unk_def, unk_len}), {}, 0};
    });
}

int32_t vbt_dict_from_parts(const char* lex_csv, size_t lex_len, const int16_t* matrix, uint32_t num_right,
                            uint32_t num_left, const char* char_def, size_t char_len, const char* unk_def,
                            size_t unk_len, vbt_dict** out) {
    return guarded([&] {
        need(out, "out");
        need(matrix, "matrix");
        *out = new vbt_dict{vbt::Dictionary::from_parts({lex_csv, lex_len}, matrix, num_right, num_left,
                                                       {char_def, char_len}, {unk_def, unk_len}), {}, 0};
    });
}

int32_t vbt_dict_from_bigram(const char* lex_csv, size_t lex_len, const char* bigram_right, size_t right_len,
                             const char* bigram_left, size_t left_len, const char* bigram_cost, size_t cost_len,
                             const char* char_def, size_t char_len, const char* unk_def, size_t unk_len,
                             int32_t dual_connector, vbt_dict** out) {
    return guarded([&] {
        need(out, "out");
        *out = new vbt_dict{vbt::Dictionary::from_bigram({lex_csv, lex_len}, {bigram_right, right_len}, {bigram_left, left_len},
                                                        {bigram_cost, cost_len}, {char_def, char_len}, {unk_def, unk_len},
                                                        dual_connector != 0),
                            {}, 0};
    });
}

int32_t vbt_scorer_accumulate(const int32_t* triples, size_t n_triples, const uint32_t* keys1, const uint32_t* keys2,
                              size_t n_keys, int32_t* cost) {
    return guarded([&] {
        need(cost, "cost");
        vbt::RawConnector c;
        std::vector<std::array<int64_t, 3>> t(n_triples);
        for (size_t i = 0; i < n_triples; ++i) t[i] = {int64_t(triples[3 * i]), int64_t(triples[3 * i + 1]), int64_t(triples[3 * i + 2])};
        c.build_scorer(std::move(t));
        *cost = c.accumulate(keys1, keys2, n_keys);
    });
}

int32_t vbt_mecab_generate_bigram_info(const char* feature_def, size_t feature_len, const char* right_id_def,
                                       size_t right_id_len, const char* left_id_def, size_t left_id_len,
                                       const char* model_def, size_t model_len, double cost_factor,
                                       uint8_t** bigram_right, size_t* right_n, uint8_t** bigram_left,
                                       size_t* left_n, uint8_t** bigram_cost, size_t* cost_n) {
    return guarded([&] {
        need(bigram_right, "bigram_right");
        need(right_n, "right_n");
        need(bigram_left, "bigram_left");
        need(left_n, "left_n");
        need(bigram_cost, "bigram_cost");
        need(cost_n, "cost_n");
        vbt::BigramInfoText t = vbt::generate_bigram_info({feature_def, feature_len}, {right_id_def, right_id_len},
                                                          {left_id_def, left_id_len}, {model_def, model_len}, cost_factor);
        const std::string* src[3] = {&t.right, &t.left, &t.cost};
        uint8_t* p[3] = {};
        for (int i = 0; i < 3; ++i) {
            p[i] = static_cast<uint8_t*>(std::malloc(src[i]->size() ? src[i]->size() : 1));
            if (!p[i]) {
                for (int k = 0; k < i; ++k) std::free(p[k]);
                throw std::bad_alloc();
            }
            std::memcpy(p[i], src[i]->data(), src[i]->size());
        }
        *bigram_right = p[0], *right_n = t.right.size();
        *bigram_left = p[1], *left_n = t.left.size();
        *bigram_cost = p[2], *cost_n = t.cost.size();
    });
}

int32_t vbt_dict_write(const vbt_dict* d, uint8_t** out, size_t* n) {
    return guarded([&] {
        need(d, "d");
        need(out, "out");
        need(n, "n");
        std::vector<uint8_t> buf;
        d->d.write(buf);
        uint8_t* p = static_cast<uint8_t*>(std::malloc(buf.size() ? buf.size() : 1));
        if (!p) throw std::bad_alloc();
        std::memcpy(p, buf.data(), buf.size());
        *out = p;
        *n = buf.size();
    });
}

int32_t vbt_dict_write_zstd_file(const vbt_dict* d, const char* path, int32_t level) {
    return guarded([&] {
        need(d, "d");
        need(path, "path");
        std::vector<uint8_t> buf;
        d->d.write(buf);
        vbt::zstd_compress_to_file(buf, path, level);
    });
}

void vbt_bytes_free(uint8_t* p) { std::free(p); }

int32_t vbt_dict_set_user_lexicon_csv(vbt_dict* d, const char* csv, size_t n) {
    return guarded([&] {
        need(d, "d");
        d->drop_image();
        if (csv)
            d->d.reset_user_lexicon(std::string_view(csv, n));
        else
            d->d.reset_user_lexicon(std::nullopt);
    });
}

void vbt_dict_free(vbt_dict* d) { delete d; }

int32_t vbt_dict_feature(const vbt_dict* d, uint32_t word_idx, const char** p, size_t* len) {
    return guarded([&] {
        need(d, "d");
        need(p, "p");
        need(len, "len");
        std::string_view f = d->d.word_feature(word_idx);
        *p = f.data();
        *len = f.size();
    });
}

int32_t vbt_dict_word_param(const vbt_dict* d, uint32_t word_idx, uint16_t* left_id, uint16_t* right_id,
                            int16_t* word_cost) {
    return guarded([&] {
        need(d, "d");
        vbt::WordParam p = d->d.word_param(word_idx);
        if (left_id) *left_id = p.left_id;
        if (right_id) *right_id = p.right_id;
        if (word_cost) *word_cost = p.word_cost;
    });
}

int32_t vbt_dict_shape(const vbt_dict* d, uint32_t* num_left, uint32_t* num_right, uint32_t* n_system, uint32_t* n_user,
                       uint32_t* n_unknown) {
    return guarded([&] {
        need(d, "d");
        if (num_left) *num_left = d->d.num_left();
        if (num_right) *num_right = d->d.num_right();
        if (n_system) *n_system = d->d.system.num_words();
        if (n_user) *n_user = d->d.user ? d->d.user->num_words() : 0;
        if (n_unknown) *n_unknown = uint32_t(d->d.unk.entries.size());
    });
}

int32_t vbt_dict_common_prefix(const vbt_dict* d, int32_t lex_type, const uint32_t* chars, size_t n_chars,
                               uint32_t* word_ids, uint32_t* end_chars, size_t cap, size_t* n_out) {
    return guarded([&] {
        need(d, "d");
        need(n_out, "n_out");
        if (n_chars) need(chars, "chars");
        if (cap) {
            need(word_ids, "word_ids");
            need(end_chars, "end_chars");
        }
        const vbt::Lexicon* lx = lex_type == 0 ? &d->d.system : (lex_type == 1 && d->d.user ? &*d->d.user : nullptr);
        if (!lx) throw vbt::Error(vbt::kInvalidArgument, "no such lexicon");
        std::vector<std::pair<uint32_t, uint32_t>> hits;
        lx->trie.common_prefix_search(reinterpret_cast<const char32_t*>(chars), n_chars, hits);
        size_t k = 0;
        for (auto& h : hits) {
            uint32_t len = lx->postings[h.first];
            for (uint32_t j = 0; j < len; ++j, ++k)
                if (k < cap) {
                    word_ids[k] = lx->postings[h.first + 1 + j];
                    end_chars[k] = h.second;
                }
        }
        *n_out = k;
    });
}

int32_t vbt_dict_audit(const vbt_dict* d, int32_t lex_type, uint64_t* out, size_t n_out) {
    return guarded([&] {
        need(d, "d");
        need(out, "out");
        if (n_out < 6) throw vbt::Error(vbt::kInvalidArgument, "out needs 6 entries");
        const vbt::Lexicon* lx = lex_type == 0 ? &d->d.system : (lex_type == 1 && d->d.user ? &*d->d.user : nullptr);
        if (!lx) throw vbt::Error(vbt::kInvalidArgument, "no such lexicon");
        // every key the trie holds, looked up again through the search the tokenizer uses
        uint64_t keys = 0, listed = 0, longest = 0, missed = 0;
        std::vector<uint8_t> seen(lx->params.size(), 0);
        uint64_t twice = 0;
        std::vector<std::pair<uint32_t, uint32_t>> hits;
        for (auto& kv : lx->trie.enumerate()) {
            ++keys;
            longest = std::max<uint64_t>(longest, kv.first.size());
            lx->trie.common_prefix_search(kv.first.data(), kv.first.size(), hits);
            bool found = false;
            for (auto& h : hits) found = found || (h.second == kv.first.size() && h.first == kv.second);
            if (!found) ++missed;
            if (kv.second < lx->postings.size()) {
                const uint32_t len = lx->postings[kv.second];
                for (uint32_t j = 0; j < len && kv.second + 1 + j < lx->postings.size(); ++j) {
                    const uint32_t id = lx->postings[kv.second + 1 + j];
                    ++listed;
                    if (id < seen.size()) {
                        if (seen[id]) ++twice;
                        seen[id] = 1;
                    }
                }
            }
        }
        uint64_t unlisted = 0;
        for (uint8_t v : seen) unlisted += v ? 0 : 1;
        out[0] = keys;
        out[1] = lx->params.size();
        out[2] = listed;
        out[3] = longest;
        out[4] = missed;
        out[5] = unlisted + twice;
    });
}

int32_t vbt_dict_map_connection_ids(vbt_dict* d, const uint16_t* lmap, size_t n_lmap, const uint16_t* rmap, size_t n_rmap) {
    return guarded([&] {
        need(d, "d");
        if (n_lmap) need(lmap, "lmap");
        if (n_rmap) need(rmap, "rmap");
        d->drop_image();
        d->d.map_connection_ids(std::vector<uint16_t>(lmap, lmap + n_lmap), std::vector<uint16_t>(rmap, rmap + n_rmap));
    });
}

int32_t vbt_dict_conn_cost(const vbt_dict* d, uint16_t right_id, uint16_t left_id, int32_t* cost) {
    return guarded([&] {
        need(d, "d");
        need(cost, "cost");
        if (right_id >= d->d.num_right() || left_id >= d->d.num_left())
            throw vbt::Error(vbt::kInvalidArgument, "connection id out of range");
        *cost = d->d.conn_cost(right_id, left_id);
    });
}

int32_t vbt_dict_char_info(const vbt_dict* d, uint32_t code_point, uint32_t* char_info) {
    return guarded([&] {
        need(d, "d");
        need(char_info, "char_info");
        *char_info = d->d.char_prop.char_info(code_point);
    });
}

int32_t vbt_dict_cate_id(const vbt_dict* d, const char* name, size_t len, int32_t* id) {
    return guarded([&] {
        need(d, "d");
        need(id, "id");
        *id = d->d.char_prop.cate_id(std::string_view(name, len));
    });
}

int32_t vbt_dict_blob_size(const vbt_dict* d, uint64_t* n_bytes) {
    return guarded([&] {
        need(d, "d");
        need(n_bytes, "n_bytes");
        *n_bytes = d->packed().size();  // kept until vbt_dict_pack_blob / vbt_tokenizer_new hands it out
    });
}

int32_t vbt_dict_pack_blob(const vbt_dict* d, uint8_t* host_dst, uint64_t n_bytes) {
    return guarded([&] {
        need(d, "d");
        need(host_dst, "host_dst");
        const std::vector<uint8_t>& blob = d->packed();
        if (blob.size() != n_bytes) throw vbt::Error(vbt::kInvalidArgument, "n_bytes differs from vbt_dict_blob_size");
        std::memcpy(host_dst, blob.data(), blob.size());
        d->drop_image();
    });
}

int32_t vbt_tokenizer_new(const vbt_dict* d, int32_t ignore_space, uint64_t max_grouping_len, int32_t device,
                          vbt_tokenizer** out) {
    return guarded([&] {
        need(d, "d");
        need(out, "out");
        if (ignore_space && d->d.char_prop.cate_id("SPACE") < 0)  // tokenizer.rs:44-49
            throw vbt::Error(vbt::kInvalidArgument, "dict: SPACE is not defined in the input dictionary (i.e., char.def).");
        const std::vector<uint8_t>& blob = d->packed();
        *out = new vbt_tokenizer{std::shared_ptr<vbt::Engine>(vbt::Engine::create(device, blob.data(), 0, blob.size(), ignore_space != 0, max_grouping_len))};
        d->drop_image();
    });
}

int32_t vbt_tokenizer_new_from_device_blob(uint64_t d_blob, uint64_t n_bytes, int32_t ignore_space,
                                           uint64_t max_grouping_len, int32_t device, vbt_tokenizer** out) {
    return guarded([&] {
        need(out, "out");
        *out = new vbt_tokenizer{std::shared_ptr<vbt::Engine>(vbt::Engine::create(device, nullptr, d_blob, n_bytes, ignore_space != 0, max_grouping_len))};
    });
}

int32_t vbt_tokenizer_new_multi(const vbt_dict* d, int32_t ignore_space, uint64_t max_grouping_len, const int32_t* devices,
                                int32_t n_devices, vbt_tokenizer** out) {
    return guarded([&] {
        need(d, "d");
        need(out, "out");
        need(devices, "devices");
        if (n_devices < 1) throw vbt::Error(vbt::kInvalidArgument, "n_devices must be at least 1");
        if (ignore_space && d->d.char_prop.cate_id("SPACE") < 0)  // tokenizer.rs:44-49
            throw vbt::Error(vbt::kInvalidArgument, "dict: SPACE is not defined in the input dictionary (i.e., char.def).");
        const std::vector<uint8_t>& blob = d->packed();
        std::vector<int> devs(devices, devices + n_devices);
        *out = new vbt_tokenizer{std::shared_ptr<vbt::Engine>(
            vbt::Engine::create_multi(devs, blob.data(), blob.size(), ignore_space != 0, max_grouping_len))};
        d->drop_image();
    });
}

int32_t vbt_tokenizer_describe(const vbt_tokenizer* t, char* buf, size_t cap) {
    return guarded([&] {
        need(t, "t");
        need(buf, "buf");
        const std::string s = t->e->describe();
        if (s.size() + 1 > cap) throw vbt::Error(vbt::kInvalidArgument, "buffer too small");
        std::memcpy(buf, s.c_str(), s.size() + 1);
    });
}

int32_t vbt_pin_thread_to_device(int32_t device) {
    return guarded([&] { vbt::pin_thread_to_device_numa_node(device); });
}

void vbt_tokenizer_free(vbt_tokenizer* t) { delete t; }

int32_t vbt_tokenize_batch(vbt_tokenizer* t, const char* utf8, const uint64_t* byte_offsets, uint64_t n_sent,
                           vbt_result** out) {
    return guarded([&] {
        need(t, "t");
        need(out, "out");
        need(byte_offsets, "byte_offsets");
        if (n_sent && byte_offsets[n_sent] > byte_offsets[0]) need(utf8, "utf8");
        for (uint64_t i = 0; i < n_sent; ++i)
            if (byte_offsets[i] > byte_offsets[i + 1]) throw vbt::Error(vbt::kInvalidArgument, "byte_offsets must be non-decreasing");
        vbt::HostResult* r = t->e->run_host(utf8, byte_offsets, n_sent);
        *out = new vbt_result{t->e, r};
    });
}

int32_t vbt_result_view(const vbt_result* r, const uint64_t** tok_offsets, const vbt_token** toks, uint64_t* n_sent,
                        uint64_t* n_tokens) {
    return guarded([&] {
        need(r, "r");
        if (toks && r->r->token_bytes != sizeof(vbt_token))
            throw vbt::Error(vbt::kInvalidArgument, "compact result: read it with vbt_result_view_compact");
        if (tok_offsets) *tok_offsets = r->r->tok_off;
        if (toks) *toks = static_cast<const vbt_token*>(r->r->tokens);
        if (n_sent) *n_sent = r->r->n_sent;
        if (n_tokens) *n_tokens = r->r->n_tokens;
    });
}

int32_t vbt_result_view_compact(const vbt_result* r, const uint64_t** tok_offsets, const vbt_token16** toks, uint64_t* n_sent,
                                uint64_t* n_tokens) {
    return guarded([&] {
        need(r, "r");
        if (toks && r->r->token_bytes != sizeof(vbt_token16))
            throw vbt::Error(vbt::kInvalidArgument, "not a compact result: set the tokenizer option \"compact_tokens\" first");
        if (tok_offsets) *tok_offsets = r->r->tok_off;
        if (toks) *toks = static_cast<const vbt_token16*>(r->r->tokens);
        if (n_sent) *n_sent = r->r->n_sent;
        if (n_tokens) *n_tokens = r->r->n_tokens;
    });
}

int32_t vbt_result_text(const vbt_result* r, const uint64_t** text_offsets, const char** text, uint64_t* n_bytes) {
    return guarded([&] {
        need(r, "r");
        if (!r->r->has_text)
            throw vbt::Error(vbt::kInvalidArgument, "no text: set the tokenizer option \"output_mode\" before tokenising");
        if (text_offsets) *text_offsets = r->r->text_off;
        if (text) *text = r->r->text;
        if (n_bytes) *n_bytes = r->r->text_bytes;
    });
}

int32_t vbt_evaluate(const vbt_dict* d, vbt_tokenizer* t, const char* corpus, size_t len, const uint64_t* feature_indices,
                     size_t n_indices, uint64_t* num_ref, uint64_t* num_sys, uint64_t* num_cor) {
    return guarded([&] {
        need(d, "d");
        need(t, "t");
        if (len) need(corpus, "corpus");
        if (n_indices) need(feature_indices, "feature_indices");
        const vbt::EvalCounts c = vbt::evaluate(d->d, *t->e, std::string_view(corpus, len),
                                                std::vector<uint64_t>(feature_indices, feature_indices + n_indices));
        if (num_ref) *num_ref = c.num_ref;
        if (num_sys) *num_sys = c.num_sys;
        if (num_cor) *num_cor = c.num_cor;
    });
}

void vbt_result_free(vbt_result* r) {
    if (!r) return;
    r->owner->release(r->r);
    delete r;
}

int32_t vbt_tokenize_batch_device(vbt_tokenizer* t, uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent,
                                  uint64_t n_bytes, uint64_t* d_tok_offsets, uint64_t* d_tokens, uint64_t* n_tokens) {
    return guarded([&] {
        need(t, "t");
        need(d_tok_offsets, "d_tok_offsets");
        need(d_tokens, "d_tokens");
        need(n_tokens, "n_tokens");
        t->e->run_device(d_utf8, d_byte_offsets, n_sent, n_bytes, d_tok_offsets, d_tokens, n_tokens);
    });
}

int32_t vbt_host_alloc(size_t n_bytes, void** out) {
    return guarded([&] {
        need(out, "out");
        *out = vbt::pinned_alloc(n_bytes);
    });
}

void vbt_host_free(void* p) { vbt::pinned_free(p); }

int32_t vbt_tokenizer_set_counting(vbt_tokenizer* t, int32_t on) {
    return guarded([&] {
        need(t, "t");
        t->e->set_counting(on != 0);
    });
}

int32_t vbt_tokenizer_set_option(vbt_tokenizer* t, const char* name, int64_t value) {
    return guarded([&] {
        need(t, "t");
        need(name, "name");
        t->e->set_option(name, value);
    });
}

int32_t vbt_tokenizer_set_stream(vbt_tokenizer* t, uint64_t stream) {
    return guarded([&] {
        need(t, "t");
        t->e->set_stream(stream);
    });
}

int32_t vbt_connid_counts(vbt_tokenizer* t, uint64_t* lid_count, uint64_t* rid_count, uint32_t* num_left, uint32_t* num_right) {
    return guarded([&] {
        need(t, "t");
        t->e->connid_counts(lid_count, rid_count, num_left, num_right);
    });
}

int32_t vbt_last_stage_ms(const vbt_tokenizer* t, float* ms, int32_t cap, int32_t* n_stages) {
    return guarded([&] {
        need(t, "t");
        const float* s = t->e->stage_ms();
        for (int i = 0; i < vbt::kNumStages && i < cap; ++i) ms[i] = s[i];
        if (n_stages) *n_stages = vbt::kNumStages;
    });
}

const char* vbt_stage_names(void) { return vbt::kStageNames; }

int32_t vbt_last_launch_count(const vbt_tokenizer* t, uint64_t* n_launches) {
    return guarded([&] {
        need(t, "t");
        need(n_launches, "n_launches");
        *n_launches = t->e->launch_count();
    });
}

int32_t vbt_last_counters(const vbt_tokenizer* t, uint64_t* cnt) {
    return guarded([&] {
        need(t, "t");
        need(cnt, "cnt");
        std::memcpy(cnt, t->e->counters(), 10 * sizeof(uint64_t));
    });
}

}  // extern "C"
