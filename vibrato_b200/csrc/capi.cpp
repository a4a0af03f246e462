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
#include "format.hpp"
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
    // The strings of the output format in force (node, unk, bos, eos; empty when none is), and the option
    // "sample_text": switching sample text on compiles the format again, so that a refusal names the directive.
    std::vector<std::pair<bool, std::string>> fmt = {};
    bool sample_text = false;
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

void put(uint64_t* dst, uint64_t value) {
    if (dst) *dst = value;
}

// A device-resident batch (vbt_tokenize_batch_device*): its token arrays, left on the device.
void run_device(vbt_tokenizer* t, uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent, uint64_t n_bytes,
                const vbt::Bounds* b, uint64_t* d_tok_offsets, uint64_t* d_tokens, uint64_t* n_tokens) {
    t->e->run_device(d_utf8, d_byte_offsets, n_sent, n_bytes, b);
    const vbt::DeviceOutputs& d = t->e->last_device();
    *d_tok_offsets = d.addr[vbt::kTokOff];
    *d_tokens = d.addr[vbt::kTokens];
    *n_tokens = d.total[vbt::kGroupTokens];
}

// What the last device-resident call left on the device (vbt_last_device_*), refused when that call did not produce
// array a: it ran without `what`, or it failed.
const vbt::DeviceOutputs& last_device(const vbt_tokenizer* t, int a, const char* what) {
    need(t, "t");
    const vbt::DeviceOutputs& d = t->e->last_device();
    if (!d.made.has(a)) throw vbt::Error(vbt::kInvalidArgument, std::string("the last device-resident call ran without ") + what);
    return d;
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

int32_t vbt_tokenize_batch_bounded(vbt_tokenizer* t, const char* utf8, const uint64_t* byte_offsets, uint64_t n_sent,
                                   const uint64_t* bnd_offsets, const uint32_t* bnd, vbt_result** out) {
    return guarded([&] {
        need(t, "t");
        need(out, "out");
        need(byte_offsets, "byte_offsets");
        need(bnd_offsets, "bnd_offsets");
        if (n_sent && byte_offsets[n_sent] > byte_offsets[0]) need(utf8, "utf8");
        if (bnd_offsets[n_sent] > bnd_offsets[0]) need(bnd, "bnd");
        for (uint64_t i = 0; i < n_sent; ++i)
            if (byte_offsets[i] > byte_offsets[i + 1]) throw vbt::Error(vbt::kInvalidArgument, "byte_offsets must be non-decreasing");
        const vbt::Bounds b{bnd_offsets, bnd, bnd_offsets[n_sent], {}};  // the boundary lists are checked on the device
        vbt::HostResult* r = t->e->run_host(utf8, byte_offsets, n_sent, &b);
        *out = new vbt_result{t->e, r};
    });
}

namespace {
// The pattern table of vbt_tokenize_batch_spans (engine.hpp Spans): each pattern split like a feature (csv_fields in
// kernels.cu), every field that is not exactly "*" kept as {field index, first byte, length}.
struct SpanPatterns {
    std::vector<uint32_t> off{0}, pf;
    std::vector<uint8_t> bytes;

    SpanPatterns(const char* patterns, const uint64_t* pattern_offsets, uint64_t n) {
        if (n >= VBT_SPAN_ANY) throw vbt::Error(vbt::kInvalidArgument, "too many patterns");
        if (n) need(pattern_offsets, "pattern_offsets");
        for (uint64_t k = 0; k < n; ++k) {
            if (pattern_offsets[k + 1] < pattern_offsets[k])
                throw vbt::Error(vbt::kInvalidArgument, "pattern_offsets must be non-decreasing");
            const uint64_t len = pattern_offsets[k + 1] - pattern_offsets[k];
            if (len) need(patterns, "patterns");
            if (len) add(k, reinterpret_cast<const uint8_t*>(patterns) + pattern_offsets[k], len);
            off.push_back(uint32_t(pf.size() / 3));
        }
    }

   private:
    void add(uint64_t k, const uint8_t* p, uint64_t n) {
        uint32_t field = 0, kept = 0;
        uint64_t start = 0;
        std::string cur;
        auto close = [&] {
            if (cur == "*") return;
            auto fail = [&](const char* why) {
                throw vbt::Error(vbt::kInvalidArgument, "pattern " + std::to_string(k) + ", byte " + std::to_string(start) +
                                                            ": " + why);
            };
            if (field > vbt::kFmtMaxFieldIndex) fail("field index above 255");
            if (kept == vbt::kFmtMaxFields) fail("more than 16 constrained fields");
            ++kept;
            pf.insert(pf.end(), {field, uint32_t(bytes.size()), uint32_t(cur.size())});
            bytes.insert(bytes.end(), cur.begin(), cur.end());
        };
        bool quoted = false, at_start = true;
        for (uint64_t i = 0; i < n; ++i) {  // csv_fields of kernels.cu
            const uint8_t c = p[i];
            if (quoted) {
                if (c != '"') {
                    cur.push_back(char(c));
                } else if (i + 1 < n && p[i + 1] == '"') {
                    cur.push_back(char(c));
                    ++i;
                } else {
                    quoted = false;
                }
            } else if (c == '"' && at_start) {
                quoted = true;
            } else if (c == ',') {
                close();
                ++field;
                cur.clear();
                start = i + 1;
                at_start = true;
                continue;
            } else {
                cur.push_back(char(c));
            }
            at_start = false;
        }
        close();
    }

   public:
    void fill(vbt::Spans& s) const {
        s.pat_off = off.data();
        s.pf = pf.data();
        s.pat_bytes = bytes.data();
        s.n_pat = uint32_t(off.size() - 1);
        s.n_pat_bytes = bytes.size();
    }
};
}  // namespace

int32_t vbt_tokenize_batch_spans(vbt_tokenizer* t, const char* utf8, const uint64_t* byte_offsets, uint64_t n_sent,
                                 const uint64_t* bnd_offsets, const uint32_t* bnd, const uint64_t* span_offsets,
                                 const vbt_span* spans, const char* patterns, const uint64_t* pattern_offsets,
                                 uint64_t n_patterns, vbt_result** out) {
    return guarded([&] {
        need(t, "t");
        need(out, "out");
        need(byte_offsets, "byte_offsets");
        need(span_offsets, "span_offsets");
        if (n_sent && byte_offsets[n_sent] > byte_offsets[0]) need(utf8, "utf8");
        if (bnd_offsets && bnd_offsets[n_sent] > bnd_offsets[0]) need(bnd, "bnd");
        if (span_offsets[n_sent] > span_offsets[0]) need(spans, "spans");
        for (uint64_t i = 0; i < n_sent; ++i)
            if (byte_offsets[i] > byte_offsets[i + 1]) throw vbt::Error(vbt::kInvalidArgument, "byte_offsets must be non-decreasing");
        const SpanPatterns pat(patterns, pattern_offsets, n_patterns);
        vbt::Bounds b;  // the lists themselves are checked on the device
        if (bnd_offsets) b = vbt::Bounds{bnd_offsets, bnd, bnd_offsets[n_sent], {}};
        b.spans.off = span_offsets;
        b.spans.rec = reinterpret_cast<const uint32_t*>(spans);
        b.spans.n = span_offsets[n_sent];
        pat.fill(b.spans);
        vbt::HostResult* r = t->e->run_host(utf8, byte_offsets, n_sent, &b);
        *out = new vbt_result{t->e, r};
    });
}

int32_t vbt_result_view(const vbt_result* r, const uint64_t** tok_offsets, const vbt_token** toks, uint64_t* n_sent,
                        uint64_t* n_tokens) {
    return guarded([&] {
        need(r, "r");
        if (toks && r->r->out.token_bytes != sizeof(vbt_token))
            throw vbt::Error(vbt::kInvalidArgument, "compact result: read it with vbt_result_view_compact");
        if (tok_offsets) *tok_offsets = r->r->ptr<uint64_t>(vbt::kTokOff);
        if (toks) *toks = r->r->ptr<const vbt_token>(vbt::kTokens);
        if (n_sent) *n_sent = r->r->n_sent;
        if (n_tokens) *n_tokens = r->r->total[vbt::kGroupTokens];
    });
}

int32_t vbt_result_view_compact(const vbt_result* r, const uint64_t** tok_offsets, const vbt_token16** toks, uint64_t* n_sent,
                                uint64_t* n_tokens) {
    return guarded([&] {
        need(r, "r");
        if (toks && r->r->out.token_bytes != sizeof(vbt_token16))
            throw vbt::Error(vbt::kInvalidArgument, "not a compact result: set the tokenizer option \"compact_tokens\" first");
        if (tok_offsets) *tok_offsets = r->r->ptr<uint64_t>(vbt::kTokOff);
        if (toks) *toks = r->r->ptr<const vbt_token16>(vbt::kTokens);
        if (n_sent) *n_sent = r->r->n_sent;
        if (n_tokens) *n_tokens = r->r->total[vbt::kGroupTokens];
    });
}

int32_t vbt_result_text(const vbt_result* r, const uint64_t** text_offsets, const char** text, uint64_t* n_bytes) {
    return guarded([&] {
        need(r, "r");
        if (!r->r->out.text)
            throw vbt::Error(vbt::kInvalidArgument, "no text: set the tokenizer option \"output_mode\" before tokenising");
        if (text_offsets) *text_offsets = r->r->ptr<uint64_t>(vbt::kTextOff);
        if (text) *text = r->r->ptr<const char>(vbt::kText);
        if (n_bytes) *n_bytes = r->r->total[vbt::kGroupText];
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
        run_device(t, d_utf8, d_byte_offsets, n_sent, n_bytes, nullptr, d_tok_offsets, d_tokens, n_tokens);
    });
}

int32_t vbt_tokenize_batch_device_bounded(vbt_tokenizer* t, uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent,
                                          uint64_t n_bytes, uint64_t d_bnd_offsets, uint64_t d_bnd, uint64_t n_bnd,
                                          uint64_t* d_tok_offsets, uint64_t* d_tokens, uint64_t* n_tokens) {
    return guarded([&] {
        need(t, "t");
        need(d_tok_offsets, "d_tok_offsets");
        need(d_tokens, "d_tokens");
        need(n_tokens, "n_tokens");
        if (!d_bnd_offsets) throw vbt::Error(vbt::kInvalidArgument, "d_bnd_offsets is null");
        if (n_bnd && !d_bnd) throw vbt::Error(vbt::kInvalidArgument, "d_bnd is null");
        const vbt::Bounds b{reinterpret_cast<const uint64_t*>(d_bnd_offsets), reinterpret_cast<const uint32_t*>(d_bnd), n_bnd, {}};
        run_device(t, d_utf8, d_byte_offsets, n_sent, n_bytes, &b, d_tok_offsets, d_tokens, n_tokens);
    });
}

int32_t vbt_tokenize_batch_device_spans(vbt_tokenizer* t, uint64_t d_utf8, uint64_t d_byte_offsets, uint64_t n_sent,
                                        uint64_t n_bytes, uint64_t d_bnd_offsets, uint64_t d_bnd, uint64_t n_bnd,
                                        uint64_t d_span_offsets, uint64_t d_spans, uint64_t n_spans, const char* patterns,
                                        const uint64_t* pattern_offsets, uint64_t n_patterns, uint64_t* d_tok_offsets,
                                        uint64_t* d_tokens, uint64_t* n_tokens) {
    return guarded([&] {
        need(t, "t");
        need(d_tok_offsets, "d_tok_offsets");
        need(d_tokens, "d_tokens");
        need(n_tokens, "n_tokens");
        if (n_bnd && !d_bnd) throw vbt::Error(vbt::kInvalidArgument, "d_bnd is null");
        if (!d_span_offsets) throw vbt::Error(vbt::kInvalidArgument, "d_span_offsets is null");
        if (n_spans && !d_spans) throw vbt::Error(vbt::kInvalidArgument, "d_spans is null");
        const SpanPatterns pat(patterns, pattern_offsets, n_patterns);
        vbt::Bounds b;
        if (d_bnd_offsets)
            b = vbt::Bounds{reinterpret_cast<const uint64_t*>(d_bnd_offsets), reinterpret_cast<const uint32_t*>(d_bnd), n_bnd, {}};
        b.spans.off = reinterpret_cast<const uint64_t*>(d_span_offsets);
        b.spans.rec = reinterpret_cast<const uint32_t*>(d_spans);
        b.spans.n = n_spans;
        pat.fill(b.spans);
        run_device(t, d_utf8, d_byte_offsets, n_sent, n_bytes, &b, d_tok_offsets, d_tokens, n_tokens);
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
        const std::string opt = name;
        if (opt == "sample_text" && value == 1 && !t->fmt.empty()) {
            vbt::FormatText s[4];
            for (int i = 0; i < 4; ++i) s[i] = {t->fmt[i].first ? t->fmt[i].second.data() : nullptr, t->fmt[i].second.size()};
            vbt::compile_format(s[0], s[1], s[2], s[3], t->e->marginals() > 0, false, true);  // throws at %pP / %pb
        }
        t->e->set_option(opt, value);
        if (opt == "sample_text") t->sample_text = value != 0;
        if (opt == "output_mode") t->fmt.clear();  // a fixed mode replaces the format
    });
}

int32_t vbt_tokenizer_set_output_format(vbt_tokenizer* t, const char* node, size_t node_len, const char* unk, size_t unk_len,
                                        const char* bos, size_t bos_len, const char* eos, size_t eos_len) {
    return guarded([&] {
        need(t, "t");
        if (!node) {
            t->e->set_format(nullptr);
            t->fmt.clear();
            return;
        }
        // an empty string may come with any pointer: only NULL means "not given"
        // %pP has a value only while the tokenizer computes marginals, %pb only in lattice text (where the "prev"
        // directives have none); sample text has neither
        const vbt::FormatProgram p = vbt::compile_format({node, node_len}, {unk, unk_len}, {bos, bos_len}, {eos, eos_len},
                                                         t->e->marginals() > 0, t->e->lattice() == 2, t->sample_text);
        t->fmt.clear();  // set_format replaces (or, failing, clears) the format in force
        t->e->set_format(&p);
        const char* ptr[4] = {node, unk, bos, eos};
        const size_t len[4] = {node_len, unk_len, bos_len, eos_len};
        for (int i = 0; i < 4; ++i) t->fmt.emplace_back(ptr[i] != nullptr, ptr[i] ? std::string(ptr[i], len[i]) : std::string());
    });
}

int32_t vbt_tokenizer_set_marginals(vbt_tokenizer* t, double theta) {
    return guarded([&] {
        need(t, "t");
        t->e->set_marginals(theta);
    });
}

int32_t vbt_result_marginals(const vbt_result* r, const float** token_prob, const float** path_prob) {
    return guarded([&] {
        need(r, "r");
        if (!r->r->out.marg)
            throw vbt::Error(vbt::kInvalidArgument, "no marginals: switch them on with vbt_tokenizer_set_marginals before tokenising");
        if (token_prob) *token_prob = r->r->ptr<const float>(vbt::kTokenProb);
        if (path_prob) *path_prob = r->r->ptr<const float>(vbt::kPathProb);
    });
}

int32_t vbt_last_device_marginals(const vbt_tokenizer* t, uint64_t* d_token_prob, uint64_t* d_path_prob) {
    return guarded([&] {
        const vbt::DeviceOutputs& d = last_device(t, vbt::kTokenProb, "marginals");
        put(d_token_prob, d.addr[vbt::kTokenProb]);
        put(d_path_prob, d.addr[vbt::kPathProb]);
    });
}

int32_t vbt_result_uncertainty(const vbt_result* r, const double** entropy, const double** log_path_prob,
                               const uint64_t** boundary_offsets, const float** boundary_prob) {
    return guarded([&] {
        need(r, "r");
        if (!r->r->out.has(vbt::kEntropy))
            throw vbt::Error(vbt::kInvalidArgument,
                             "no uncertainty: set the tokenizer option \"uncertainty\" (with marginals on) before tokenising");
        if (entropy) *entropy = r->r->ptr<const double>(vbt::kEntropy);
        if (log_path_prob) *log_path_prob = r->r->ptr<const double>(vbt::kLogPathProb);
        const bool pos = r->r->out.has(vbt::kBoundaryProb);  // level 2
        if (boundary_offsets) *boundary_offsets = pos ? r->r->ptr<const uint64_t>(vbt::kPosOff) : nullptr;
        if (boundary_prob) *boundary_prob = pos ? r->r->ptr<const float>(vbt::kBoundaryProb) : nullptr;
    });
}

int32_t vbt_last_device_uncertainty(const vbt_tokenizer* t, uint64_t* d_entropy, uint64_t* d_log_path_prob,
                                    uint64_t* d_boundary_offsets, uint64_t* d_boundary_prob, uint64_t* n_positions) {
    return guarded([&] {
        const vbt::DeviceOutputs& d = last_device(t, vbt::kEntropy, "the option \"uncertainty\"");
        put(d_entropy, d.addr[vbt::kEntropy]);
        put(d_log_path_prob, d.addr[vbt::kLogPathProb]);
        put(d_boundary_offsets, d.addr[vbt::kPosOff]);  // 0 at level 1
        put(d_boundary_prob, d.addr[vbt::kBoundaryProb]);
        put(n_positions, d.made.has(vbt::kBoundaryProb) ? d.total[vbt::kGroupPositions] : 0);
    });
}

int32_t vbt_result_lattice(const vbt_result* r, const uint64_t** node_offsets, const vbt_token** nodes,
                           const vbt_lattice_link** links, const float** node_prob, uint64_t* n_nodes) {
    return guarded([&] {
        need(r, "r");
        if (!r->r->out.lat)
            throw vbt::Error(vbt::kInvalidArgument, "no lattice: set the tokenizer option \"lattice\" before tokenising");
        if (node_offsets) *node_offsets = r->r->ptr<uint64_t>(vbt::kNodeOff);
        if (nodes) *nodes = r->r->ptr<const vbt_token>(vbt::kNodes);
        if (links) *links = r->r->ptr<const vbt_lattice_link>(vbt::kLinks);
        if (node_prob) *node_prob = r->r->out.marg ? r->r->ptr<const float>(vbt::kNodeProb) : nullptr;
        if (n_nodes) *n_nodes = r->r->total[vbt::kGroupLattice];
    });
}

int32_t vbt_last_device_lattice(const vbt_tokenizer* t, uint64_t* d_node_offsets, uint64_t* d_nodes, uint64_t* d_links,
                                uint64_t* d_node_prob, uint64_t* n_nodes) {
    return guarded([&] {
        const vbt::DeviceOutputs& d = last_device(t, vbt::kNodes, "the lattice");
        put(d_node_offsets, d.addr[vbt::kNodeOff]);
        put(d_nodes, d.addr[vbt::kNodes]);
        put(d_links, d.addr[vbt::kLinks]);
        put(d_node_prob, d.addr[vbt::kNodeProb]);  // 0 without marginals
        put(n_nodes, d.total[vbt::kGroupLattice]);
    });
}

int32_t vbt_result_lattice_margins(const vbt_result* r, const int64_t** node_margin) {
    return guarded([&] {
        need(r, "r");
        if (!r->r->out.has(vbt::kNodeMargin))
            throw vbt::Error(vbt::kInvalidArgument,
                             "no lattice margins: set the tokenizer options \"lattice\" and \"lattice_margin\" before tokenising");
        if (node_margin) *node_margin = r->r->ptr<const int64_t>(vbt::kNodeMargin);
    });
}

int32_t vbt_last_device_lattice_margins(const vbt_tokenizer* t, uint64_t* d_node_margin) {
    return guarded([&] {
        put(d_node_margin, last_device(t, vbt::kNodeMargin, "the lattice's cost margin").addr[vbt::kNodeMargin]);
    });
}

int32_t vbt_tokenizer_set_sampling(vbt_tokenizer* t, uint32_t n, double theta, uint64_t seed) {
    return guarded([&] {
        need(t, "t");
        t->e->set_sampling(n, theta, seed);
    });
}

int32_t vbt_result_samples(const vbt_result* r, const uint64_t** sample_offsets, const vbt_token** samples,
                           uint64_t* n_sample_tokens) {
    return guarded([&] {
        need(r, "r");
        if (!r->r->out.n_samp)
            throw vbt::Error(vbt::kInvalidArgument, "no samples: switch sampling on with vbt_tokenizer_set_sampling before tokenising");
        if (sample_offsets) *sample_offsets = r->r->ptr<uint64_t>(vbt::kSampleOff);
        if (samples) *samples = r->r->ptr<const vbt_token>(vbt::kSamples);
        if (n_sample_tokens) *n_sample_tokens = r->r->total[vbt::kGroupSamples];
    });
}

int32_t vbt_last_device_samples(const vbt_tokenizer* t, uint64_t* d_sample_offsets, uint64_t* d_samples,
                                uint64_t* n_sample_tokens) {
    return guarded([&] {
        const vbt::DeviceOutputs& d = last_device(t, vbt::kSamples, "sampling");
        put(d_sample_offsets, d.addr[vbt::kSampleOff]);
        put(d_samples, d.addr[vbt::kSamples]);
        put(n_sample_tokens, d.total[vbt::kGroupSamples]);
    });
}

int32_t vbt_tokenizer_set_posterior(vbt_tokenizer* t, int32_t on, double gamma) {
    return guarded([&] {
        need(t, "t");
        t->e->set_posterior(on != 0, gamma);
    });
}

int32_t vbt_result_posterior(const vbt_result* r, const uint64_t** posterior_offsets, const vbt_token** posterior_tokens,
                             const float** posterior_probs, const double** posterior_gains, uint64_t* n_posterior_tokens) {
    return guarded([&] {
        need(r, "r");
        if (!r->r->out.has(vbt::kPostTokens))
            throw vbt::Error(vbt::kInvalidArgument, "no posterior paths: switch posterior decoding on with vbt_tokenizer_set_posterior before tokenising");
        if (posterior_offsets) *posterior_offsets = r->r->ptr<const uint64_t>(vbt::kPostOff);
        if (posterior_tokens) *posterior_tokens = r->r->ptr<const vbt_token>(vbt::kPostTokens);
        if (posterior_probs) *posterior_probs = r->r->ptr<const float>(vbt::kPostProb);
        if (posterior_gains) *posterior_gains = r->r->ptr<const double>(vbt::kPostGain);
        if (n_posterior_tokens) *n_posterior_tokens = r->r->total[vbt::kGroupPosterior];
    });
}

int32_t vbt_last_device_posterior(const vbt_tokenizer* t, uint64_t* d_posterior_offsets, uint64_t* d_posterior_tokens,
                                  uint64_t* d_posterior_probs, uint64_t* d_posterior_gains, uint64_t* n_posterior_tokens) {
    return guarded([&] {
        const vbt::DeviceOutputs& d = last_device(t, vbt::kPostTokens, "posterior decoding");
        put(d_posterior_offsets, d.addr[vbt::kPostOff]);
        put(d_posterior_tokens, d.addr[vbt::kPostTokens]);
        put(d_posterior_probs, d.addr[vbt::kPostProb]);
        put(d_posterior_gains, d.addr[vbt::kPostGain]);
        put(n_posterior_tokens, d.total[vbt::kGroupPosterior]);
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
