// Host-side dictionary model: MeCab-format parsers, double-array construction, `.dic` (bincode)
// reader/writer.  See host_dict.hpp.  Citations are relative to /root/reference/vibrato/src/.
#include "host_dict.hpp"

#include <dlfcn.h>

#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <limits>
#include <map>
#include <numeric>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <type_traits>

namespace vbt {

// ---------------------------------------------------------------------------------------------
// UTF-8
// ---------------------------------------------------------------------------------------------

bool utf8_valid(const uint8_t* s, size_t n) {
    size_t i = 0;
    while (i < n) {
        uint8_t c = s[i];
        if (c < 0x80) {
            ++i;
            continue;
        }
        size_t need;
        uint32_t lo;
        uint32_t cp;
        if ((c & 0xE0) == 0xC0) {
            need = 1, lo = 0x80, cp = c & 0x1F;
        } else if ((c & 0xF0) == 0xE0) {
            need = 2, lo = 0x800, cp = c & 0x0F;
        } else if ((c & 0xF8) == 0xF0) {
            need = 3, lo = 0x10000, cp = c & 0x07;
        } else {
            return false;
        }
        if (i + need >= n) return false;  // truncated sequence
        for (size_t k = 1; k <= need; ++k) {
            uint8_t cc = s[i + k];
            if ((cc & 0xC0) != 0x80) return false;
            cp = (cp << 6) | (cc & 0x3F);
        }
        if (cp < lo || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return false;
        i += need + 1;
    }
    return true;
}

std::u32string utf8_to_u32(std::string_view s) {
    std::u32string out;
    out.reserve(s.size());
    const uint8_t* p = reinterpret_cast<const uint8_t*>(s.data());
    size_t n = s.size(), i = 0;
    while (i < n) {
        uint8_t c = p[i];
        if (c < 0x80) {
            out.push_back(c);
            i += 1;
        } else if (c < 0xE0) {
            out.push_back(((c & 0x1Fu) << 6) | (p[i + 1] & 0x3Fu));
            i += 2;
        } else if (c < 0xF0) {
            out.push_back(((c & 0x0Fu) << 12) | ((p[i + 1] & 0x3Fu) << 6) | (p[i + 2] & 0x3Fu));
            i += 3;
        } else {
            out.push_back(((c & 0x07u) << 18) | ((p[i + 1] & 0x3Fu) << 12) | ((p[i + 2] & 0x3Fu) << 6) | (p[i + 3] & 0x3Fu));
            i += 4;
        }
    }
    return out;
}

// ---------------------------------------------------------------------------------------------
// number parsing with Rust's FromStr strictness
// ---------------------------------------------------------------------------------------------

template <typename T>
static bool parse_strict(std::string_view s, T& out) {
    constexpr bool is_signed = std::is_signed<T>::value;
    if (s.empty()) return false;
    size_t i = 0;
    bool neg = false;
    if (s[0] == '+') {
        i = 1;
    } else if (s[0] == '-') {
        if (!is_signed) return false;
        neg = true;
        i = 1;
    }
    if (i == s.size()) return false;
    unsigned long long v = 0;
    for (; i < s.size(); ++i) {
        if (s[i] < '0' || s[i] > '9') return false;
        v = v * 10 + unsigned(s[i] - '0');
        if (v > (1ull << 62)) return false;
    }
    long long sv = neg ? -static_cast<long long>(v) : static_cast<long long>(v);
    if (sv < static_cast<long long>(std::numeric_limits<T>::min()) ||
        (!neg && v > static_cast<unsigned long long>(std::numeric_limits<T>::max())))
        return false;
    out = static_cast<T>(sv);
    return true;
}

// ---------------------------------------------------------------------------------------------
// CSV (lexicon.rs:111-200 on top of csv-core's field reader)
// ---------------------------------------------------------------------------------------------

namespace {

// One pass over csv-core's DFA: ',' delimiter, '"' quoting with doubled-quote escapes, records
// ending in \n, \r or \r\n, blank lines skipped.
class CsvFields {
   public:
    explicit CsvFields(std::string_view b) : b_(b) {}

    enum class Kind { kEnd, kField };
    struct Field {
        Kind kind;
        bool record_end;  // the record ended with this field
        bool input_empty; // csv-core's InputEmpty: EOF hit inside the field (lexicon.rs:133-137)
        size_t begin;     // input offset where this read started (after skipped terminators)
        size_t next;      // input offset after the delimiter / first terminator byte
    };

    static constexpr size_t kMaxField = 4096;  // lexicon.rs:124,138-140

    Field read(std::string& out) {
        out.clear();
        if (at_record_start_) {
            while (pos_ < b_.size() && (b_[pos_] == '\n' || b_[pos_] == '\r')) ++pos_;
            if (pos_ >= b_.size()) return {Kind::kEnd, false, false, pos_, pos_};
            at_record_start_ = false;
        }
        Field f{Kind::kField, false, false, pos_, pos_};
        if (pos_ >= b_.size()) {  // EOF right behind a delimiter: one empty closing field
            f.record_end = true;
            at_record_start_ = true;
            return f;
        }
        enum { kStart, kPlain, kQuoted, kQuoteSeen } st = kStart;
        for (;;) {
            if (pos_ >= b_.size()) {
                f.record_end = f.input_empty = true;
                at_record_start_ = true;
                f.next = pos_;
                return f;
            }
            char c = b_[pos_];
            if (st == kStart) {
                st = kPlain;
                if (c == '"') {
                    st = kQuoted;
                    ++pos_;
                    continue;
                }
            }
            if (st == kQuoted) {
                if (c == '"') {
                    st = kQuoteSeen;
                    ++pos_;
                    continue;
                }
            } else {
                if (st == kQuoteSeen && c == '"') {
                    st = kQuoted;  // "" inside quotes
                } else if (c == ',') {
                    f.next = ++pos_;
                    return f;
                } else if (c == '\n' || c == '\r') {
                    f.next = ++pos_;
                    f.record_end = true;
                    at_record_start_ = true;
                    return f;
                } else if (st == kQuoteSeen) {
                    st = kPlain;  // text after a closing quote is kept verbatim
                }
            }
            if (out.size() >= kMaxField) throw Error(kInvalidFormat, "Field too large");
            out.push_back(c);
            ++pos_;
        }
    }

   private:
    std::string_view b_;
    size_t pos_ = 0;
    bool at_record_start_ = true;
};

}  // namespace

std::vector<RawWordEntry> parse_lexicon_csv(std::string_view bytes, const char* name) {
    std::vector<RawWordEntry> entries;
    CsvFields rdr(bytes);
    std::string field, surface;
    WordParam param{0, 0, 0};
    size_t n_fields = 0, feature_begin = 0;
    auto fail = [&](Status st, const std::string& m) -> Error { return Error(st, std::string(name) + ": " + m); };
    for (;;) {
        CsvFields::Field f;
        try {
            f = rdr.read(field);
        } catch (const Error& e) {
            throw fail(e.code, e.what());
        }
        if (f.kind == CsvFields::Kind::kEnd) break;
        if (f.record_end && n_fields == 0 && f.next == f.begin && !f.input_empty) continue;  // lexicon.rs:170
        if (f.input_empty) {
            // the unfinished field is not counted (lexicon.rs:133-137): rows need >= 5 items (:171-177)
            if (n_fields <= 3) throw fail(kInvalidFormat, "A csv row of lexicon must have five items at least");
        } else {
            switch (n_fields) {
                case 0:
                    surface = field;
                    if (!utf8_valid(reinterpret_cast<const uint8_t*>(surface.data()), surface.size()))
                        throw fail(kUtf8, "invalid utf-8");
                    break;
                case 1:
                    if (!parse_strict<uint16_t>(field, param.left_id)) throw fail(kParseInt, "invalid left_id: " + field);
                    break;
                case 2:
                    if (!parse_strict<uint16_t>(field, param.right_id)) throw fail(kParseInt, "invalid right_id: " + field);
                    break;
                case 3:
                    if (!parse_strict<int16_t>(field, param.word_cost)) throw fail(kParseInt, "invalid word_cost: " + field);
                    feature_begin = f.next;  // lexicon.rs:155
                    break;
                default:
                    break;
            }
        }
        if (!f.record_end) {
            ++n_fields;
            continue;
        }
        if (n_fields <= 3) throw fail(kInvalidFormat, "A csv row of lexicon must have five items at least");
        size_t feature_end = f.input_empty ? f.next : f.next - 1;  // lexicon.rs:178 drops the terminator byte
        if (feature_end < feature_begin) throw fail(kInvalidFormat, "truncated final record");
        std::string_view feat = bytes.substr(feature_begin, feature_end - feature_begin);
        if (!utf8_valid(reinterpret_cast<const uint8_t*>(feat.data()), feat.size())) throw fail(kUtf8, "invalid utf-8");
        if (!surface.empty())  // lexicon.rs:179-183 skips empty surfaces
            entries.push_back(RawWordEntry{surface, param, feat});
        surface.clear();
        n_fields = 0;
    }
    return entries;
}

// ---------------------------------------------------------------------------------------------
// Trie
// ---------------------------------------------------------------------------------------------

namespace {

class DoubleArrayBuilder {
   public:
    explicit DoubleArrayBuilder(uint32_t alphabet) {
        block_ = 256;
        while (block_ < alphabet) block_ <<= 1;
        grow();
        occupy(0);
        base_[0] = 0;
        check_[0] = Trie::kMask;
    }

    uint32_t place(const std::vector<uint32_t>& codes) {
        if (head_ != kNil) {
            if (codes.size() == 1) return head_ ^ codes[0];
            uint32_t s = prev_[head_];  // newest vacant slot
            for (int tries = 0; tries < 400; ++tries) {
                uint32_t b = s ^ codes[0];
                bool ok = true;
                for (size_t j = 1; j < codes.size(); ++j)
                    if (!vacant(b ^ codes[j])) {
                        ok = false;
                        break;
                    }
                if (ok) return b;
                if (s == head_) break;
                s = prev_[s];
            }
        }
        uint32_t b = uint32_t(base_.size());
        grow();
        return b;
    }

    void occupy(uint32_t i) {
        uint32_t p = prev_[i], n = next_[i];
        if (n == i) {
            head_ = kNil;
        } else {
            next_[p] = n;
            prev_[n] = p;
            if (head_ == i) head_ = n;
        }
        used_[i] = 1;
    }

    bool vacant(uint32_t i) const { return !used_[i]; }

    std::vector<uint32_t> base_, check_;

   private:
    static constexpr uint32_t kNil = 0xFFFFFFFFu;
    void grow() {
        uint32_t old = uint32_t(base_.size()), nsz = old + block_;
        if (nsz >= Trie::kMask) throw Error(kInvalidArgument, "trie too large");
        base_.resize(nsz, Trie::kMask);
        check_.resize(nsz, Trie::kMask);
        used_.resize(nsz, 0);
        prev_.resize(nsz);
        next_.resize(nsz);
        for (uint32_t i = old; i < nsz; ++i) {
            prev_[i] = i - 1;
            next_[i] = i + 1;
        }
        if (head_ == kNil) {
            head_ = old;
            prev_[old] = nsz - 1;
            next_[nsz - 1] = old;
        } else {
            uint32_t tail = prev_[head_];
            next_[tail] = old;
            prev_[old] = tail;
            next_[nsz - 1] = head_;
            prev_[head_] = nsz - 1;
        }
    }
    uint32_t block_;
    uint32_t head_ = kNil;
    std::vector<uint32_t> prev_, next_;
    std::vector<uint8_t> used_;
};

}  // namespace

Trie Trie::from_records(const std::vector<std::pair<std::u32string, uint32_t>>& recs) {
    Trie t;
    // frequency-ordered code mapper; code 0 is the terminator
    uint32_t max_cp = 0;
    for (auto& r : recs)
        for (char32_t c : r.first) max_cp = std::max<uint32_t>(max_cp, c);
    std::vector<uint32_t> freq(recs.empty() ? 0 : max_cp + 1, 0);
    for (auto& r : recs)
        for (char32_t c : r.first) ++freq[c];
    std::vector<uint32_t> used;
    for (uint32_t c = 0; c < freq.size(); ++c)
        if (freq[c]) used.push_back(c);
    std::stable_sort(used.begin(), used.end(), [&](uint32_t a, uint32_t b) { return freq[a] > freq[b]; });
    t.table.assign(freq.size(), kInvalidCode);
    for (uint32_t i = 0; i < used.size(); ++i) t.table[used[i]] = i + 1;
    t.alphabet_size = uint32_t(used.size()) + 1;

    DoubleArrayBuilder da(t.alphabet_size);
    struct Frame {
        uint32_t node, lo, hi, depth;
    };
    std::vector<Frame> stack;
    if (!recs.empty()) stack.push_back({0, 0, uint32_t(recs.size()), 0});
    std::vector<uint32_t> codes, bounds;
    while (!stack.empty()) {
        Frame f = stack.back();
        stack.pop_back();
        uint32_t lo = f.lo;
        bool terminal = recs[lo].first.size() == f.depth;
        uint32_t tvalue = terminal ? recs[lo].second : 0;
        if (terminal) ++lo;
        if (lo == f.hi) {
            da.base_[f.node] = kFlag | tvalue;  // is_leaf
            continue;
        }
        codes.clear();
        bounds.clear();
        if (terminal) {
            codes.push_back(0);
            bounds.push_back(lo);
        }
        for (uint32_t i = lo; i < f.hi;) {
            char32_t c = recs[i].first[f.depth];
            uint32_t j = i + 1;
            while (j < f.hi && recs[j].first[f.depth] == c) ++j;
            codes.push_back(t.table[c]);
            bounds.push_back(i);
            i = j;
        }
        bounds.push_back(f.hi);
        uint32_t b = da.place(codes);
        da.base_[f.node] = b;
        if (terminal) da.check_[f.node] |= kFlag;  // has_leaf
        for (size_t c = 0; c < codes.size(); ++c) {
            uint32_t child = b ^ codes[c];
            da.occupy(child);
            da.check_[child] = f.node;
            if (terminal && c == 0) {
                da.base_[child] = kFlag | tvalue;
            } else {
                da.base_[child] = 0;
                stack.push_back({child, bounds[c], bounds[c + 1], f.depth + 1});
            }
        }
    }
    t.nodes.resize(da.base_.size() * 2);
    for (size_t i = 0; i < da.base_.size(); ++i) {
        t.nodes[2 * i] = da.base_[i];
        t.nodes[2 * i + 1] = da.check_[i];
    }
    return t;
}

void Trie::common_prefix_search(const char32_t* s, size_t n, std::vector<std::pair<uint32_t, uint32_t>>& out) const {
    out.clear();
    if (nodes.empty()) return;
    uint32_t node = 0;
    for (size_t pos = 0; pos < n; ++pos) {
        uint32_t c = s[pos];
        if (c >= table.size()) return;
        uint32_t code = table[c];
        if (code == kInvalidCode) return;
        uint32_t b = nodes[2 * node];
        if (b & kFlag) return;
        uint32_t child = (b ^ code);
        if (child >= num_nodes() || (nodes[2 * child + 1] & kMask) != node) return;
        node = child;
        uint32_t nb = nodes[2 * node];
        if (nb & kFlag) {
            out.emplace_back(nb & kMask, uint32_t(pos + 1));
            return;
        }
        if (nodes[2 * node + 1] & kFlag) out.emplace_back(nodes[2 * size_t(nb)] & kMask, uint32_t(pos + 1));
    }
}

void Trie::serialize(std::vector<uint8_t>& out) const {
    auto put = [&](uint32_t v) {
        uint8_t b[4] = {uint8_t(v), uint8_t(v >> 8), uint8_t(v >> 16), uint8_t(v >> 24)};
        out.insert(out.end(), b, b + 4);
    };
    put(uint32_t(table.size()));
    for (uint32_t v : table) put(v);
    put(alphabet_size);
    put(num_nodes());
    for (uint32_t v : nodes) put(v);
}

Trie Trie::deserialize(const uint8_t* p, size_t n) {
    size_t pos = 0;
    auto get = [&]() -> uint32_t {
        if (pos + 4 > n) throw Error(kDecode, "crawdad trie blob truncated");
        uint32_t v;
        std::memcpy(&v, p + pos, 4);
        pos += 4;
        return v;
    };
    Trie t;
    uint32_t tl = get();
    if (size_t(tl) * 4 > n) throw Error(kDecode, "crawdad trie blob: bad table length");
    t.table.resize(tl);
    for (auto& v : t.table) v = get();
    t.alphabet_size = get();
    uint32_t nn = get();
    if (size_t(nn) * 8 > n) throw Error(kDecode, "crawdad trie blob: bad node count");
    t.nodes.resize(size_t(nn) * 2);
    for (auto& v : t.nodes) v = get();
    return t;
}

std::vector<std::pair<std::u32string, uint32_t>> Trie::enumerate() const {
    std::vector<std::pair<std::u32string, uint32_t>> out;
    uint32_t nn = num_nodes();
    if (nn == 0) return out;
    std::vector<char32_t> inv(alphabet_size + 1, 0);
    for (uint32_t c = 0; c < table.size(); ++c)
        if (table[c] != kInvalidCode && table[c] < inv.size()) inv[table[c]] = c;
    // children by parent via the check field
    std::vector<uint32_t> cnt(nn + 1, 0);
    auto vacant = [&](uint32_t i) { return nodes[2 * i] == kMask && nodes[2 * i + 1] == kMask; };
    for (uint32_t i = 1; i < nn; ++i)
        if (!vacant(i)) {
            uint32_t par = nodes[2 * i + 1] & kMask;
            if (par < nn) ++cnt[par + 1];
        }
    std::partial_sum(cnt.begin(), cnt.end(), cnt.begin());
    std::vector<uint32_t> kids(cnt[nn]);
    std::vector<uint32_t> fill(cnt.begin(), cnt.end() - 1);
    for (uint32_t i = 1; i < nn; ++i)
        if (!vacant(i)) {
            uint32_t par = nodes[2 * i + 1] & kMask;
            if (par < nn) kids[fill[par]++] = i;
        }
    struct Item {
        uint32_t node;
        size_t len;
    };
    std::vector<Item> stack{{0, 0}};
    std::u32string key;
    while (!stack.empty()) {
        Item it = stack.back();
        stack.pop_back();
        key.resize(it.len);
        uint32_t b = nodes[2 * it.node];
        if (it.node != 0) {
            uint32_t par = nodes[2 * it.node + 1] & kMask;
            uint32_t code = (nodes[2 * par] & kMask) ^ it.node;
            if (code == 0) {  // terminal child
                out.emplace_back(key.substr(0, it.len - 1), b & kMask);
                continue;
            }
            if (code >= inv.size()) throw Error(kDecode, "crawdad trie blob: a node's check does not match its parent's base");
            key[it.len - 1] = inv[code];
            if (b & kFlag) {
                out.emplace_back(key, b & kMask);
                continue;
            }
        }
        for (uint32_t k = cnt[it.node]; k < cnt[it.node + 1]; ++k) stack.push_back({kids[k], it.len + 1});
    }
    return out;
}

// ---------------------------------------------------------------------------------------------
// Lexicon
// ---------------------------------------------------------------------------------------------

Lexicon Lexicon::from_entries(const std::vector<RawWordEntry>& entries, uint8_t lex_type) {
    Lexicon lx;
    lx.lex_type = lex_type;
    size_t n = entries.size();
    if (n >= (1u << 30)) throw Error(kTryFromInt, "too many words");
    lx.params.reserve(n);
    lx.feature_off.reserve(n + 1);
    size_t total = 0;
    for (auto& e : entries) total += e.feature.size();
    lx.feature_blob.reserve(total);
    for (auto& e : entries) {
        lx.params.push_back(e.param);
        lx.feature_off.push_back(lx.feature_blob.size());
        lx.feature_blob.append(e.feature);
    }
    lx.feature_off.push_back(lx.feature_blob.size());
    // WordMapBuilder (map.rs:46-73): BTreeMap<String, Vec<u32>>, ids in input order, keys in byte order
    std::vector<uint32_t> order(n);
    std::iota(order.begin(), order.end(), 0u);
    std::stable_sort(order.begin(), order.end(),
                     [&](uint32_t a, uint32_t b) { return entries[a].surface < entries[b].surface; });
    std::vector<std::pair<std::u32string, uint32_t>> recs;
    lx.postings.reserve(2 * n);
    for (size_t i = 0; i < n;) {
        size_t j = i + 1;
        while (j < n && entries[order[j]].surface == entries[order[i]].surface) ++j;
        uint32_t offset = uint32_t(lx.postings.size());  // PostingsBuilder::push posting.rs:33-38
        lx.postings.push_back(uint32_t(j - i));
        for (size_t q = i; q < j; ++q) lx.postings.push_back(order[q]);
        recs.emplace_back(utf8_to_u32(entries[order[i]].surface), offset);
        i = j;
    }
    lx.trie = Trie::from_records(recs);  // UTF-8 byte order == code point order
    return lx;
}

bool Lexicon::verify(uint32_t num_left, uint32_t num_right) const {
    for (auto& p : params)
        if (num_left <= p.left_id || num_right <= p.right_id) return false;
    return true;
}

// ---------------------------------------------------------------------------------------------
// matrix.def
// ---------------------------------------------------------------------------------------------

namespace {

// BufRead::lines(): '\n'-separated, a "\r\n" ending loses the '\r' too.
struct LineReader {
    std::string_view b;
    size_t pos = 0;
    bool next(std::string_view& line) {
        if (pos >= b.size()) return false;
        size_t e = b.find('\n', pos);
        bool has_nl = e != std::string_view::npos;
        if (!has_nl) e = b.size();
        size_t end = e;
        if (has_nl && end > pos && b[end - 1] == '\r') --end;
        line = b.substr(pos, end - pos);
        pos = has_nl ? e + 1 : e;
        return true;
    }
};

std::vector<std::string_view> split_on(std::string_view s, char sep) {
    std::vector<std::string_view> out;
    size_t st = 0;
    for (size_t i = 0; i <= s.size(); ++i)
        if (i == s.size() || s[i] == sep) {
            out.push_back(s.substr(st, i - st));
            st = i + 1;
        }
    return out;
}

bool is_space(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\v' || c == '\f'; }

std::vector<std::string_view> split_ws(std::string_view s) {
    std::vector<std::string_view> out;
    size_t i = 0;
    while (i < s.size()) {
        while (i < s.size() && is_space(s[i])) ++i;
        size_t st = i;
        while (i < s.size() && !is_space(s[i])) ++i;
        if (i > st) out.push_back(s.substr(st, i - st));
    }
    return out;
}

}  // namespace

MatrixConnector MatrixConnector::from_text(std::string_view text) {
    LineReader lr{text};
    std::string_view line;
    if (!lr.next(line)) throw Error(kInvalidFormat, "matrix.def: empty");
    auto cols = split_on(line, ' ');
    uint16_t nr, nl;
    if (cols.size() != 2)  // parse_header :53-64
        throw Error(kInvalidFormat, "matrix.def: The header must consists of two integers separated by spaces, " + std::string(line));
    if (!parse_strict<uint16_t>(cols[0], nr) || !parse_strict<uint16_t>(cols[1], nl))
        throw Error(kParseInt, "matrix.def: invalid header " + std::string(line));
    MatrixConnector m;
    m.num_right = nr;
    m.num_left = nl;
    m.data.assign(size_t(nr) * nl, 0);
    while (lr.next(line)) {
        if (line.empty()) continue;
        cols = split_on(line, ' ');  // parse_body :66-77
        if (cols.size() != 3)
            throw Error(kInvalidFormat, "matrix.def: A row other than the header must consists of three integers separated by spaces, " + std::string(line));
        uint64_t r, l;
        int16_t c;
        if (!parse_strict<uint64_t>(cols[0], r) || !parse_strict<uint64_t>(cols[1], l) || !parse_strict<int16_t>(cols[2], c))
            throw Error(kParseInt, "matrix.def: invalid row " + std::string(line));
        if (nr <= r || nl <= l) throw Error(kInvalidFormat, "matrix.def: left/right_id must be within num_left/right.");
        m.data[size_t(l) * nr + size_t(r)] = c;
    }
    return m;
}

// ---------------------------------------------------------------------------------------------
// char.def
// ---------------------------------------------------------------------------------------------

namespace {
constexpr int kCateBits = 18, kBaseBits = 8;
constexpr uint32_t kCateMask = (1u << kCateBits) - 1;

uint32_t make_char_info(uint32_t cate_idset, uint32_t base_id, bool invoke, bool group, uint32_t length) {  // character.rs:40-63
    return cate_idset | (base_id << kCateBits) | (uint32_t(invoke) << (kCateBits + kBaseBits)) |
           (uint32_t(group) << (kCateBits + kBaseBits + 1)) | (length << (kCateBits + kBaseBits + 2));
}

bool parse_hex_usize(std::string_view s, uint64_t& out) {
    while (s.size() >= 2 && s[0] == '0' && s[1] == 'x') s.remove_prefix(2);  // trim_start_matches("0x")
    if (!s.empty() && s[0] == '+') s.remove_prefix(1);
    if (s.empty() || s.size() > 15) return false;
    uint64_t v = 0;
    for (char c : s) {
        int d = (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : (c >= 'A' && c <= 'F') ? c - 'A' + 10 : -1;
        if (d < 0) return false;
        v = v * 16 + unsigned(d);
    }
    out = v;
    return true;
}
}  // namespace

int CharProperty::cate_id(std::string_view name) const {
    for (size_t i = 0; i < categories.size(); ++i)
        if (categories[i] == name) return int(i);
    return -1;
}

CharProperty CharProperty::from_text(std::string_view text) {
    CharProperty cp;
    cp.categories.push_back("DEFAULT");  // :148
    std::map<uint32_t, uint32_t> cate2info;
    struct Range {
        uint32_t start, end;
        std::vector<std::string_view> cats;
    };
    std::vector<Range> ranges;
    LineReader lr{text};
    std::string_view line;
    while (lr.next(line)) {
        while (!line.empty() && is_space(line.front())) line.remove_prefix(1);
        while (!line.empty() && is_space(line.back())) line.remove_suffix(1);
        if (line.empty() || line[0] == '#') continue;
        auto cols = split_ws(line);
        if (line.substr(0, 2) != "0x") {  // parse_char_category :218-244
            if (cols.size() < 4)
                throw Error(kInvalidFormat, "char.def: A character category must consists of four items separated by spaces, " + std::string(line));
            if (cols[1] != "0" && cols[1] != "1") throw Error(kInvalidFormat, "char.def: INVOKE must be 1 or 0.");
            if (cols[2] != "0" && cols[2] != "1") throw Error(kInvalidFormat, "char.def: GROUP must be 1 or 0.");
            uint16_t length;
            if (!parse_strict<uint16_t>(cols[3], length)) throw Error(kParseInt, "char.def: invalid LENGTH");
            int id = cp.cate_id(cols[0]);
            if (id < 0) {
                id = int(cp.categories.size());
                cp.categories.emplace_back(cols[0]);
            }
            if (id >= 256 || length >= 16)  // CharInfo::new(..).unwrap() :165
                throw Error(kInvalidFormat, "char.def: category id or LENGTH out of range");
            cate2info[uint32_t(id)] = make_char_info(0, uint32_t(id), cols[1] == "1", cols[2] == "1", length);
        } else {  // parse_char_range :246-281
            if (cols.size() < 2)
                throw Error(kInvalidFormat, "char.def: A character range must have two items at least, " + std::string(line));
            uint64_t start, end;
            size_t dd = cols[0].find("..");
            if (dd == std::string_view::npos) {
                if (!parse_hex_usize(cols[0], start)) throw Error(kParseInt, "char.def: invalid code point");
                end = start + 1;
            } else {
                std::string_view rhs = cols[0].substr(dd + 2);
                size_t d2 = rhs.find("..");
                if (d2 != std::string_view::npos) rhs = rhs.substr(0, d2);
                if (!parse_hex_usize(cols[0].substr(0, dd), start) || !parse_hex_usize(rhs, end))
                    throw Error(kParseInt, "char.def: invalid code point range");
                end += 1;
            }
            if (start >= end)
                throw Error(kInvalidFormat, "char.def: The start of a character range must be no more than the end, " + std::string(line));
            if (start > 0xFFFF || end > 0x10000)
                throw Error(kInvalidFormat, "char.def: A character range must be no more 0xFFFF, " + std::string(line));
            Range r{uint32_t(start), uint32_t(end), {}};
            for (size_t i = 1; i < cols.size(); ++i) {
                if (cols[i][0] == '#') break;
                r.cats.push_back(cols[i]);
            }
            ranges.push_back(std::move(r));
        }
    }
    auto encode = [&](const std::vector<std::string_view>& targets) -> uint32_t {  // encode_cate_info :193-216
        int base_id = targets.empty() ? -1 : cp.cate_id(targets[0]);
        auto it = base_id < 0 ? cate2info.end() : cate2info.find(uint32_t(base_id));
        if (it == cate2info.end())
            throw Error(kInvalidFormat, "char.def: Undefined category: " + std::string(targets.empty() ? "" : targets[0]));
        uint32_t info = it->second;
        uint32_t idset = info & kCateMask;
        for (auto t : targets) {
            int id = cp.cate_id(t);
            auto jt = id < 0 ? cate2info.end() : cate2info.find(uint32_t(id));
            if (jt == cate2info.end()) throw Error(kInvalidFormat, "char.def: Undefined category: " + std::string(t));
            idset |= 1u << ((jt->second >> kCateBits) & 0xFF);
        }
        return (info & ~kCateMask) | idset;  // reset_cate_idset :66-69
    };
    uint32_t init = encode({std::string_view("DEFAULT")});
    cp.chr2inf.assign(1u << 16, init);
    for (auto& r : ranges) {
        uint32_t ci = encode(r.cats);
        for (uint32_t c = r.start; c < r.end; ++c) cp.chr2inf[c] = ci;
    }
    return cp;
}

// ---------------------------------------------------------------------------------------------
// unk.def
// ---------------------------------------------------------------------------------------------

UnkHandler UnkHandler::from_text(std::string_view text, const CharProperty& cp) {
    auto parsed = parse_lexicon_csv(text, "unk.def");
    std::vector<std::vector<UnkEntry>> by_cate(cp.categories.size());
    for (auto& item : parsed) {
        int id = cp.cate_id(item.surface);
        if (id < 0) throw Error(kInvalidFormat, "unk.def: Undefined category: " + item.surface);
        by_cate[size_t(id)].push_back(UnkEntry{uint16_t(id), item.param.left_id, item.param.right_id,
                                               item.param.word_cost, std::string(item.feature)});
    }
    UnkHandler h;
    for (auto& v : by_cate) {
        h.offsets.push_back(h.entries.size());
        for (auto& e : v) h.entries.push_back(std::move(e));
    }
    h.offsets.push_back(h.entries.size());
    return h;
}

bool UnkHandler::verify(uint32_t num_left, uint32_t num_right) const {
    for (auto& e : entries)
        if (num_left <= e.left_id || num_right <= e.right_id) return false;
    return true;
}

// ---------------------------------------------------------------------------------------------
// Dictionary
// ---------------------------------------------------------------------------------------------

void Dictionary::finish_build(std::string_view lex_csv, std::string_view char_def, std::string_view unk_def) {
    auto entries = parse_lexicon_csv(lex_csv, "lex.csv");     // builder.rs:79
    char_prop = CharProperty::from_text(char_def);           // :81
    unk = UnkHandler::from_text(unk_def, char_prop);         // :82
    system = Lexicon::from_entries(entries, kSystem);        // builder.rs:22
    if (!system.verify(num_left(), num_right()))             // :24-29
        throw Error(kInvalidArgument, "system_lexicon_rdr includes invalid connection ids.");
    if (!unk.verify(num_left(), num_right()))                // :30-35
        throw Error(kInvalidArgument, "unk_handler_rdr includes invalid connection ids.");
}

Dictionary Dictionary::from_mecab(std::string_view lex_csv, std::string_view matrix_def, std::string_view char_def,
                                  std::string_view unk_def) {
    Dictionary d;
    d.matrix = MatrixConnector::from_text(matrix_def);
    d.finish_build(lex_csv, char_def, unk_def);
    return d;
}

Dictionary Dictionary::from_parts(std::string_view lex_csv, const int16_t* matrix, uint32_t num_right, uint32_t num_left,
                                  std::string_view char_def, std::string_view unk_def) {
    if (num_right > 65535 || num_left > 65535) throw Error(kInvalidArgument, "connection ids must fit u16");
    Dictionary d;
    d.matrix.num_right = num_right;
    d.matrix.num_left = num_left;
    d.matrix.data.assign(matrix, matrix + size_t(num_right) * num_left);
    d.finish_build(lex_csv, char_def, unk_def);
    return d;
}

// ---------------------------------------------------------------------------------------------
// RawConnector (connector/raw_connector.rs, raw_connector/scorer.rs)
// ---------------------------------------------------------------------------------------------

bool next_line(std::string_view text, size_t& pos, std::string_view& line) {
    LineReader lr{text, pos};
    const bool ok = lr.next(line);
    pos = lr.pos;
    return ok;
}

// utils::parse_csv_row (utils.rs:41-61)
std::vector<std::string> parse_csv_row(std::string_view row) {
    std::vector<std::string> out;
    if (row.empty()) {
        out.emplace_back();
        return out;
    }
    CsvFields rdr(row);
    std::string field;
    for (;;) {
        CsvFields::Field f = rdr.read(field);
        if (f.kind == CsvFields::Kind::kEnd) break;
        out.push_back(field);
        if (f.record_end) break;
    }
    return out;
}

void RawConnector::build_scorer(std::vector<std::array<int64_t, 3>> triples, size_t min_bases) {
    // BTreeMap per key1 (scorer.rs:115-121): ascending key2, the last insert of a pair wins
    std::stable_sort(triples.begin(), triples.end(), [](const auto& a, const auto& b) {
        return a[0] != b[0] ? a[0] < b[0] : a[1] < b[1];
    });
    std::vector<std::array<int64_t, 3>> uniq;
    for (size_t i = 0; i < triples.size(); ++i) {
        if (i + 1 < triples.size() && triples[i + 1][0] == triples[i][0] && triples[i + 1][1] == triples[i][1]) continue;
        uniq.push_back(triples[i]);
    }
    bases.assign(std::max(min_bases, uniq.empty() ? size_t(0) : size_t(uniq.back()[0]) + 1), 0);
    checks.clear();
    costs.clear();
    for (size_t i = 0; i < uniq.size();) {
        size_t j = i;
        while (j < uniq.size() && uniq[j][0] == uniq[i][0]) ++j;
        uint32_t base = 0;
        for (;; ++base) {  // check_base scorer.rs:123-131: slots beyond the current end are free
            bool ok = true;
            for (size_t q = i; q < j && ok; ++q) {
                size_t pos = base ^ uint32_t(uniq[q][1]);
                ok = pos >= checks.size() || checks[pos] == kUnusedCheck;
            }
            if (ok) break;
        }
        bases[size_t(uniq[i][0])] = base;
        for (size_t q = i; q < j; ++q) {
            size_t pos = base ^ uint32_t(uniq[q][1]);
            if (pos >= checks.size()) {
                checks.resize(pos + 1, kUnusedCheck);
                costs.resize(pos + 1, 0);
            }
            checks[pos] = uint32_t(uniq[i][0]);
            costs[pos] = int32_t(uniq[q][2]);
        }
        i = j;
    }
}

int32_t RawConnector::accumulate(const uint32_t* keys1, const uint32_t* keys2, size_t n) const {
    uint32_t score = 0;
    for (size_t t = 0; t < n; ++t) {
        uint32_t k1 = keys1[t], k2 = keys2[t];
        if (k1 < bases.size()) {
            size_t pos = bases[k1] ^ k2;
            if (pos < checks.size() && checks[pos] == k1) score += uint32_t(costs[pos]);
        }
    }
    return int32_t(score);
}

namespace {
// RawConnectorBuilder (raw_connector.rs:163-245): feature-id rows of bigram.right / bigram.left and the
// (right feature, left feature, cost) triples of bigram.cost, before any padding.
struct BigramInfo {
    std::vector<std::vector<uint32_t>> right_rows, left_rows;  // row i belongs to connection id i + 1
    size_t feat_T = 0;                                          // longest row (feat_template_size)
    std::vector<std::array<int64_t, 3>> triples;               // insertion order
    size_t trie_len = 0;                                        // ScorerBuilder::trie.len() = max key1 + 1
};

BigramInfo parse_bigram(std::string_view bigram_right, std::string_view bigram_left, std::string_view bigram_cost) {
    BigramInfo bi;
    std::unordered_map<std::string, uint32_t> rmap{{"", 0}}, lmap{{"", 0}};  // raw_connector.rs:195-198
    LineReader lr{bigram_cost};
    std::string_view line;
    while (lr.next(line)) {  // parse_cost raw_connector.rs:276-321
        auto cols = split_on(line, '\t');
        int32_t cost;
        if (cols.size() != 2) throw Error(kInvalidFormat, "bigram.cost: The format must be right/left<tab>cost, " + std::string(line));
        if (!parse_strict<int32_t>(cols[1], cost)) throw Error(kParseInt, "bigram.cost: invalid cost " + std::string(line));
        auto feats = split_on(cols[0], '/');
        if (feats.size() != 2) throw Error(kInvalidFormat, "bigram.cost: The format must be right/left<tab>cost, " + std::string(line));
        uint32_t rid = rmap.try_emplace(std::string(feats[0]), uint32_t(rmap.size())).first->second;
        uint32_t lid = lmap.try_emplace(std::string(feats[1]), uint32_t(lmap.size())).first->second;
        bi.triples.push_back({int64_t(rid), int64_t(lid), int64_t(cost)});
        bi.trie_len = std::max(bi.trie_len, size_t(rid) + 1);
    }
    auto read_side = [&](std::string_view text, const std::unordered_map<std::string, uint32_t>& ids, const char* name) {
        std::vector<std::vector<uint32_t>> rows;
        LineReader r{text};
        std::string_view ln;
        while (r.next(ln)) {  // parse_features raw_connector.rs:252-274
            auto cols = split_on(ln, '\t');
            uint64_t id;
            if (cols.size() != 2) throw Error(kInvalidFormat, std::string(name) + ": The format must be id<tab>csv_row, " + std::string(ln));
            if (!parse_strict<uint64_t>(cols[0], id)) throw Error(kParseInt, std::string(name) + ": invalid id");
            if (id != rows.size() + 1) throw Error(kInvalidFormat, std::string(name) + ": must be ascending order");
            std::vector<uint32_t> feats;
            for (auto& f : parse_csv_row(cols[1])) {
                auto it = ids.find(f);
                feats.push_back(it == ids.end() ? RawConnector::kInvalidFeature : it->second);
            }
            bi.feat_T = std::max(bi.feat_T, feats.size());
            rows.push_back(std::move(feats));
        }
        return rows;
    };
    bi.right_rows = read_side(bigram_right, rmap, "bigram.right");
    bi.left_rows = read_side(bigram_left, lmap, "bigram.left");
    if (bi.right_rows.size() + 1 > 65536 || bi.left_rows.size() + 1 > 65536)
        throw Error(kTryFromInt, "bigram: too many connection ids");
    return bi;
}

RawConnector raw_from_bigram(BigramInfo&& bi) {
    RawConnector c;
    size_t T = bi.feat_T;
    if (T != 0) T = ((T - 1) / 8 + 1) * 8;  // raw_connector.rs:64-66
    c.feat_T = uint32_t(T);
    c.num_right = uint32_t(bi.right_rows.size()) + 1;
    c.num_left = uint32_t(bi.left_rows.size()) + 1;
    auto fill = [&](std::vector<uint32_t>& dst, const std::vector<std::vector<uint32_t>>& rows) {
        dst.assign((rows.size() + 1) * T, RawConnector::kInvalidFeature);  // raw_connector.rs:72-92
        std::fill(dst.begin(), dst.begin() + T, 0u);                        // BOS/EOS row: zeros
        for (size_t i = 0; i < rows.size(); ++i) std::copy(rows[i].begin(), rows[i].end(), dst.begin() + (i + 1) * T);
    };
    fill(c.right_feats, bi.right_rows);
    fill(c.left_feats, bi.left_rows);
    c.build_scorer(std::move(bi.triples));
    return c;
}

struct VecHash {
    size_t operator()(const std::vector<uint32_t>& v) const {
        uint64_t h = 0xcbf29ce484222325ull ^ v.size();
        for (uint32_t x : v) h = (h ^ x) * 0x100000001b3ull;
        return size_t(h ^ (h >> 29));
    }
};

// DualConnector::remove_feature_templates_greedy (dual_connector.rs:27-70): eight times, drop the
// template whose removal leaves the smallest (distinct right rows) x (distinct left rows) product.
// The reference walks a hashbrown HashSet here, so which of several equally good templates it drops
// follows that set's iteration order; ties are settled by ascending template index in this build (the
// last minimal one wins, as `<=` does over an ascending walk).  The split only decides where a
// template's cost is stored: DualConnector::cost is the same sum over all templates either way, up to
// the i16 clamp of the matrix part (dual_connector.rs:104).
std::vector<char> dual_matrix_templates(const BigramInfo& bi, size_t raw_templates) {
    const size_t T = bi.feat_T;
    std::vector<char> in(T, 1);
    auto distinct = [&](const std::vector<std::vector<uint32_t>>& rows, size_t trial) {
        std::unordered_set<std::vector<uint32_t>, VecHash> seen;
        std::vector<uint32_t> key;
        for (auto& row : rows) {
            key.clear();
            for (size_t i = 0; i < T && i < row.size(); ++i)
                if (in[i] && i != trial) key.push_back(row[i]);
            seen.insert(key);
        }
        return seen.size();
    };
    for (size_t round = 0; round < raw_templates; ++round) {
        size_t cand = 0, best = bi.left_rows.size() * bi.right_rows.size();
        for (size_t trial = 0; trial < T; ++trial) {
            if (!in[trial]) continue;
            const size_t sz = distinct(bi.right_rows, trial) * distinct(bi.left_rows, trial);
            if (sz <= best) {
                best = sz;
                cand = trial;
            }
        }
        in[cand] = 0;
    }
    return in;
}

// DualConnector::from_readers (dual_connector.rs:155-213)
void dual_from_bigram(Dictionary& d, BigramInfo&& bi) {
    const size_t T = bi.feat_T;
    if (T < 8)  // `feat_template_size - SIMD_SIZE` (dual_connector.rs:82) underflows in the reference
        throw Error(kInvalidArgument, "bigram: the Dual connector needs at least 8 feature templates");
    RawConnector full;
    full.build_scorer(bi.triples);
    const std::vector<char> in = dual_matrix_templates(bi, 8);
    std::vector<size_t> matrix_idx, raw_idx;
    for (size_t i = 0; i < T; ++i) (in[i] ? matrix_idx : raw_idx).push_back(i);

    // create_matrix_connector (dual_connector.rs:72-110)
    const size_t P = (matrix_idx.size() + 7) / 8 * 8;  // U31x8::to_simd_vec pads with zeros (scorer.rs:27-46)
    auto feature_map = [&](const std::vector<std::vector<uint32_t>>& rows, std::vector<uint16_t>& conn_id_map,
                           std::vector<std::vector<uint32_t>>& by_id) {
        std::unordered_map<std::vector<uint32_t>, uint32_t, VecHash> feats_map;
        conn_id_map.assign(1, 0);
        feats_map.emplace(std::vector<uint32_t>(matrix_idx.size(), 0u), 0u);
        by_id.assign(1, std::vector<uint32_t>(P, 0u));
        for (auto& row : rows) {
            std::vector<uint32_t> feats;
            for (size_t idx : matrix_idx) feats.push_back(idx < row.size() ? row[idx] : RawConnector::kInvalidFeature);
            auto [it, fresh] = feats_map.try_emplace(feats, uint32_t(feats_map.size()));
            if (it->second > 0xFFFF) throw Error(kTryFromInt, "bigram: the reduced matrix has too many ids");
            if (fresh) {
                feats.resize(P, 0u);
                by_id.push_back(std::move(feats));
            }
            conn_id_map.push_back(uint16_t(it->second));
        }
    };
    std::vector<std::vector<uint32_t>> rfeat, lfeat;
    feature_map(bi.right_rows, d.dual_right_map, rfeat);
    feature_map(bi.left_rows, d.dual_left_map, lfeat);
    d.matrix.num_right = uint32_t(rfeat.size());
    d.matrix.num_left = uint32_t(lfeat.size());
    d.matrix.data.assign(rfeat.size() * lfeat.size(), 0);
    for (size_t l = 0; l < lfeat.size(); ++l)
        for (size_t r = 0; r < rfeat.size(); ++r) {
            const int32_t c = full.accumulate(rfeat[r].data(), lfeat[l].data(), P);
            d.matrix.data[l * rfeat.size() + r] = int16_t(std::clamp(c, -32768, 32767));
        }

    // create_raw_connector (dual_connector.rs:112-153): a zero row for BOS/EOS, then the eight raw templates
    auto raw_rows = [&](const std::vector<std::vector<uint32_t>>& rows, std::vector<uint32_t>& out) {
        out.assign(8, 0u);
        for (auto& row : rows)
            for (size_t idx : raw_idx) out.push_back(idx < row.size() ? row[idx] : RawConnector::kInvalidFeature);
    };
    d.raw = RawConnector{};
    raw_rows(bi.right_rows, d.raw.right_feats);
    raw_rows(bi.left_rows, d.raw.left_feats);
    d.raw.feat_T = 8;
    d.raw.num_right = uint32_t(bi.right_rows.size()) + 1;
    d.raw.num_left = uint32_t(bi.left_rows.size()) + 1;
    std::unordered_set<uint32_t> right_used(d.raw.right_feats.begin(), d.raw.right_feats.end()),
        left_used(d.raw.left_feats.begin(), d.raw.left_feats.end());
    std::vector<std::array<int64_t, 3>> kept;  // the scorer keeps only pairs the raw rows can reach
    for (auto& t : bi.triples)
        if (right_used.count(uint32_t(t[0])) && left_used.count(uint32_t(t[1]))) kept.push_back(t);
    d.raw.build_scorer(std::move(kept), bi.trie_len);
}
}  // namespace

RawConnector RawConnector::from_text(std::string_view bigram_right, std::string_view bigram_left,
                                     std::string_view bigram_cost) {
    return raw_from_bigram(parse_bigram(bigram_right, bigram_left, bigram_cost));
}

Dictionary Dictionary::from_bigram(std::string_view lex_csv, std::string_view bigram_right, std::string_view bigram_left,
                                   std::string_view bigram_cost, std::string_view char_def, std::string_view unk_def,
                                   bool dual_connector) {
    Dictionary d;
    BigramInfo bi = parse_bigram(bigram_right, bigram_left, bigram_cost);
    if (dual_connector) {
        d.connector_kind = kDual;
        dual_from_bigram(d, std::move(bi));
    } else {
        d.connector_kind = kRaw;
        d.raw = raw_from_bigram(std::move(bi));
    }
    d.finish_build(lex_csv, char_def, unk_def);
    return d;
}

void Dictionary::reset_user_lexicon(std::optional<std::string_view> csv) {
    if (!csv) {
        user.reset();
        return;
    }
    auto entries = parse_lexicon_csv(*csv, "lex.csv");  // Lexicon::from_reader lexicon.rs:99-109
    Lexicon lx = Lexicon::from_entries(entries, kUser);
    if (mapper) {  // dictionary.rs:215-217
        for (auto& p : lx.params) {
            if (p.left_id >= mapper->left.size() || p.right_id >= mapper->right.size())
                throw Error(kInvalidArgument, "user_lexicon_rdr includes invalid connection ids.");
            p.left_id = mapper->left[p.left_id];
            p.right_id = mapper->right[p.right_id];
        }
    }
    if (!lx.verify(num_left(), num_right()))  // :218-223
        throw Error(kInvalidArgument, "user_lexicon_rdr includes invalid connection ids.");
    user = std::move(lx);
}

namespace {
// ConnIdMapper::parse (mapper.rs:49-80) -> new_ids[old_id]
std::vector<uint16_t> parse_conn_id_map(const std::vector<uint16_t>& map) {
    if (map.size() + 1 > 65536) throw Error(kTryFromInt, "map: too many ids");
    std::vector<uint16_t> new_ids(map.size() + 1, 0xFFFF);
    new_ids[0] = 0;  // BOS_EOS_CONNECTION_ID stays (common.rs:18)
    for (size_t i = 0; i < map.size(); ++i) {
        uint16_t old_id = map[i];
        if (old_id == 0) throw Error(kInvalidArgument, "map: Id 0 is reserved.");
        if (old_id >= new_ids.size()) throw Error(kInvalidArgument, "map: ids are out of range.");
        if (new_ids[old_id] != 0xFFFF) throw Error(kInvalidArgument, "map: ids are duplicate.");
        new_ids[old_id] = uint16_t(i + 1);
    }
    return new_ids;
}
}  // namespace

void Dictionary::map_connection_ids(const std::vector<uint16_t>& lmap, const std::vector<uint16_t>& rmap) {
    ConnIdMapper m{parse_conn_id_map(lmap), parse_conn_id_map(rmap)};
    // MatrixConnector::map_connection_ids asserts an exact cover (matrix_connector.rs:100-101)
    if (m.left.size() != num_left() || m.right.size() != num_right())
        throw Error(kInvalidArgument, "map: the mapping must cover every connection id of the connector");
    auto remap = [&](Lexicon& lx) {  // WordParams::map_connection_ids param.rs:48-53
        for (auto& p : lx.params) {
            p.left_id = m.left[p.left_id];
            p.right_id = m.right[p.right_id];
        }
    };
    remap(system);
    if (user) remap(*user);
    if (connector_kind != kMatrix) {  // RawConnector::map_connection_ids raw_connector.rs:124-152;
        const size_t T = raw.feat_T;  // DualConnector moves its feature rows the same way (dual_connector.rs:227-245)
        std::vector<uint32_t> mr(raw.right_feats.size()), ml(raw.left_feats.size());
        for (size_t r = 0; r < raw.num_right; ++r)
            std::copy_n(raw.right_feats.begin() + r * T, T, mr.begin() + size_t(m.right[r]) * T);
        for (size_t l = 0; l < raw.num_left; ++l)
            std::copy_n(raw.left_feats.begin() + l * T, T, ml.begin() + size_t(m.left[l]) * T);
        raw.right_feats.swap(mr);
        raw.left_feats.swap(ml);
    }
    auto remap_matrix = [&](const std::vector<uint16_t>& new_left, const std::vector<uint16_t>& new_right) {
        const size_t nr = matrix.num_right, nl = matrix.num_left;
        std::vector<int16_t> mapped(matrix.data.size(), 0);  // matrix_connector.rs:103-115
        for (size_t l = 0; l < nl; ++l) {
            const int16_t* src = matrix.data.data() + l * nr;
            int16_t* dst = mapped.data() + size_t(new_left[l]) * nr;
            for (size_t r = 0; r < nr; ++r) dst[new_right[r]] = src[r];
        }
        matrix.data.swap(mapped);
    };
    if (connector_kind == kMatrix) remap_matrix(m.left, m.right);
    if (connector_kind == kDual) {  // dual_connector.rs:227-266
        auto move_ids = [](std::vector<uint16_t>& ids, const std::vector<uint16_t>& new_of_old) {
            std::vector<uint16_t> moved(ids.size(), 0);
            for (size_t i = 0; i < ids.size(); ++i) moved[new_of_old[i]] = ids[i];
            ids.swap(moved);
        };
        move_ids(dual_right_map, m.right);
        move_ids(dual_left_map, m.left);
        // the reduced matrix is renumbered in the order its ids now appear (dual_connector.rs:247-265)
        auto first_seen = [](std::vector<uint16_t>& ids, size_t n_matrix_ids) {
            std::vector<uint16_t> renum(n_matrix_ids, 0xFFFF);
            uint16_t next = 0;
            for (auto& i : ids) {
                if (renum[i] == 0xFFFF) renum[i] = next++;
                i = renum[i];
            }
            return renum;
        };
        std::vector<uint16_t> ml2 = first_seen(dual_left_map, matrix.num_left);
        std::vector<uint16_t> mr2 = first_seen(dual_right_map, matrix.num_right);
        for (uint16_t v : ml2)
            if (v == 0xFFFF) throw Error(kInvalidArgument, "map: the reduced matrix holds an id no connection id uses");
        for (uint16_t v : mr2)
            if (v == 0xFFFF) throw Error(kInvalidArgument, "map: the reduced matrix holds an id no connection id uses");
        remap_matrix(ml2, mr2);
    }
    for (auto& e : unk.entries) {  // unknown.rs:203-208
        e.left_id = m.left[e.left_id];
        e.right_id = m.right[e.right_id];
    }
    mapper = std::move(m);  // dictionary.rs:257
}

WordParam Dictionary::word_param(uint32_t word_idx) const {
    uint32_t lex = word_idx >> 30, id = word_idx & 0x3FFFFFFFu;
    if (lex == kUnknown) {
        if (id >= unk.entries.size()) throw Error(kInvalidArgument, "word_idx out of range");
        auto& e = unk.entries[id];
        return WordParam{e.left_id, e.right_id, e.word_cost};
    }
    const Lexicon* lx = lex == kSystem ? &system : (user ? &*user : nullptr);
    if (lex > kUnknown || !lx || id >= lx->num_words()) throw Error(kInvalidArgument, "word_idx out of range");
    return lx->params[id];
}

std::string_view Dictionary::word_feature(uint32_t word_idx) const {
    uint32_t lex = word_idx >> 30, id = word_idx & 0x3FFFFFFFu;
    if (lex == kUnknown) {
        if (id >= unk.entries.size()) throw Error(kInvalidArgument, "word_idx out of range");
        return unk.entries[id].feature;
    }
    const Lexicon* lx = lex == kSystem ? &system : (user ? &*user : nullptr);
    if (lex > kUnknown || !lx || id >= lx->num_words()) throw Error(kInvalidArgument, "word_idx out of range");
    return lx->feature(id);
}

// ---------------------------------------------------------------------------------------------
// `.dic` stream: magic + bincode 2 (little endian, fixed-width ints; common.rs:5-9).
// Layout per SURVEY.md Appendix A — derived from the struct definitions, not pinned by any
// reference test ("parity unpinned" for the byte layout).
// ---------------------------------------------------------------------------------------------

namespace {
const char kMagic[] = "VibratoTokenizer 0.5\n";  // dictionary.rs:27

struct BinReader {
    const uint8_t* p;
    size_t n, pos = 0;
    void need(size_t k) {
        if (k > n - pos) throw Error(kDecode, "unexpected end of dictionary stream");
    }
    template <typename T>
    T get() {
        need(sizeof(T));
        T v;
        std::memcpy(&v, p + pos, sizeof(T));
        pos += sizeof(T);
        return v;
    }
    uint64_t len(size_t elem) {
        uint64_t l = get<uint64_t>();
        if (elem && l > (n - pos) / elem) throw Error(kDecode, "length prefix exceeds the stream");
        return l;
    }
    template <typename T>
    void vec(std::vector<T>& out) {
        uint64_t l = len(sizeof(T));
        out.resize(l);
        if (l) std::memcpy(out.data(), p + pos, l * sizeof(T));
        pos += l * sizeof(T);
    }
    std::string_view str() {
        uint64_t l = len(1);
        std::string_view s(reinterpret_cast<const char*>(p + pos), l);
        if (!utf8_valid(p + pos, l)) throw Error(kDecode, "invalid utf-8 in string");
        pos += l;
        return s;
    }
};

struct BinWriter {
    std::vector<uint8_t>& out;
    template <typename T>
    void put(T v) {
        const uint8_t* b = reinterpret_cast<const uint8_t*>(&v);
        out.insert(out.end(), b, b + sizeof(T));
    }
    template <typename T>
    void vec(const std::vector<T>& v) {
        put<uint64_t>(v.size());
        const uint8_t* b = reinterpret_cast<const uint8_t*>(v.data());
        out.insert(out.end(), b, b + v.size() * sizeof(T));
    }
    void str(std::string_view s) {
        put<uint64_t>(s.size());
        out.insert(out.end(), s.begin(), s.end());
    }
};

Lexicon read_lexicon(BinReader& r) {
    Lexicon lx;
    std::vector<uint8_t> blob;
    r.vec(blob);  // trie.rs:14-19
    lx.trie = Trie::deserialize(blob.data(), blob.size());
    r.vec(lx.postings);
    {  // Vec<WordParam>: 3 x 16 bit, no padding
        uint64_t l = r.len(6);
        lx.params.resize(l);
        for (auto& p : lx.params) {
            p.left_id = r.get<uint16_t>();
            p.right_id = r.get<uint16_t>();
            p.word_cost = r.get<int16_t>();
        }
    }
    uint64_t nf = r.len(8);
    lx.feature_off.reserve(nf + 1);
    for (uint64_t i = 0; i < nf; ++i) {
        lx.feature_off.push_back(lx.feature_blob.size());
        lx.feature_blob.append(r.str());
    }
    lx.feature_off.push_back(lx.feature_blob.size());
    uint32_t lt = r.get<uint32_t>();
    if (lt > 2) throw Error(kDecode, "bad LexType variant");
    lx.lex_type = uint8_t(lt);
    if (nf != lx.params.size()) throw Error(kDecode, "lexicon: params/features length mismatch");
    // The blob layout is not pinned by any reference test: cross-check it against the rest of the
    // lexicon.  Every key's value must be the start of a postings list, and together the lists must
    // name every word exactly once (WordMapBuilder::build, map.rs:60-70).
    {
        std::vector<uint8_t> is_start(lx.postings.size() + 1, 0);
        for (size_t i = 0; i < lx.postings.size(); i += 1 + size_t(lx.postings[i])) is_start[i] = 1;
        size_t words = 0;
        for (auto& kv : lx.trie.enumerate()) {
            if (kv.second >= lx.postings.size() || !is_start[kv.second])
                throw Error(kDecode, "lexicon: a trie value is not a postings offset (unexpected crawdad blob layout?)");
            words += lx.postings[kv.second];
        }
        if (words != lx.params.size())
            throw Error(kDecode, "lexicon: trie keys and word parameters disagree (unexpected crawdad blob layout?)");
    }
    // postings ids and trie values must stay inside their arrays (the device trusts them)
    for (size_t i = 0; i < lx.postings.size();) {
        uint64_t l = lx.postings[i];
        if (i + 1 + l > lx.postings.size()) throw Error(kDecode, "lexicon: postings overrun");
        for (uint64_t k = 0; k < l; ++k)
            if (lx.postings[i + 1 + k] >= lx.params.size()) throw Error(kDecode, "lexicon: word id out of range");
        i += 1 + l;
    }
    return lx;
}

void write_lexicon(BinWriter& w, const Lexicon& lx) {
    std::vector<uint8_t> blob;
    lx.trie.serialize(blob);
    w.vec(blob);
    w.vec(lx.postings);
    w.put<uint64_t>(lx.params.size());
    for (auto& p : lx.params) {
        w.put<uint16_t>(p.left_id);
        w.put<uint16_t>(p.right_id);
        w.put<int16_t>(p.word_cost);
    }
    w.put<uint64_t>(lx.num_words());
    for (uint32_t i = 0; i < lx.num_words(); ++i) w.str(lx.feature(i));
    w.put<uint32_t>(lx.lex_type);
}
}  // namespace

Dictionary Dictionary::read(const uint8_t* p, size_t n) {
    const size_t ml = sizeof(kMagic) - 1;
    if (n < ml) throw Error(kIo, "failed to fill whole buffer");  // read_exact dictionary.rs:187
    if (std::memcmp(p, kMagic, ml) != 0)
        throw Error(kInvalidArgument, "rdr: The magic number of the input model mismatches.");  // :188-193
    BinReader r{p + ml, n - ml};
    Dictionary d;
    d.system = read_lexicon(r);
    if (uint8_t tag = r.get<uint8_t>(); tag == 1)
        d.user = read_lexicon(r);
    else if (tag != 0)
        throw Error(kDecode, "bad Option tag");
    uint32_t kind = r.get<uint32_t>();
    auto feat_rows = [&](std::vector<uint32_t>& out) {  // Vec<U31x8>: u64 count, then 8 x u32 each
        uint64_t cnt = r.len(32);
        out.resize(cnt * 8);
        for (auto& v : out) {
            v = r.get<uint32_t>();
            if (v > RawConnector::kInvalidFeature) throw Error(kDecode, "U31 out of range");  // num.rs:38-47
        }
    };
    auto read_matrix = [&] {  // MatrixConnector matrix_connector.rs:11-15
        r.vec(d.matrix.data);
        uint64_t nr = r.get<uint64_t>(), nl = r.get<uint64_t>();
        if (nr > 65536 || nl > 65536 || nr * nl != d.matrix.data.size()) throw Error(kDecode, "matrix: shape mismatch");
        d.matrix.num_right = uint32_t(nr);
        d.matrix.num_left = uint32_t(nl);
    };
    if (kind == kDual) {  // DualConnector dual_connector.rs:15-23
        d.connector_kind = kDual;
        read_matrix();
        r.vec(d.dual_right_map);
        r.vec(d.dual_left_map);
        feat_rows(d.raw.right_feats);
        feat_rows(d.raw.left_feats);
        d.raw.feat_T = 8;
        d.raw.num_right = uint32_t(d.raw.right_feats.size() / 8);
        d.raw.num_left = uint32_t(d.raw.left_feats.size() / 8);
        r.vec(d.raw.bases);
        r.vec(d.raw.checks);
        r.vec(d.raw.costs);
        if (d.raw.checks.size() != d.raw.costs.size()) throw Error(kDecode, "scorer: checks/costs length mismatch");
        if (d.dual_right_map.empty() || d.dual_left_map.empty() || d.dual_right_map.size() > 65536 ||
            d.dual_left_map.size() > 65536 || d.raw.num_right != d.dual_right_map.size() ||
            d.raw.num_left != d.dual_left_map.size())
            throw Error(kDecode, "dual connector: id maps and feature rows disagree");
        for (uint16_t v : d.dual_right_map)
            if (v >= d.matrix.num_right) throw Error(kDecode, "dual connector: right id map leaves the matrix");
        for (uint16_t v : d.dual_left_map)
            if (v >= d.matrix.num_left) throw Error(kDecode, "dual connector: left id map leaves the matrix");
    } else if (kind == kRaw) {  // RawConnector raw_connector.rs:22-27, Scorer scorer.rs:198-227
        d.connector_kind = kRaw;
        feat_rows(d.raw.right_feats);
        feat_rows(d.raw.left_feats);
        uint64_t t8 = r.get<uint64_t>();  // feat_template_size in units of SIMD_SIZE
        if (t8 == 0 || t8 > 4096) throw Error(kDecode, "raw connector: bad feat_template_size");
        d.raw.feat_T = uint32_t(t8 * 8);
        if (d.raw.right_feats.size() % d.raw.feat_T || d.raw.left_feats.size() % d.raw.feat_T)
            throw Error(kDecode, "raw connector: feature rows do not divide by the template size");
        d.raw.num_right = uint32_t(d.raw.right_feats.size() / d.raw.feat_T);
        d.raw.num_left = uint32_t(d.raw.left_feats.size() / d.raw.feat_T);
        if (d.raw.num_right > 65536 || d.raw.num_left > 65536) throw Error(kDecode, "raw connector: too many ids");
        r.vec(d.raw.bases);
        r.vec(d.raw.checks);
        r.vec(d.raw.costs);
        if (d.raw.checks.size() != d.raw.costs.size()) throw Error(kDecode, "scorer: checks/costs length mismatch");  // scorer.rs:204-209
    } else if (kind == kMatrix) {
        d.connector_kind = kMatrix;
        read_matrix();
    } else {
        throw Error(kDecode, "bad ConnectorWrapper variant");
    }
    if (uint8_t tag = r.get<uint8_t>(); tag == 1) {
        ConnIdMapper m;
        r.vec(m.left);
        r.vec(m.right);
        d.mapper = std::move(m);
    } else if (tag != 0) {
        throw Error(kDecode, "bad Option tag");
    }
    r.vec(d.char_prop.chr2inf);
    if (d.char_prop.chr2inf.empty()) throw Error(kDecode, "char_prop: empty table");
    uint64_t nc = r.len(8);
    for (uint64_t i = 0; i < nc; ++i) d.char_prop.categories.emplace_back(r.str());
    r.vec(d.unk.offsets);
    uint64_t ne = r.len(16);
    d.unk.entries.resize(ne);
    for (auto& e : d.unk.entries) {
        e.cate_id = r.get<uint16_t>();
        e.left_id = r.get<uint16_t>();
        e.right_id = r.get<uint16_t>();
        e.word_cost = r.get<int16_t>();
        e.feature = std::string(r.str());
    }
    if (d.unk.offsets.empty() || d.unk.offsets.back() > ne) throw Error(kDecode, "unk_handler: bad offsets");
    for (size_t i = 1; i < d.unk.offsets.size(); ++i)
        if (d.unk.offsets[i] < d.unk.offsets[i - 1]) throw Error(kDecode, "unk_handler: bad offsets");
    if (!d.system.verify(d.num_left(), d.num_right()) || !d.unk.verify(d.num_left(), d.num_right()) ||
        (d.user && !d.user->verify(d.num_left(), d.num_right())))
        throw Error(kDecode, "dictionary stream holds connection ids outside the matrix");
    return d;
}

void Dictionary::write(std::vector<uint8_t>& out) const {
    out.insert(out.end(), kMagic, kMagic + sizeof(kMagic) - 1);
    BinWriter w{out};
    write_lexicon(w, system);
    w.put<uint8_t>(user ? 1 : 0);
    if (user) write_lexicon(w, *user);
    if (connector_kind == kDual) {
        w.put<uint32_t>(kDual);
        w.vec(matrix.data);
        w.put<uint64_t>(matrix.num_right);
        w.put<uint64_t>(matrix.num_left);
        w.vec(dual_right_map);
        w.vec(dual_left_map);
        w.put<uint64_t>(raw.right_feats.size() / 8);
        for (uint32_t v : raw.right_feats) w.put<uint32_t>(v);
        w.put<uint64_t>(raw.left_feats.size() / 8);
        for (uint32_t v : raw.left_feats) w.put<uint32_t>(v);
        w.vec(raw.bases);
        w.vec(raw.checks);
        w.vec(raw.costs);
    } else if (connector_kind == kRaw) {
        w.put<uint32_t>(kRaw);
        w.put<uint64_t>(raw.right_feats.size() / 8);
        for (uint32_t v : raw.right_feats) w.put<uint32_t>(v);
        w.put<uint64_t>(raw.left_feats.size() / 8);
        for (uint32_t v : raw.left_feats) w.put<uint32_t>(v);
        w.put<uint64_t>(raw.feat_T / 8);
        w.vec(raw.bases);
        w.vec(raw.checks);
        w.vec(raw.costs);
    } else {
        w.put<uint32_t>(kMatrix);
        w.vec(matrix.data);
        w.put<uint64_t>(matrix.num_right);
        w.put<uint64_t>(matrix.num_left);
    }
    w.put<uint8_t>(mapper ? 1 : 0);
    if (mapper) {
        w.vec(mapper->left);
        w.vec(mapper->right);
    }
    w.vec(char_prop.chr2inf);
    w.put<uint64_t>(char_prop.categories.size());
    for (auto& c : char_prop.categories) w.str(c);
    w.vec(unk.offsets);
    w.put<uint64_t>(unk.entries.size());
    for (auto& e : unk.entries) {
        w.put<uint16_t>(e.cate_id);
        w.put<uint16_t>(e.left_id);
        w.put<uint16_t>(e.right_id);
        w.put<int16_t>(e.word_cost);
        w.str(e.feature);
    }
}

// ---------------------------------------------------------------------------------------------
// zstd through dlopen (only libzstd.so.1 exists in this image; no zstd.h)
// ---------------------------------------------------------------------------------------------

std::vector<uint8_t> zstd_decompress_file(const char* path) {
    FILE* f = std::fopen(path, "rb");
    if (!f) throw Error(kIo, std::string("cannot open ") + path);
    std::vector<uint8_t> in;
    uint8_t buf[1 << 16];
    size_t k;
    while ((k = std::fread(buf, 1, sizeof(buf), f)) > 0) in.insert(in.end(), buf, buf + k);
    std::fclose(f);
    void* h = dlopen("libzstd.so.1", RTLD_NOW | RTLD_LOCAL);
    if (!h) throw Error(kIo, "libzstd.so.1 is not available: pass the decompressed stream to vbt_dict_from_bytes");
    struct Buf {
        const void* p;
        size_t size, pos;
    };
    struct OBuf {
        void* p;
        size_t size, pos;
    };
    using CreateFn = void* (*)();
    using FreeFn = size_t (*)(void*);
    using StepFn = size_t (*)(void*, OBuf*, Buf*);
    using IsErrFn = unsigned (*)(size_t);
    auto create = reinterpret_cast<CreateFn>(dlsym(h, "ZSTD_createDStream"));
    auto destroy = reinterpret_cast<FreeFn>(dlsym(h, "ZSTD_freeDStream"));
    auto step = reinterpret_cast<StepFn>(dlsym(h, "ZSTD_decompressStream"));
    auto is_err = reinterpret_cast<IsErrFn>(dlsym(h, "ZSTD_isError"));
    if (!create || !destroy || !step || !is_err) throw Error(kIo, "libzstd.so.1 lacks the streaming API");
    void* ds = create();
    std::vector<uint8_t> out;
    std::vector<uint8_t> chunk(1 << 20);
    Buf ib{in.data(), in.size(), 0};
    size_t rc = 1;
    while (ib.pos < ib.size || rc != 0) {
        OBuf ob{chunk.data(), chunk.size(), 0};
        size_t before = ib.pos;
        rc = step(ds, &ob, &ib);
        if (is_err(rc)) {
            destroy(ds);
            throw Error(kIo, "zstd: corrupt frame");
        }
        out.insert(out.end(), chunk.data(), chunk.data() + ob.pos);
        if (ib.pos == before && ob.pos == 0) break;
    }
    destroy(ds);
    return out;
}

void zstd_compress_to_file(const std::vector<uint8_t>& data, const char* path, int level) {
    void* h = dlopen("libzstd.so.1", RTLD_NOW | RTLD_LOCAL);
    if (!h) throw Error(kIo, "libzstd.so.1 is not available: write the stream of vbt_dict_write and compress it yourself");
    struct Buf {
        const void* p;
        size_t size, pos;
    };
    struct OBuf {
        void* p;
        size_t size, pos;
    };
    enum { kLevel = 100, kWorkers = 400, kEnd = 2 };  // ZSTD_c_compressionLevel, ZSTD_c_nbWorkers, ZSTD_e_end
    using CreateFn = void* (*)();
    using FreeFn = size_t (*)(void*);
    using SetParamFn = size_t (*)(void*, int, int);
    using PledgeFn = size_t (*)(void*, unsigned long long);
    using StepFn = size_t (*)(void*, OBuf*, Buf*, int);
    using IsErrFn = unsigned (*)(size_t);
    using ErrNameFn = const char* (*)(size_t);
    auto create = reinterpret_cast<CreateFn>(dlsym(h, "ZSTD_createCCtx"));
    auto destroy = reinterpret_cast<FreeFn>(dlsym(h, "ZSTD_freeCCtx"));
    auto set_param = reinterpret_cast<SetParamFn>(dlsym(h, "ZSTD_CCtx_setParameter"));
    auto pledge = reinterpret_cast<PledgeFn>(dlsym(h, "ZSTD_CCtx_setPledgedSrcSize"));
    auto step = reinterpret_cast<StepFn>(dlsym(h, "ZSTD_compressStream2"));
    auto is_err = reinterpret_cast<IsErrFn>(dlsym(h, "ZSTD_isError"));
    auto err_name = reinterpret_cast<ErrNameFn>(dlsym(h, "ZSTD_getErrorName"));
    if (!create || !destroy || !set_param || !pledge || !step || !is_err || !err_name)
        throw Error(kIo, "libzstd.so.1 lacks the streaming compression API");
    FILE* f = std::fopen(path, "wb");
    if (!f) throw Error(kIo, std::string("cannot create ") + path + ": " + std::strerror(errno));
    void* cs = create();
    // On any failure the partly written file is removed, so a failed write never leaves a truncated dictionary.
    auto fail = [&](const std::string& msg) {
        if (cs) destroy(cs);
        std::fclose(f);
        std::remove(path);
        throw Error(kIo, msg);
    };
    if (!cs) fail("zstd: cannot create a compression context");
    size_t rc = set_param(cs, kLevel, level);
    if (is_err(rc)) fail(std::string("zstd: compression level ") + std::to_string(level) + ": " + err_name(rc));
    // Worker threads only change how fast the frame is made, not what it decodes to; a libzstd built without them
    // refuses the parameter and compresses on this thread.  Each worker holds its own match tables (tens of MB at
    // the high levels), hence the cap.
    set_param(cs, kWorkers, int(std::min(std::thread::hardware_concurrency(), 16u)));
    rc = pledge(cs, data.size());  // the frame header then carries the content size
    if (is_err(rc)) fail(std::string("zstd: ") + err_name(rc));
    std::vector<uint8_t> chunk(1 << 20);
    Buf ib{data.data(), data.size(), 0};
    do {
        OBuf ob{chunk.data(), chunk.size(), 0};
        rc = step(cs, &ob, &ib, kEnd);
        if (is_err(rc)) fail(std::string("zstd: ") + err_name(rc));
        if (std::fwrite(chunk.data(), 1, ob.pos, f) != ob.pos) fail(std::string("cannot write ") + path + ": " + std::strerror(errno));
    } while (rc != 0);
    destroy(cs);
    cs = nullptr;
    if (std::fclose(f) != 0) {
        const std::string msg = std::string("cannot write ") + path + ": " + std::strerror(errno);
        std::remove(path);
        throw Error(kIo, msg);
    }
}

}  // namespace vbt
