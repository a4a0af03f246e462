// mecab::generate_bigram_info (mecab.rs:31-181): the bigram.right / bigram.left / bigram.cost files of a compact
// (Raw or Dual connector) dictionary, made from a trained MeCab model.  Exact text processing, no training: the
// bigram half of FeatureExtractor (trainer/feature_extractor.rs:39-147, 154-195, 217-249) names each connection
// id's features, and model.def's weights become integer costs.
#include <charconv>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "host_dict.hpp"

namespace vbt {

namespace {

// char::is_whitespace (the Unicode White_Space property), which str::trim uses
bool is_unicode_space(char32_t c) {
    return (c >= 0x09 && c <= 0x0D) || c == 0x20 || c == 0x85 || c == 0xA0 || c == 0x1680 || (c >= 0x2000 && c <= 0x200A) ||
           c == 0x2028 || c == 0x2029 || c == 0x202F || c == 0x205F || c == 0x3000;
}

// str::trim on valid UTF-8
std::string_view trim(std::string_view s) {
    auto lead_len = [](unsigned char b) { return b < 0x80 ? 1 : b < 0xE0 ? 2 : b < 0xF0 ? 3 : 4; };
    auto decode = [](std::string_view s, size_t i, size_t n) {
        if (n == 1) return char32_t(uint8_t(s[i]));
        char32_t c = uint8_t(s[i]) & (0xFF >> (n + 1));
        for (size_t k = 1; k < n; ++k) c = (c << 6) | (uint8_t(s[i + k]) & 0x3F);
        return c;
    };
    while (!s.empty()) {
        const size_t n = lead_len(uint8_t(s[0]));
        if (!is_unicode_space(decode(s, 0, n))) break;
        s.remove_prefix(n);
    }
    while (!s.empty()) {
        size_t i = s.size() - 1;
        while (i > 0 && (uint8_t(s[i]) & 0xC0) == 0x80) --i;
        if (!is_unicode_space(decode(s, i, s.size() - i))) break;
        s.remove_suffix(s.size() - i);
    }
    return s;
}

// BufRead::lines() over one file: a line that is not UTF-8 fails the read as an I/O error
struct Lines {
    std::string_view text;
    size_t pos = 0;
    bool next(std::string_view& line) {
        if (!next_line(text, pos, line)) return false;
        if (!utf8_valid(reinterpret_cast<const uint8_t*>(line.data()), line.size()))
            throw Error(kIo, "stream did not contain valid UTF-8");
        return true;
    }
};

bool is_digit(char c) { return c >= '0' && c <= '9'; }

// A run of ASCII digits as usize::from_str reads it
uint64_t parse_usize(std::string_view digits) {
    uint64_t v = 0;
    for (char c : digits) {
        if (v > (UINT64_MAX - uint64_t(c - '0')) / 10) throw Error(kParseInt, "number too large to fit in target type");
        v = v * 10 + uint64_t(c - '0');
    }
    return v;
}

// One bigram template of one side: the placeholders `%X[i]` / `%X?[i]` (X = L or R) and the text between them
// (feature_extractor.rs:79-134).
struct Template {
    struct Capture {
        size_t begin, end;
        uint64_t idx;
    };
    std::string raw;
    std::vector<uint64_t> required;  // the `?` indices
    std::vector<Capture> captures;

    // Regex `%(X|X\?)\[([0-9]+)\]`: leftmost, non-overlapping matches
    Template(std::string_view t, char x) : raw(t) {
        for (size_t i = 0; i < raw.size();) {
            size_t p = i;
            bool ok = raw[p] == '%' && p + 1 < raw.size() && raw[p + 1] == x;
            bool req = false;
            if (ok) {
                p += 2;
                if (p < raw.size() && raw[p] == '?') req = true, ++p;
                ok = p < raw.size() && raw[p] == '[';
            }
            size_t d = p + 1, e = d;
            if (ok) {
                while (e < raw.size() && is_digit(raw[e])) ++e;
                ok = e > d && e < raw.size() && raw[e] == ']';
            }
            if (!ok) {
                ++i;
                continue;
            }
            const uint64_t idx = parse_usize(std::string_view(raw).substr(d, e - d));
            if (req) required.push_back(idx);
            captures.push_back({i, e + 1, idx});
            i = e + 1;
        }
    }
};

// One side's templates and its feature-id map, shared by all of them (FeatureExtractor::extract_feature_ids).
struct Side {
    std::vector<Template> templates;
    std::unordered_map<std::string, uint32_t> ids;
    uint32_t next_id = 1;

    // Feature ids of one connection id's CSV fields, 0 for None
    std::vector<uint32_t> extract(const std::vector<std::string>& features) {
        static const std::string kStar = "*";
        auto field = [&](uint64_t i) -> const std::string& { return i < features.size() ? features[i] : kStar; };
        std::vector<uint32_t> out;
        std::string s;
        for (const Template& t : templates) {
            bool none = false;
            for (uint64_t i : t.required) none = none || field(i) == "*";
            if (none) {
                out.push_back(0);
                continue;
            }
            s.clear();
            size_t start = 0;
            for (const auto& c : t.captures) {
                s.append(t.raw, start, c.begin - start).append(field(c.idx));
                start = c.end;
            }
            s.append(t.raw, start, std::string::npos);
            auto [it, fresh] = ids.try_emplace(s, next_id);
            if (fresh) ++next_id;
            out.push_back(it->second);
        }
        return out;
    }
};

// TrainerConfig::parse_feature_config (trainer/config.rs:64-101); UNIGRAM templates are read and left unused.
void parse_feature_def(std::string_view text, Side& left, Side& right) {
    Lines lines{text};
    std::string_view line;
    while (lines.next(line)) {
        line = trim(line);
        if (line.empty() || line[0] == '#') continue;
        if (line.substr(0, 8) == "UNIGRAM ") {
            Template(line.substr(8), 'F');  // the index must still parse (feature_extractor.rs:57)
        } else if (line.substr(0, 7) == "BIGRAM ") {
            const std::string_view t = line.substr(7);
            const size_t slash = t.find('/');
            if (slash == std::string_view::npos || t.find('/', slash + 1) != std::string_view::npos)
                throw Error(kInvalidFormat, "feature.def: Invalid bigram template");
            left.templates.emplace_back(t.substr(0, slash), 'L');
            right.templates.emplace_back(t.substr(slash + 1), 'R');
        } else {
            throw Error(kInvalidFormat, "feature: ");
        }
    }
}

// One id-def file (mecab.rs:53-98): lines `^([0-9]+) (.*)$`, the features of id 0 must start with BOS/EOS, and a
// repeated id replaces the earlier one.
std::unordered_map<uint64_t, std::vector<uint32_t>> read_id_def(std::string_view text, Side& side, const char* name) {
    std::unordered_map<uint64_t, std::vector<uint32_t>> out;
    Lines lines{text};
    std::string_view line;
    while (lines.next(line)) {
        size_t e = 0;
        while (e < line.size() && is_digit(line[e])) ++e;
        if (e == 0 || e == line.size() || line[e] != ' ')
            throw Error(kInvalidFormat, std::string(name) + ": each line must be a pair of an ID and features");
        const uint64_t id = parse_usize(line.substr(0, e));
        const std::vector<std::string> features = parse_csv_row(line.substr(e + 1));
        if (id == 0 && !features.empty() && features[0] != "BOS/EOS")
            throw Error(kInvalidFormat, std::string(name) + ": ID 0 must be BOS/EOS");
        out[id] = side.extract(features);
    }
    return out;
}

// f64::from_str on what `[0-9\-\.]+` admits: an optional '-', then digits with at most one '.', at least one digit
bool parse_weight(std::string_view s, double& w) {
    size_t i = s[0] == '-' ? 1 : 0, digits = 0, dots = 0;
    for (size_t k = i; k < s.size(); ++k) {
        if (s[k] == '.') ++dots;
        else if (is_digit(s[k])) ++digits;
        else return false;
    }
    if (digits == 0 || dots > 1) return false;
    w = std::strtod(std::string(s).c_str(), nullptr);  // correctly rounded, as Rust's; overflow gives +-inf as Rust does
    return true;
}

// `-(weight * cost_factor) as i32`: the negation comes first, then the cast, which truncates toward zero, saturates
// at the i32 bounds and maps NaN to 0
int32_t to_cost(double weight, double cost_factor) {
    const double x = -(weight * cost_factor);
    if (std::isnan(x)) return 0;
    if (x <= -2147483648.0) return INT32_MIN;
    if (x >= 2147483647.0) return INT32_MAX;
    return int32_t(x);
}

void append_int(std::string& out, uint64_t v) {
    char buf[24];
    auto r = std::to_chars(buf, buf + sizeof(buf), v);
    out.append(buf, r.ptr);
}

// `{id}\t{f1},{f2},..` for ids 1..features.len() (mecab.rs:134-178): a hole is an error, and without an id 0 the
// highest id is not written
std::string write_features(const std::unordered_map<uint64_t, std::vector<uint32_t>>& features, const char* name) {
    std::string out;
    for (uint64_t id = 1; id < features.size(); ++id) {
        auto it = features.find(id);
        if (it == features.end())
            throw Error(kInvalidFormat, std::string(name) + ": feature ID " + std::to_string(id) + " is undefined");
        append_int(out, id);
        out += '\t';
        for (size_t i = 0; i < it->second.size(); ++i) {
            if (i) out += ',';
            if (it->second[i]) append_int(out, it->second[i]);
            else out += '*';
        }
        out += '\n';
    }
    return out;
}

}  // namespace

BigramInfoText generate_bigram_info(std::string_view feature_def, std::string_view right_id_def,
                                    std::string_view left_id_def, std::string_view model_def, double cost_factor) {
    // right-id.def holds the right-hand ids of the left context, so its features are the *left* features, and
    // left-id.def's the right ones (mecab.rs:49-51)
    Side left, right;
    parse_feature_def(feature_def, left, right);
    const auto left_features = read_id_def(right_id_def, left, "right_id_def_rdr");
    const auto right_features = read_id_def(left_id_def, right, "left_id_def_rdr");

    BigramInfoText out;
    Lines lines{model_def};
    std::string_view line;
    std::string feature;
    while (lines.next(line)) {  // mecab.rs:100-132
        size_t e = 0;
        while (e < line.size() && (is_digit(line[e]) || line[e] == '-' || line[e] == '.')) ++e;
        if (e == 0 || e == line.size() || line[e] != '\t') continue;  // not `^([0-9\-\.]+)\t(.*)$`: header lines
        double weight;
        if (!parse_weight(line.substr(0, e), weight)) throw Error(kParseFloat, "invalid float literal");
        const int32_t cost = to_cost(weight, cost_factor);
        if (cost == 0) continue;
        // .replace("BOS/EOS", "") and the first two pieces of .split('/')
        feature.clear();
        const std::string_view rest = line.substr(e + 1);
        for (size_t p = 0;;) {
            const size_t q = rest.find("BOS/EOS", p);
            feature.append(rest.substr(p, q == std::string_view::npos ? std::string_view::npos : q - p));
            if (q == std::string_view::npos) break;
            p = q + 7;
        }
        const size_t slash = feature.find('/');
        if (slash == std::string::npos) continue;
        const size_t end = feature.find('/', slash + 1);
        const std::string_view fs(feature);
        const std::string_view lf = fs.substr(0, slash), rf = fs.substr(slash + 1, end == std::string::npos ? end : end - slash - 1);
        uint32_t lid = 0, rid = 0;
        if (!lf.empty()) {
            auto it = left.ids.find(std::string(lf));
            if (it == left.ids.end()) continue;
            lid = it->second;
        }
        if (!rf.empty()) {
            auto it = right.ids.find(std::string(rf));
            if (it == right.ids.end()) continue;
            rid = it->second;
        }
        if (lid) append_int(out.cost, lid);
        out.cost += '/';
        if (rid) append_int(out.cost, rid);
        out.cost += '\t';
        out.cost += std::to_string(cost);
        out.cost += '\n';
    }
    out.right = write_features(left_features, "right_id_def_rdr");
    out.left = write_features(right_features, "left_id_def_rdr");
    return out;
}

}  // namespace vbt
