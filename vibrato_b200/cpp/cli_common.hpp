// Shared bits of the look-alike CLIs (`tokenize`, `benchmark`, `evaluate`, `compile`, `reorder`, `map`).
#pragma once

#include <sys/stat.h>

#include <charconv>
#include <cmath>
#include <cstdio>
#include <fstream>
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "vibrato_b200.hpp"

namespace cli {

inline std::string slurp(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error("cannot open " + path);
    std::ostringstream ss;
    ss << f.rdbuf();
    return ss.str();
}

// -i accepts what the reference accepts (a zstd-compressed `.dic`), plus — an extension for
// environments without released dictionaries — a directory holding lex.csv, matrix.def, char.def, unk.def.
inline vibrato_b200::Dictionary load_dictionary(const std::string& path) {
    struct stat st {};
    if (stat(path.c_str(), &st) == 0 && S_ISDIR(st.st_mode)) {
        std::string lex = slurp(path + "/lex.csv"), mat = slurp(path + "/matrix.def"), chr = slurp(path + "/char.def"),
                    unk = slurp(path + "/unk.def");
        return vibrato_b200::Dictionary::from_readers(lex, mat, chr, unk);
    }
    return vibrato_b200::Dictionary::read_zstd_file(path);
}

// BufRead::lines(): '\n'-separated, "\r\n" stripped; input must be valid UTF-8 (checked on the device).
inline bool read_line(std::istream& in, std::string& line) {
    if (!std::getline(in, line)) return false;
    if (!line.empty() && line.back() == '\r') line.pop_back();
    return true;
}

// --devices 0,1,..: the GPUs one tokenizer spreads every batch over (Tokenizer::devices); an empty list keeps the
// single-device tokenizer.
inline std::vector<int32_t> parse_devices(const std::string& list) {
    std::vector<int32_t> devices;
    for (size_t p = 0; p < list.size();) {
        size_t q = list.find(',', p);
        if (q == std::string::npos) q = list.size();
        devices.push_back(int32_t(std::stol(list.substr(p, q - p))));
        p = q + 1;
    }
    return devices;
}

// tokenize --boundary-marker C: removes every occurrence of the ASCII byte `marker` from `line` and returns the byte
// offsets, in the line without markers, where they stood: required token boundaries.  Adjacent markers give one
// boundary; markers at either end give 0 / the length, which constrain nothing.
inline std::vector<uint32_t> strip_boundary_markers(std::string& line, char marker) {
    std::vector<uint32_t> bnd;
    size_t w = 0;
    for (size_t r = 0; r < line.size(); ++r) {
        if (line[r] == marker) {
            if (bnd.empty() || bnd.back() != w) bnd.push_back(uint32_t(w));
        } else {
            line[w++] = line[r];
        }
    }
    line.resize(w);
    return bnd;
}

// tokenize -p: MeCab's partial-analysis input.  Lines up to a line that is exactly "EOS" form one sentence (lines
// after the last "EOS" one more).  A line with a TAB is a required token: its surface is the text before the first
// TAB, its feature pattern the rest.  Every line's start and end are required boundaries.
struct PartialSentence {
    std::string text;
    std::vector<uint32_t> bnd;
    std::vector<std::pair<std::pair<uint32_t, uint32_t>, std::string>> toks;  // {{start, end}, pattern}
    bool pending = false;  // lines since the last EOS
    // false for a line that starts with a TAB (an empty token)
    bool add_line(const std::string& line) {
        pending = true;
        const size_t tab = line.find('\t');
        if (tab == 0) return false;
        const uint32_t start = uint32_t(text.size());
        text.append(line, 0, tab);
        if (tab != std::string::npos) toks.push_back({{start, uint32_t(text.size())}, line.substr(tab + 1)});
        bnd.push_back(start);
        bnd.push_back(uint32_t(text.size()));
        return true;
    }
    void clear() {
        text.clear();
        bnd.clear();
        toks.clear();
        pending = false;
    }
};

struct Packed {
    std::string utf8;
    std::vector<uint64_t> off{0};
    std::vector<uint64_t> bnd_off{0};  // required boundaries per line (--boundary-marker), bnd_off / bnd as CSR
    std::vector<uint32_t> bnd;
    // required tokens per sentence (tokenize -p), span_off / spans as CSR; the batch's distinct patterns in pat / pat_off
    std::vector<uint64_t> span_off{0};
    std::vector<vbt_span> spans;
    std::string pat;
    std::vector<uint64_t> pat_off{0};
    std::map<std::string, uint32_t> pat_idx;
    void add(const std::string& s) {
        utf8 += s;
        off.push_back(utf8.size());
        bnd_off.push_back(bnd.size());
        span_off.push_back(spans.size());
    }
    // A span of the sentence about to be added; an empty pattern or "*" matches any feature.
    void add_span(uint32_t start, uint32_t end, const std::string& pattern) {
        uint32_t k = VBT_SPAN_ANY;
        if (!pattern.empty() && pattern != "*") {
            auto it = pat_idx.find(pattern);
            if (it == pat_idx.end()) {
                it = pat_idx.emplace(pattern, uint32_t(pat_off.size() - 1)).first;
                pat += pattern;
                pat_off.push_back(pat.size());
            }
            k = it->second;
        }
        spans.push_back(vbt_span{start, end, k});
    }
    void add(const std::string& s, const std::vector<uint32_t>& b) {
        bnd.insert(bnd.end(), b.begin(), b.end());
        add(s);
    }
    uint64_t size() const { return off.size() - 1; }
    void clear() {
        utf8.clear();
        off.assign(1, 0);
        bnd_off.assign(1, 0);
        bnd.clear();
        span_off.assign(1, 0);
        spans.clear();
        pat.clear();
        pat_off.assign(1, 0);
        pat_idx.clear();
    }
};

// Rust's `{}` for f64: shortest digits that round-trip, never an exponent, "NaN" / "inf"
inline std::string rust_f64(double v) {
    if (std::isnan(v)) return "NaN";
    if (std::isinf(v)) return v < 0 ? "-inf" : "inf";
    char buf[512];
    auto r = std::to_chars(buf, buf + sizeof(buf), v, std::chars_format::fixed);
    return std::string(buf, r.ptr);
}

// A `.lmap` / `.rmap` file of `reorder`: `{id}\t{p}\n` per id (map/src/reorder.rs:50-52)
inline std::string mapping_text(const vibrato_b200::ConnIdProbs& probs) {
    std::string text;
    for (const auto& [id, p] : probs) text.append(std::to_string(id)).append("\t").append(rust_f64(p)).append("\n");
    return text;
}

// Rust's `{:?}` for a path: quoted, with `\`, `"` and control characters escaped (char::escape_debug)
inline std::string rust_debug_path(const std::string& path) {
    std::string out = "\"";
    for (unsigned char c : path) {
        if (c == '\\' || c == '"') out += '\\', out += char(c);
        else if (c == '\t') out += "\\t";
        else if (c == '\r') out += "\\r";
        else if (c == '\n') out += "\\n";
        else if (c == 0) out += "\\0";
        else if (c < 0x20 || c == 0x7F) {
            char b[16];
            std::snprintf(b, sizeof(b), "\\u{%x}", c);
            out += b;
        } else out += char(c);
    }
    return out + "\"";
}

// PathBuf::set_extension: the extension of the last component is replaced, or added when it has none (".hidden" has
// none).  A path without a last file name ("", "/", ".", "..", "a/..") stays as it is.  Like Rust, everything after
// the file stem goes, trailing "/" and "/." included.
inline std::string set_extension(const std::string& path, const std::string& ext) {
    size_t end = path.size();
    for (;;) {  // Path::components() drops trailing separators and "." components
        while (end > 1 && path[end - 1] == '/') --end;
        if (end > 1 && path[end - 1] == '.' && path[end - 2] == '/') end -= 2;
        else break;
    }
    size_t start = path.rfind('/', end ? end - 1 : 0);
    start = (start == std::string::npos || end == 0) ? 0 : start + 1;
    if (end > 0 && start == end) return path;  // the root
    const std::string name = path.substr(start, end - start);
    if (name.empty() || name == "." || name == "..") return path;
    const size_t dot = name.rfind('.');
    const size_t stem = (dot == std::string::npos || dot == 0) ? name.size() : dot;
    return path.substr(0, start + stem) + "." + ext;
}

// u16::from_str: an optional '+', then ASCII digits only, at most 65535 (no sign, space or empty string)
inline uint16_t parse_u16(std::string_view s) {
    if (s.empty()) throw std::runtime_error("cannot parse integer from empty string");
    if (s[0] == '+' && s.size() > 1) s.remove_prefix(1);
    uint32_t v = 0;
    for (char c : s) {
        if (c < '0' || c > '9') throw std::runtime_error("invalid digit found in string");
        v = v * 10 + uint32_t(c - '0');
        if (v > 0xFFFF) throw std::runtime_error("number too large to fit in target type");
    }
    return uint16_t(v);
}

}  // namespace cli
