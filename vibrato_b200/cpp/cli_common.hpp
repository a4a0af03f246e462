// Shared bits of the `tokenize` / `benchmark` look-alike CLIs.
#pragma once

#include <sys/stat.h>

#include <cstdio>
#include <fstream>
#include <iostream>
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

struct Packed {
    std::string utf8;
    std::vector<uint64_t> off{0};
    void add(const std::string& s) {
        utf8 += s;
        off.push_back(utf8.size());
    }
    uint64_t size() const { return off.size() - 1; }
    void clear() {
        utf8.clear();
        off.assign(1, 0);
    }
};

}  // namespace cli
