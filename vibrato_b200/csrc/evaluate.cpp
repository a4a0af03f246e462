// Accuracy harness: the library half of the reference's `evaluate` tool (evaluate/src/main.rs:61-138).
// The corpus is tokenised as ONE batch on the device; the set arithmetic over (char range, features) stays on
// the host because it compares feature strings.
#include "evaluate.hpp"

#include <algorithm>
#include <unordered_map>

namespace vbt {

namespace {

struct GoldToken {
    std::string_view surface, feature;
};

// One comparable key per token: char range + the chosen features (evaluate/src/main.rs:93-107)
std::string make_key(uint32_t start, uint32_t end, std::string_view feature, const std::vector<uint64_t>& indices) {
    std::string k;
    k.append(reinterpret_cast<const char*>(&start), 4).append(reinterpret_cast<const char*>(&end), 4);
    const std::vector<std::string> fields = parse_csv_row(feature);
    if (indices.empty()) {
        for (auto& f : fields) k.append(f).push_back('\x1f');
    } else {
        for (uint64_t i : indices) k.append(i < fields.size() ? fields[i] : std::string("*")).push_back('\x1f');
    }
    return k;
}

uint32_t count_chars(std::string_view s) {
    uint32_t n = 0;
    for (unsigned char c : s) n += (c & 0xC0) != 0x80;
    return n;
}

}  // namespace

EvalCounts evaluate(const Dictionary& d, Engine& e, std::string_view corpus, const std::vector<uint64_t>& feature_indices) {
    if (!utf8_valid(reinterpret_cast<const uint8_t*>(corpus.data()), corpus.size()))
        throw Error(kIo, "stream did not contain valid UTF-8");  // BufRead::lines() (corpus.rs:86-87)
    // Corpus::from_reader (trainer/corpus.rs:78-121)
    std::vector<std::vector<GoldToken>> examples;
    std::vector<GoldToken> tokens;
    size_t pos = 0;
    std::string_view line;
    while (next_line(corpus, pos, line)) {
        const size_t t1 = line.find('\t');
        if (t1 == std::string_view::npos) {
            if (line != "EOS")
                throw Error(kInvalidFormat, "rdr: Each line must be a pair of a surface and features or `EOS`");
            bool any = false;
            for (auto& t : tokens) any |= !t.surface.empty();
            if (any) examples.push_back(std::move(tokens));  // examples with an empty input are dropped (:105-108)
            tokens.clear();
            continue;
        }
        if (line.find('\t', t1 + 1) != std::string_view::npos)
            throw Error(kInvalidFormat, "rdr: Each line must be a pair of a surface and features or `EOS`");
        tokens.push_back({line.substr(0, t1), line.substr(t1 + 1)});
    }

    // the batch: one sentence per example = its surfaces concatenated (evaluate/src/main.rs:88-90)
    std::string utf8;
    std::vector<uint64_t> off{0};
    for (auto& ex : examples) {
        for (auto& t : ex) utf8.append(t.surface);
        off.push_back(utf8.size());
    }
    if (e.token_bytes() != 24) throw Error(kInvalidArgument, "evaluate needs full token records: switch compact_tokens off");
    HostResult* r = e.run_host(utf8.data(), off.data(), examples.size());
    struct Release {
        Engine& e;
        HostResult* r;
        ~Release() { e.release(r); }
    } guard{e, r};
    struct Tok {
        uint32_t start_char, end_char, start_byte, end_byte, word_idx;
        int32_t total_cost;
    };
    const bool post = r->out.has(kPostTokens);  // posterior decoding on: its paths are scored
    const Tok* toks = r->ptr<const Tok>(post ? kPostTokens : kTokens);
    const uint64_t* tok_off = r->ptr<const uint64_t>(post ? kPostOff : kTokOff);

    EvalCounts c{0, 0, 0};
    std::vector<std::string> refs, syss, both;
    for (size_t i = 0; i < examples.size(); ++i) {
        refs.clear();
        syss.clear();
        both.clear();
        uint32_t start = 0;
        for (auto& t : examples[i]) {
            const uint32_t len = count_chars(t.surface);
            refs.push_back(make_key(start, start + len, t.feature, feature_indices));
            start += len;
        }
        for (uint64_t k = tok_off[i]; k < tok_off[i + 1]; ++k)
            syss.push_back(make_key(toks[k].start_char, toks[k].end_char, d.word_feature(toks[k].word_idx), feature_indices));
        auto uniq = [](std::vector<std::string>& v) {  // HashSet semantics: duplicates count once
            std::sort(v.begin(), v.end());
            v.erase(std::unique(v.begin(), v.end()), v.end());
        };
        uniq(refs);
        uniq(syss);
        std::set_intersection(refs.begin(), refs.end(), syss.begin(), syss.end(), std::back_inserter(both));
        c.num_ref += refs.size();
        c.num_sys += syss.size();
        c.num_cor += both.size();
    }
    return c;
}

}  // namespace vbt
