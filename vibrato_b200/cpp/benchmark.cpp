// `benchmark` look-alike: the reference's measurement protocol (/root/reference/benchmark/src/main.rs:
// all stdin lines pre-loaded :47-51; RUNS=10 timed passes per trial :14,:53-65; one warm-up trial
// :69-72; TRIALS=10, fastest and slowest pass of each trial dropped :76-84; prints
// Number_of_sentences and [min,avg,max] seconds :90-91) with the inner per-line loop replaced by one
// batched GPU call per pass (host buffers in, host tokens out — the e2e path).
#include <algorithm>
#include <chrono>
#include <numeric>

#include "cli_common.hpp"

using namespace vibrato_b200;

namespace {
constexpr int kRuns = 10, kTrials = 10;

struct PassTimes {
    std::vector<double> secs;
    void drop_fastest() { secs.erase(std::min_element(secs.begin(), secs.end())); }
    void drop_slowest() { secs.erase(std::max_element(secs.begin(), secs.end())); }
    double lo() const { return *std::min_element(secs.begin(), secs.end()); }
    double hi() const { return *std::max_element(secs.begin(), secs.end()); }
    double mean() const { return std::accumulate(secs.begin(), secs.end(), 0.0) / double(secs.size()); }
};
}  // namespace

int main(int argc, char** argv) {
    std::string sysdic;
    bool ignore_space = false;
    size_t max_grouping_len = 0;
    std::vector<int32_t> devices;  // extension: --devices 0,1,2,3 = one tokenizer over several GPUs
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        if ((a == "-i" || a == "--sysdic") && i + 1 < argc) sysdic = argv[++i];
        else if (a == "--devices" && i + 1 < argc) devices = cli::parse_devices(argv[++i]);
        else if (a == "-S" || a == "--ignore-space") ignore_space = true;
        else if ((a == "-M" || a == "--max-grouping-len") && i + 1 < argc) max_grouping_len = std::stoull(argv[++i]);
        else {
            std::fprintf(stderr, "benchmark -i <system.dic.zst | mecab-source-dir> [-S] [-M n] [--devices 0,1,..] < corpus.txt\n");
            return 2;
        }
    }
    if (sysdic.empty()) {
        std::fprintf(stderr, "benchmark -i <system.dic.zst | mecab-source-dir> [-S] [-M n] [--devices 0,1,..] < corpus.txt\n");
        return 2;
    }
    try {
        Dictionary dict = cli::load_dictionary(sysdic);
        Tokenizer tokenizer =
            Tokenizer(std::move(dict)).ignore_space(ignore_space).max_grouping_len(max_grouping_len).devices(devices);
        cli::Packed pk;
        std::string line;
        while (cli::read_line(std::cin, line)) pk.add(line);
        auto trial = [&](PassTimes& t) {
            uint64_t n_words = 0;
            for (int r = 0; r < kRuns; ++r) {
                auto t0 = std::chrono::steady_clock::now();
                BatchResult res = tokenizer.tokenize_batch(pk.utf8.data(), pk.off.data(), pk.size());
                n_words += res.n_tokens();
                t.secs.push_back(std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
            }
            std::fprintf(stderr, "[benchmark.cpp] n_words = %llu\n", (unsigned long long)n_words);
        };
        PassTimes warm;
        trial(warm);
        std::printf("Warmup: %.17g\n", warm.mean());
        double lo = 0, avg = 0, hi = 0;
        for (int k = 0; k < kTrials; ++k) {
            PassTimes t;
            trial(t);
            t.drop_fastest();
            t.drop_slowest();
            lo += t.lo();
            avg += t.mean();
            hi += t.hi();
        }
        std::printf("Number_of_sentences: %llu\n", (unsigned long long)pk.size());
        std::printf("Elapsed_seconds_to_tokenize_all_sentences: [%.17g,%.17g,%.17g]\n", lo / kTrials, avg / kTrials,
                    hi / kTrials);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "Error: %s\n", e.what());
        return 1;
    }
    return 0;
}
