// `evaluate` look-alike: same flags and output as the reference tool (/root/reference/evaluate/src/main.rs:13-38
// flags, :61-138 loop, :132-136 output), with the whole test corpus tokenised as one batch on the GPU.
#include <cmath>
#include <cstring>

#include "cli_common.hpp"

using namespace vibrato_b200;
using cli::rust_f64;

static void usage() {
    std::fprintf(stderr,
                 "evaluate -t <test corpus> -i <system.dic.zst | mecab-source-dir> [-u user.csv] [-M n]\n"
                 "         [--feature-indices i,j,...]\n"
                 "         [--theta F --posterior G]   (score each sentence's posterior-decoded path, from the marginals\n"
                 "                                      at temperature F > 0 with weight G >= 0, in place of the best path)\n");
}

int main(int argc, char** argv) {
    std::string test_in, sysdic, userlex;
    size_t max_grouping_len = 0;
    std::vector<uint64_t> feature_indices;
    double theta = 0, gamma = 0;
    bool has_theta = false, has_gamma = false;
    auto number = [](const std::string& v, double& out) {  // a finite number, else a usage error
        char* end = nullptr;
        out = std::strtod(v.c_str(), &end);
        return !v.empty() && !*end && std::isfinite(out);
    };
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        auto next = [&]() -> std::string {
            if (i + 1 >= argc) {
                usage();
                std::exit(2);
            }
            return argv[++i];
        };
        if (a == "-t" || a == "--test-in") test_in = next();
        else if (a == "-i" || a == "--sysdic-in") sysdic = next();
        else if (a == "-u" || a == "--userlex-csv-in") userlex = next();
        else if (a == "-M" || a == "--max-grouping-len") max_grouping_len = std::stoull(next());
        else if (a == "--theta" || a == "--posterior") {
            double& v = a == "--theta" ? theta : gamma;
            if (!number(next(), v) || (a == "--theta" ? !(v > 0) : !(v >= 0))) {
                usage();
                return 2;
            }
            (a == "--theta" ? has_theta : has_gamma) = true;
        } else if (a == "--feature-indices") {
            std::stringstream ss(next());
            std::string item;
            while (std::getline(ss, item, ',')) feature_indices.push_back(std::stoull(item));
        } else {
            usage();
            return 2;
        }
    }
    if (test_in.empty() || sysdic.empty() || has_theta != has_gamma) {
        usage();
        return 2;
    }
    try {
        std::fprintf(stderr, "Loading the dictionary...\n");
        Dictionary dict = cli::load_dictionary(sysdic);
        if (!userlex.empty()) {
            std::string csv = cli::slurp(userlex);
            dict = std::move(dict).reset_user_lexicon_from_reader(&csv);
        }
        Tokenizer tokenizer = Tokenizer(std::move(dict)).max_grouping_len(max_grouping_len);  // main.rs:72
        if (has_gamma) {
            tokenizer.marginals(theta);
            tokenizer.posterior(true, gamma);
        }
        std::fprintf(stderr, "Tokenizing...\n");
        const std::string corpus = cli::slurp(test_in);
        const Tokenizer::EvalCounts c = tokenizer.evaluate(corpus, feature_indices);
        const double precision = double(c.num_cor) / double(c.num_sys);  // main.rs:129-131
        const double recall = double(c.num_cor) / double(c.num_ref);
        const double f1 = 2.0 * precision * recall / (precision + recall);
        std::printf("Precision = %s\nRecall = %s\nF1 = %s\n", rust_f64(precision).c_str(), rust_f64(recall).c_str(),
                    rust_f64(f1).c_str());
    } catch (const std::exception& e) {
        std::fprintf(stderr, "Error: %s\n", e.what());
        return 1;
    }
    return 0;
}
