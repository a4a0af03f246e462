// `mecab_smalldic` look-alike: same flags, messages and output as the reference's example tool
// (examples/mecab_smalldic/src/main.rs).  Converts a trained MeCab model to bigram.* files
// (mecab::generate_bigram_info), builds a Raw or Dual connector dictionary from them and writes it in zstd (level 19).
// Runs on the host only.  The dictionary is built before the output file is created, so an error leaves no file.
#include <cctype>
#include <chrono>
#include <cstdlib>

#include "cli_common.hpp"

using namespace vibrato_b200;

static void usage() {
    std::fprintf(stderr,
                 "Usage: mecab_smalldic -l <lex.csv> -u <unk.def> -c <char.def> -f <feature.def> -a <right-id.def>\n"
                 "                      -b <left-id.def> -m <model.def> -r <cost-factor> [--dual-connector]\n"
                 "                      -o <system.dic.zst>\n");
}

// The subset of f64::from_str that a cost factor needs: no leading space, no hexadecimal form
static bool parse_f64(const std::string& s, double& v) {
    if (s.empty() || std::isspace(static_cast<unsigned char>(s[0])) || s.find_first_of("xX(") != std::string::npos)
        return false;
    char* end = nullptr;
    v = std::strtod(s.c_str(), &end);
    return end == s.c_str() + s.size();
}

int main(int argc, char** argv) {
    std::string lexicon_in, unk_in, char_in, feature_in, right_id_in, left_id_in, model_in, cost_factor_in, sysdic_out;
    bool dual_connector = false;
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        auto next = [&]() -> std::string {
            if (i + 1 >= argc) {
                usage();
                std::exit(2);
            }
            return argv[++i];
        };
        if (a == "-l" || a == "--lexicon-in") lexicon_in = next();
        else if (a == "-u" || a == "--unk-in") unk_in = next();
        else if (a == "-c" || a == "--char-in") char_in = next();
        else if (a == "-f" || a == "--feature-in") feature_in = next();
        else if (a == "-a" || a == "--right-id-in") right_id_in = next();
        else if (a == "-b" || a == "--left-id-in") left_id_in = next();
        else if (a == "-m" || a == "--text-model-in") model_in = next();
        else if (a == "-r" || a == "--cost-factor") cost_factor_in = next();
        else if (a == "--dual-connector") dual_connector = true;
        else if (a == "-o" || a == "--sysdic-out") sysdic_out = next();
        else {
            usage();
            return 2;
        }
    }
    double cost_factor = 0;
    if (lexicon_in.empty() || unk_in.empty() || char_in.empty() || feature_in.empty() || right_id_in.empty() ||
        left_id_in.empty() || model_in.empty() || sysdic_out.empty() || !parse_f64(cost_factor_in, cost_factor)) {
        usage();
        return 2;
    }
    try {
        std::fprintf(stderr, "Compiling the system dictionary...\n");
        const auto start = std::chrono::steady_clock::now();
        const mecab::BigramInfo bi = mecab::generate_bigram_info(cli::slurp(feature_in), cli::slurp(right_id_in),
                                                                 cli::slurp(left_id_in), cli::slurp(model_in), cost_factor);
        Dictionary dict = Dictionary::from_readers_with_bigram_info(cli::slurp(lexicon_in), bi.right, bi.left, bi.cost,
                                                                    cli::slurp(char_in), cli::slurp(unk_in), dual_connector);
        const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - start).count();
        std::fprintf(stderr, "%s seconds\n", cli::rust_f64(secs).c_str());
        std::fprintf(stderr, "Writing the system dictionary in zstd...: %s\n", cli::rust_debug_path(sysdic_out).c_str());
        dict.write_zstd_file(sysdic_out, 19);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "Error: %s\n", e.what());
        return 1;
    }
    return 0;
}
