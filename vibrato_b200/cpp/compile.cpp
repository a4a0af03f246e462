// `compile` look-alike: same flags, messages and output as the reference tool (/root/reference/compile/src/main.rs):
// MeCab-format sources in, a zstd-compressed system dictionary (`system.dic.zst`, level 19) out.  The dictionary is
// built before the output file is created, so a source error leaves no file behind.
#include <chrono>

#include "cli_common.hpp"

using namespace vibrato_b200;

static void usage() {
    std::fprintf(stderr,
                 "Usage: compile -l <lex.csv> -u <unk.def> -c <char.def> -o <system.dic.zst>\n"
                 "               [-m <matrix.def> | --bigram-right-in <bigram.right> --bigram-left-in <bigram.left>\n"
                 "                                  --bigram-cost-in <bigram.cost> [--dual-connector]]\n");
}

int main(int argc, char** argv) {
    std::string lexicon_in, matrix_in, unk_in, char_in, sysdic_out, bigram_right_in, bigram_left_in, bigram_cost_in;
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
        else if (a == "-m" || a == "--matrix-in") matrix_in = next();
        else if (a == "-u" || a == "--unk-in") unk_in = next();
        else if (a == "-c" || a == "--char-in") char_in = next();
        else if (a == "-o" || a == "--sysdic-out") sysdic_out = next();
        else if (a == "--bigram-right-in") bigram_right_in = next();
        else if (a == "--bigram-left-in") bigram_left_in = next();
        else if (a == "--bigram-cost-in") bigram_cost_in = next();
        else if (a == "--dual-connector") dual_connector = true;
        else {
            usage();
            return 2;
        }
    }
    if (lexicon_in.empty() || unk_in.empty() || char_in.empty() || sysdic_out.empty()) {
        usage();
        return 2;
    }
    const bool bigram = !bigram_right_in.empty() && !bigram_left_in.empty() && !bigram_cost_in.empty();
    if (matrix_in.empty() && !bigram) {  // main.rs:84-91, the reference's wording
        std::fprintf(stderr, "error: At least one of --matrin-in or --bigram-{right,left,cost}-in must be specified.\n\n");
        usage();
        return 2;
    }
    try {
        std::fprintf(stderr, "Compiling the system dictionary...\n");
        const auto start = std::chrono::steady_clock::now();
        const std::string lex = cli::slurp(lexicon_in), chr = cli::slurp(char_in), unk = cli::slurp(unk_in);
        Dictionary dict =
            !matrix_in.empty()
                ? Dictionary::from_readers(lex, cli::slurp(matrix_in), chr, unk)
                : Dictionary::from_readers_with_bigram_info(lex, cli::slurp(bigram_right_in), cli::slurp(bigram_left_in),
                                                            cli::slurp(bigram_cost_in), chr, unk, dual_connector);
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
