// `tokenize` look-alike: same flags and byte-identical output as the reference CLI
// (/root/reference/tokenize/src/main.rs:31-53 flags, :83-127 formats), tokenising on the GPU.
// Lines are shipped in batches; output order and content equal the per-line loop of main.rs:78-128.
#include <unistd.h>

#include <cerrno>
#include <cstdint>
#include <cstdlib>
#include <cmath>
#include <cstring>

#include "cli_common.hpp"

using namespace vibrato_b200;

static void usage() {
    std::fprintf(stderr,
                 "tokenize -i <system.dic.zst | mecab-source-dir> [-u user.csv] [-O mecab|wakati|detail] [-S] [-M n]\n"
                 "         [-F|--node-format FMT] [--unk-format FMT] [--bos-format FMT] [--eos-format FMT]\n"
                 "                                     (MeCab-style formats, built on the device; -F takes precedence over -O;\n"
                 "                                      unk defaults to the node format, bos to \"\", eos to \"EOS\\n\")\n"
                 "         [--format-on device|host]   (where the output text is built; default device; -F needs device)\n"
                 "         [--devices 0,1,..]          (spread every batch over these GPUs)\n"
                 "         [--batch-lines N]           (lines per batch when stdin is not a terminal; default 65536)\n"
                 "         [--boundary-marker C]       (an ASCII byte other than newline: removed from every line, it\n"
                 "                                      marks a required token boundary where it stood)\n"
                 "         [-p|--partial]              (MeCab's partial-analysis input: lines up to a line \"EOS\" form a\n"
                 "                                      sentence; a line `surface\\tpattern` is one token of a feature\n"
                 "                                      matching the pattern (\"*\" or nothing: any); every line starts\n"
                 "                                      and ends a token; not with --boundary-marker)\n"
                 "         [-m|--marginal -t|--theta F] (marginal probabilities at temperature F > 0: -F may print\n"
                 "                                      each token's with %%pP; -O output is unchanged)\n"
                 "         [-a|--all-morphs]           (every lattice node in place of the tokens, like MeCab -a: -O and\n"
                 "                                      -F render nodes, -F may print %%pb; needs --format-on device)\n"
                 "         [--cost-margin D]           (with -a: only the nodes of paths whose cost is within D, 0..2^62,\n"
                 "                                      of the best path's, plus the best path)\n"
                 "         [--sample N -t|--theta F [--seed S]]\n"
                 "                                     (N segmentations per line, 1..1024, drawn from the lattice's path\n"
                 "                                      distribution at temperature F, in place of the best path: -O and -F\n"
                 "                                      print N renderings per line; S (u64, default 0) keys the draws,\n"
                 "                                      which do not depend on --batch-lines or --devices; not with -a,\n"
                 "                                      %%pP or %%pb; needs --format-on device)\n"
                 "         [--posterior G]             (with -m -t F: each line's posterior-decoded path at weight G >= 0\n"
                 "                                      in place of the best path: -O and -F render it, %%pP prints its\n"
                 "                                      tokens' marginals; not with -a or --sample; needs --format-on device)\n");
}

int main(int argc, char** argv) {
    std::string sysdic, userlex, mode = "mecab", format_on = "device";
    bool ignore_space = false;
    size_t max_grouping_len = 0, batch_lines_arg = 65536;
    std::vector<int32_t> devices;
    std::string node_format, unk_format, bos_format, eos_format;
    bool has_node = false, has_unk = false, has_bos = false, has_eos = false;
    std::string marker;
    bool partial = false;
    bool marginal = false, has_theta = false, all_morphs = false;
    double theta = 0;
    uint32_t n_sample = 0;  // --sample
    uint64_t seed = 0;
    bool has_seed = false;
    int64_t cost_margin = -1;  // --cost-margin, -1 = every node
    double gamma = 0;          // --posterior
    bool posterior = false;
    // a whole decimal number in [lo, hi], else a usage error
    auto parse_u64 = [](const std::string& v, uint64_t lo, uint64_t hi, uint64_t& out) {
        if (v.empty() || v.size() > 20 || v.find_first_not_of("0123456789") != std::string::npos) return false;
        errno = 0;
        const unsigned long long x = std::strtoull(v.c_str(), nullptr, 10);
        if (errno == ERANGE || x < lo || x > hi) return false;
        out = x;
        return true;
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
        if (a == "-i" || a == "--sysdic") sysdic = next();
        else if (a == "-u" || a == "--userlex-csv") userlex = next();
        else if (a == "-O" || a == "--output-mode") mode = next();
        else if (a == "--format-on") format_on = next();
        else if (a == "-S" || a == "--ignore-space") ignore_space = true;
        else if (a == "-M" || a == "--max-grouping-len") max_grouping_len = std::stoull(next());
        else if (a == "--devices") devices = cli::parse_devices(next());
        else if (a == "--batch-lines") batch_lines_arg = std::stoull(next());
        else if (a == "-F" || a == "--node-format") node_format = next(), has_node = true;
        else if (a == "--unk-format") unk_format = next(), has_unk = true;
        else if (a == "--bos-format") bos_format = next(), has_bos = true;
        else if (a == "--eos-format") eos_format = next(), has_eos = true;
        else if (a == "--boundary-marker") marker = next();
        else if (a == "-p" || a == "--partial") partial = true;
        else if (a == "-m" || a == "--marginal") marginal = true;
        else if (a == "-a" || a == "--all-morphs") all_morphs = true;
        else if (a == "--sample" || a == "--seed") {
            uint64_t v = 0;
            if (!parse_u64(next(), a == "--sample" ? 1 : 0, a == "--sample" ? 1024 : UINT64_MAX, v)) {
                usage();
                return 2;
            }
            if (a == "--sample") n_sample = uint32_t(v);
            else seed = v, has_seed = true;
        }
        else if (a == "--cost-margin") {
            uint64_t v = 0;
            if (!parse_u64(next(), 0, uint64_t(1) << 62, v)) {
                usage();
                return 2;
            }
            cost_margin = int64_t(v);
        }
        else if (a == "--posterior") {
            const std::string v = next();
            char* end = nullptr;
            gamma = std::strtod(v.c_str(), &end);
            if (v.empty() || *end || !(gamma >= 0) || !std::isfinite(gamma)) {
                usage();
                return 2;
            }
            posterior = true;
        }
        else if (a == "-t" || a == "--theta") {
            const std::string v = next();
            char* end = nullptr;
            theta = std::strtod(v.c_str(), &end);
            if (v.empty() || *end) {
                usage();
                return 2;
            }
            has_theta = true;
        }
        else {
            usage();
            return 2;
        }
    }
    // the formats are rendered by the device only; --unk/bos/eos-format complete -F
    const bool bounded = !marker.empty();
    // -m and --sample need --theta, and --theta belongs to them; --seed belongs to --sample
    const bool sample = n_sample != 0;
    if (batch_lines_arg == 0 || (has_node && format_on == "host") || (!has_node && (has_unk || has_bos || has_eos)) ||
        (marginal || sample) != has_theta || (all_morphs && format_on == "host") || (has_seed && !sample) ||
        (sample && (all_morphs || format_on == "host")) || (cost_margin >= 0 && !all_morphs) ||
        (posterior && (!marginal || all_morphs || sample || format_on == "host")) ||
        (bounded && (marker.size() != 1 || marker[0] == '\n' || (marker[0] & 0x80))) || (bounded && partial)) {
        usage();
        return 2;
    }
    if (sysdic.empty() || (mode != "mecab" && mode != "wakati" && mode != "detail") ||
        (format_on != "device" && format_on != "host")) {
        if (!sysdic.empty()) std::fprintf(stderr, "Could not parse a mode\n");
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
        Tokenizer tokenizer =
            Tokenizer(std::move(dict)).ignore_space(ignore_space).max_grouping_len(max_grouping_len).devices(devices);
        if (marginal) tokenizer.marginals(theta);  // before -F, which may print %pP
        if (all_morphs) tokenizer.lattice(true, true, cost_margin);  // before -F, which may print %pb
        if (sample) tokenizer.sampling(n_sample, theta, seed, true);  // before -F, which may not print %pP / %pb
        if (posterior) tokenizer.posterior(true, gamma, true);  // the text renders the posterior path
        if (has_node) {
            const std::string_view node = node_format, unk = unk_format, bos = bos_format, eos = eos_format;
            tokenizer.output_format(&node, has_unk ? &unk : nullptr, has_bos ? &bos : nullptr, has_eos ? &eos : nullptr);
        } else if (format_on == "device") {
            tokenizer.output_mode(mode);  // k_format_len / k_format_write build the text
        }
        std::fprintf(stderr, "Ready to tokenize\n");
        const bool tty_out = isatty(STDOUT_FILENO), tty_in = isatty(STDIN_FILENO);
        const size_t batch_lines = tty_in ? 1 : batch_lines_arg;
        // a line at a time: one kernel launch per line (k_small_batch has no lattice and no samples: -a and --sample
        // take the usual route)
        if (batch_lines == 1 && !all_morphs && !sample) tokenizer.small_batch(1);
        uint64_t lines_done = 0;  // input lines before the batch: the sentence index of its first line's draws
        std::string out;
        cli::Packed pk;
        std::string line;
        auto flush_batch = [&]() {
            if (pk.size() == 0) return;
            if (sample) tokenizer.sample_base(lines_done);
            lines_done += pk.size();
            BatchResult r = partial ? tokenizer.tokenize_batch(pk.utf8.data(), pk.off.data(), pk.size(), pk.bnd_off.data(),
                                                               pk.bnd.data(), pk.span_off.data(), pk.spans.data(),
                                                               pk.pat.data(), pk.pat_off.data(), pk.pat_off.size() - 1)
                            : bounded ? tokenizer.tokenize_batch(pk.utf8.data(), pk.off.data(), pk.size(), pk.bnd_off.data(),
                                                                 pk.bnd.data())
                                      : tokenizer.tokenize_batch(pk.utf8.data(), pk.off.data(), pk.size());
            if (format_on == "device") {
                std::string_view text = r.text();
                std::fwrite(text.data(), 1, text.size(), stdout);
                if (tty_out) std::fflush(stdout);
                pk.clear();
                return;
            }
            const uint64_t* to = r.tok_offsets();
            for (uint64_t s = 0; s < pk.size(); ++s) {
                std::string_view sent(pk.utf8.data() + pk.off[s], pk.off[s + 1] - pk.off[s]);
                for (uint64_t k = to[s]; k < to[s + 1]; ++k) {
                    Token t(&tokenizer, sent, r.tokens()[k]);
                    if (mode == "mecab") {
                        out.append(t.surface()).append("\t").append(t.feature()).append("\n");
                    } else if (mode == "wakati") {
                        if (k != to[s]) out.append(" ");
                        out.append(t.surface());
                    } else {
                        out.append(t.surface()).append("\t").append(t.feature());
                        out.append("\tlex_type=").append(lex_type_name(t.lex_type()));
                        out.append("\tleft_id=").append(std::to_string(t.left_id()));
                        out.append("\tright_id=").append(std::to_string(t.right_id()));
                        out.append("\tword_cost=").append(std::to_string(t.word_cost()));
                        out.append("\ttotal_cost=").append(std::to_string(t.total_cost())).append("\n");
                    }
                }
                out.append(mode == "wakati" ? "\n" : "EOS\n");
                if (tty_out || out.size() > (1u << 20)) {
                    std::fwrite(out.data(), 1, out.size(), stdout);
                    if (tty_out) std::fflush(stdout);
                    out.clear();
                }
            }
            pk.clear();
        };
        cli::PartialSentence ps;
        uint64_t line_no = 0;
        auto add_partial = [&]() {  // the sentence gathered so far, as one entry of the batch
            for (const auto& t : ps.toks) pk.add_span(t.first.first, t.first.second, t.second);
            pk.add(ps.text, ps.bnd);
            ps.clear();
            if (pk.size() >= batch_lines) flush_batch();
        };
        while (cli::read_line(std::cin, line)) {
            ++line_no;
            if (partial) {
                if (line == "EOS") {
                    add_partial();
                } else if (!ps.add_line(line)) {
                    std::fprintf(stderr, "Error: line %llu: a required token line starts with a TAB (empty surface)\n",
                                 (unsigned long long)line_no);
                    return 1;
                }
                continue;
            }
            if (bounded) {
                const std::vector<uint32_t> bnd = cli::strip_boundary_markers(line, marker[0]);
                pk.add(line, bnd);
            } else {
                pk.add(line);
            }
            if (pk.size() >= batch_lines) flush_batch();
        }
        if (partial && ps.pending) add_partial();
        flush_batch();
        std::fwrite(out.data(), 1, out.size(), stdout);
        std::fflush(stdout);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "Error: %s\n", e.what());
        return 1;
    }
    return 0;
}
