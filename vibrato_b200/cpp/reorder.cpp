// `reorder` look-alike: same flags, messages and output as the reference tool (/root/reference/map/src/reorder.rs):
// tokenises the sentences of stdin with connection-id counting on the GPU, in batches, and writes the ids by
// descending occurrence probability to `<out>.lmap` / `<out>.rmap` (`{id}\t{p}` lines), the input of `map`.
//
// An empty line counts the previous sentence's lattice once more, as in the reference: Worker::tokenize returns early on
// an empty sentence and update_connid_counts counts the lattice it left in place (worker.rs:49-55, 90-93).  So an empty
// line is tokenised as the last non-empty line before it.  The reference panics on an empty first line; this tool
// stops with an error.  Nothing is written unless every line was tokenised.
#include "cli_common.hpp"

using namespace vibrato_b200;

static void usage() {
    std::fprintf(stderr,
                 "Usage: reorder -i <system.dic.zst | mecab-source-dir> -o <mapping basename> < sentences.txt\n"
                 "               [--devices 0,1,..]   (spread every batch over these GPUs)\n"
                 "               [--batch-lines N]    (lines per batch; default 65536)\n");
}

static void write_mapping(const std::string& path, const ConnIdProbs& probs) {
    const std::string text = cli::mapping_text(probs);
    FILE* f = std::fopen(path.c_str(), "wb");
    if (!f) throw std::runtime_error("cannot create " + path);
    const bool ok = std::fwrite(text.data(), 1, text.size(), f) == text.size();
    if (std::fclose(f) != 0 || !ok) throw std::runtime_error("cannot write " + path);
    std::printf("Wrote %s\n", cli::rust_debug_path(path).c_str());
}

int main(int argc, char** argv) {
    std::string sysdic_in, mapping_out;
    size_t batch_lines = 65536;
    std::vector<int32_t> devices;
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        auto next = [&]() -> std::string {
            if (i + 1 >= argc) {
                usage();
                std::exit(2);
            }
            return argv[++i];
        };
        try {
            if (a == "-i" || a == "--sysdic-in") sysdic_in = next();
            else if (a == "-o" || a == "--mapping-out") mapping_out = next();
            else if (a == "--devices") devices = cli::parse_devices(next());
            else if (a == "--batch-lines") batch_lines = std::stoull(next());
            else {
                usage();
                return 2;
            }
        } catch (const std::logic_error&) {  // std::stoul / std::stoull: not a number
            usage();
            return 2;
        }
    }
    if (sysdic_in.empty() || mapping_out.empty() || batch_lines == 0) {
        usage();
        return 2;
    }
    try {
        std::fprintf(stderr, "Loading the dictionary...\n");
        Dictionary dict = cli::load_dictionary(sysdic_in);
        std::fprintf(stderr, "Reordering connection id mappings...\n");
        Tokenizer tokenizer = Tokenizer(std::move(dict)).devices(devices);
        tokenizer.init_connid_counter();
        cli::Packed pk;
        std::string line, last;
        uint64_t n_lines = 0;
        auto flush_batch = [&]() {
            if (pk.size() == 0) return;
            tokenizer.tokenize_batch(pk.utf8.data(), pk.off.data(), pk.size());
            pk.clear();
        };
        while (cli::read_line(std::cin, line)) {
            ++n_lines;
            if (!line.empty()) last = line;
            else if (n_lines == 1)
                throw std::runtime_error("line 1 is empty: an empty line counts the lattice of the sentence before it "
                                         "again, and the first line has none");
            pk.add(last);
            if (pk.size() >= batch_lines) flush_batch();
        }
        flush_batch();
        const auto [lid_probs, rid_probs] = tokenizer.compute_connid_probs();
        std::fprintf(stderr, "Writing connection id mappings...\n");
        write_mapping(cli::set_extension(mapping_out, "lmap"), lid_probs);
        write_mapping(cli::set_extension(mapping_out, "rmap"), rid_probs);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "Error: %s\n", e.what());
        return 1;
    }
    return 0;
}
