// `map` look-alike: same flags, messages and output as the reference tool (/root/reference/map/src/main.rs): renumbers
// the connection ids of a system dictionary by the `<mapping>.lmap` / `<mapping>.rmap` files that `reorder` writes and
// writes the result as `system.dic.zst` (level 19).  Any error leaves no output file.
#include "cli_common.hpp"

using namespace vibrato_b200;

static void usage() {
    std::fprintf(stderr, "Usage: map -i <system.dic.zst | mecab-source-dir> -m <mapping basename> -o <mapped.dic.zst>\n");
}

// load_mapping (main.rs:61-74): the first tab-separated column of every line, as a u16
static std::vector<uint16_t> load_mapping(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error("cannot open " + path);
    std::vector<uint16_t> ids;
    std::string line;
    while (cli::read_line(f, line)) {
        try {
            ids.push_back(cli::parse_u16(std::string_view(line).substr(0, line.find('\t'))));
        } catch (const std::runtime_error& e) {
            throw std::runtime_error(path + " line " + std::to_string(ids.size() + 1) + ": " + e.what());
        }
    }
    return ids;
}

int main(int argc, char** argv) {
    std::string sysdic_in, mapping_in, sysdic_out;
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        auto next = [&]() -> std::string {
            if (i + 1 >= argc) {
                usage();
                std::exit(2);
            }
            return argv[++i];
        };
        if (a == "-i" || a == "--sysdic-in") sysdic_in = next();
        else if (a == "-m" || a == "--mapping-in") mapping_in = next();
        else if (a == "-o" || a == "--sysdic-out") sysdic_out = next();
        else {
            usage();
            return 2;
        }
    }
    if (sysdic_in.empty() || mapping_in.empty() || sysdic_out.empty()) {
        usage();
        return 2;
    }
    try {
        std::fprintf(stderr, "Loading the dictionary...\n");
        Dictionary dict = cli::load_dictionary(sysdic_in);
        std::fprintf(stderr, "Loading and doing the mapping...\n");
        const std::vector<uint16_t> lmap = load_mapping(cli::set_extension(mapping_in, "lmap"));
        const std::vector<uint16_t> rmap = load_mapping(cli::set_extension(mapping_in, "rmap"));
        dict = std::move(dict).map_connection_ids_from_iter(lmap, rmap);
        std::fprintf(stderr, "Writing the mapped system dictionary...: %s\n", cli::rust_debug_path(sysdic_out).c_str());
        dict.write_zstd_file(sysdic_out, 19);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "Error: %s\n", e.what());
        return 1;
    }
    return 0;
}
