// Host-side dictionary model of the GPU tokenizer (C++17, no CUDA).
//
// Mirrors the *data* of vibrato's `Dictionary` (vibrato/src/dictionary.rs:43-51) so that the same
// MeCab-format sources and the same serialised `.dic` stream load here; the in-memory layout is
// chosen for packing into one device blob (device_blob.hpp), not copied from the reference.
// All `file:line` citations are relative to /root/reference/vibrato/src/.
#pragma once

#include <array>
#include <cstdint>
#include <optional>
#include <stdexcept>
#include <string>
#include <string_view>
#include <vector>

namespace vbt {

// Status codes crossing the C ABI (include/vibrato_b200.h). 1..9 mirror VibratoError's variants
// (errors.rs:11-42).
enum Status : int32_t {
    kOk = 0,
    kInvalidArgument = 1,
    kInvalidFormat = 2,
    kTryFromInt = 3,
    kParseInt = 4,
    kDecode = 5,  // BincodeDecode
    kEncode = 6,  // BincodeEncode
    kIo = 7,      // StdIo
    kUtf8 = 8,
    kUnsupported = 9,  // a recognised input this build cannot run (unused since the Dual connector landed)
    kCuda = 100,
    kNoDevice = 101,
    kInternal = 102,
};

struct Error : std::runtime_error {
    Status code;
    Error(Status c, const std::string& m) : std::runtime_error(m), code(c) {}
};

struct WordParam {  // lexicon/param.rs:6-10
    uint16_t left_id;
    uint16_t right_id;
    int16_t word_cost;
};

enum LexType : uint8_t { kSystem = 0, kUser = 1, kUnknown = 2 };  // dictionary.rs:30-40

// word_idx packing used across the C ABI: lex_type in the two top bits, word_id below.
inline uint32_t pack_word_idx(uint8_t lex, uint32_t id) { return (uint32_t(lex) << 30) | (id & 0x3FFFFFFFu); }

struct RawWordEntry {  // lexicon.rs:222-227
    std::string surface;
    WordParam param;
    std::string_view feature;  // borrows from the parsed buffer
};

// Lexicon::parse_csv (lexicon.rs:111-200).
std::vector<RawWordEntry> parse_lexicon_csv(std::string_view bytes, const char* name);

// Double-array trie with crawdad 0.3's search semantics and (believed) blob layout, see
// SURVEY.md Appendix B: code-mapper table + {base, check} nodes, MSB(base) = is_leaf,
// MSB(check) = has_leaf, terminal child at base ^ 0.
struct Trie {
    static constexpr uint32_t kMask = 0x7FFFFFFFu;
    static constexpr uint32_t kFlag = 0x80000000u;
    static constexpr uint32_t kInvalidCode = 0xFFFFFFFFu;

    std::vector<uint32_t> table;  // code point -> code (>= 1); kInvalidCode if unmapped
    uint32_t alphabet_size = 0;
    std::vector<uint32_t> nodes;  // interleaved base, check

    uint32_t num_nodes() const { return uint32_t(nodes.size() / 2); }
    // keys: sorted unique code-point strings with their values (map.rs:60-70).
    static Trie from_records(const std::vector<std::pair<std::u32string, uint32_t>>& records);
    // (value, end_char) pairs in ascending end_char (trie.rs:49-56).
    void common_prefix_search(const char32_t* s, size_t n, std::vector<std::pair<uint32_t, uint32_t>>& out) const;
    void serialize(std::vector<uint8_t>& out) const;           // trie.rs:14-19
    static Trie deserialize(const uint8_t* p, size_t n);       // trie.rs:21-27
    // Inverse of the construction: every (key, value), in no particular order.
    std::vector<std::pair<std::u32string, uint32_t>> enumerate() const;
};

struct Lexicon {  // lexicon.rs:24-29
    Trie trie;
    std::vector<uint32_t> postings;  // posting.rs:7-21
    std::vector<WordParam> params;   // param.rs:24-26
    std::string feature_blob;        // feature.rs:4-6, flattened
    std::vector<uint64_t> feature_off;
    uint8_t lex_type = kSystem;

    uint32_t num_words() const { return uint32_t(params.size()); }
    std::string_view feature(uint32_t id) const {
        return std::string_view(feature_blob).substr(feature_off[id], feature_off[id + 1] - feature_off[id]);
    }
    static Lexicon from_entries(const std::vector<RawWordEntry>& entries, uint8_t lex_type);  // lexicon.rs:85-96
    bool verify(uint32_t num_left, uint32_t num_right) const;                                  // lexicon.rs:68-82
};

enum ConnectorKind : uint32_t { kMatrix = 0, kRaw = 1, kDual = 2 };  // connector.rs:30-35

struct MatrixConnector {  // matrix_connector.rs:11-15
    std::vector<int16_t> data;  // data[left * num_right + right]
    uint32_t num_right = 0, num_left = 0;
    static MatrixConnector from_text(std::string_view text);  // matrix_connector.rs:27-77
    int32_t cost(uint16_t right_id, uint16_t left_id) const { return data[size_t(left_id) * num_right + right_id]; }
};

// connector/raw_connector.rs:22-27 + raw_connector/scorer.rs:171-180: connection cost = sum over the
// feature templates t of scorer(right_feats[right][t], left_feats[left][t]).
struct RawConnector {
    static constexpr uint32_t kInvalidFeature = 0x7FFFFFFFu;  // raw_connector.rs:19
    static constexpr uint32_t kUnusedCheck = 0xFFFFFFFFu;     // scorer.rs:15
    std::vector<uint32_t> right_feats, left_feats;  // [num_right][feat_T], [num_left][feat_T]
    uint32_t feat_T = 0;                             // a multiple of 8 (raw_connector.rs:64-66)
    uint32_t num_right = 0, num_left = 0;
    std::vector<uint32_t> bases, checks;  // Scorer: pos = bases[key1] ^ key2, hit iff checks[pos] == key1
    std::vector<int32_t> costs;
    static RawConnector from_text(std::string_view bigram_right, std::string_view bigram_left,
                                  std::string_view bigram_cost);  // raw_connector.rs:45-105
    // ScorerBuilder::insert x n + build (scorer.rs:110-168); triples = (key1, key2, cost) in insertion order.
    // min_bases: trie.len() of a builder whose top key1 maps were emptied afterwards (dual_connector.rs:141-152)
    void build_scorer(std::vector<std::array<int64_t, 3>> triples, size_t min_bases = 0);
    int32_t accumulate(const uint32_t* keys1, const uint32_t* keys2, size_t n) const;  // scorer.rs:240-267
    int32_t cost(uint16_t right_id, uint16_t left_id) const {                           // raw_connector.rs:155-160
        return accumulate(right_feats.data() + size_t(right_id) * feat_T, left_feats.data() + size_t(left_id) * feat_T, feat_T);
    }
};

struct ConnIdMapper {  // mapper.rs:9-12
    std::vector<uint16_t> left, right;
};

struct CharProperty {  // character.rs:105-108
    std::vector<uint32_t> chr2inf;
    std::vector<std::string> categories;
    static CharProperty from_text(std::string_view text);  // character.rs:140-191
    uint32_t char_info(uint32_t cp) const { return cp < chr2inf.size() ? chr2inf[cp] : chr2inf[0]; }  // :112-116
    int cate_id(std::string_view name) const;  // :119-124
};

struct UnkEntry {  // unknown.rs:21-27
    uint16_t cate_id, left_id, right_id;
    int16_t word_cost;
    std::string feature;
};

struct UnkHandler {  // unknown.rs:63-66
    std::vector<uint64_t> offsets;
    std::vector<UnkEntry> entries;
    static UnkHandler from_text(std::string_view text, const CharProperty& cp);  // unknown.rs:230-263
    bool verify(uint32_t num_left, uint32_t num_right) const;                     // unknown.rs:213-226
};

struct Dictionary {  // dictionary.rs:43-51
    Lexicon system;
    std::optional<Lexicon> user;
    ConnectorKind connector_kind = kMatrix;
    MatrixConnector matrix;
    RawConnector raw;  // used when connector_kind == kRaw; the 8-lane raw term of kDual
    // DualConnector (connector/dual_connector.rs:15-23): `matrix` holds the reduced matrix over the
    // matrix-side feature templates, these map a connection id to its row/column of that matrix, and
    // `raw` (feat_T == 8) scores the eight templates left out of it.
    std::vector<uint16_t> dual_right_map, dual_left_map;
    uint32_t num_left() const {
        return connector_kind == kMatrix ? matrix.num_left : connector_kind == kRaw ? raw.num_left : uint32_t(dual_left_map.size());
    }
    uint32_t num_right() const {
        return connector_kind == kMatrix ? matrix.num_right : connector_kind == kRaw ? raw.num_right : uint32_t(dual_right_map.size());
    }
    int32_t conn_cost(uint16_t right_id, uint16_t left_id) const {
        if (connector_kind == kMatrix) return matrix.cost(right_id, left_id);
        if (connector_kind == kRaw) return raw.cost(right_id, left_id);
        // DualConnector::cost (dual_connector.rs:269-280)
        return matrix.cost(dual_right_map[right_id], dual_left_map[left_id]) + raw.cost(right_id, left_id);
    }
    std::optional<ConnIdMapper> mapper;
    CharProperty char_prop;
    UnkHandler unk;

    // SystemDictionaryBuilder::from_readers (dictionary/builder.rs:64-89)
    static Dictionary from_mecab(std::string_view lex_csv, std::string_view matrix_def, std::string_view char_def,
                                 std::string_view unk_def);
    static Dictionary from_parts(std::string_view lex_csv, const int16_t* matrix, uint32_t num_right,
                                 uint32_t num_left, std::string_view char_def, std::string_view unk_def);
    // SystemDictionaryBuilder::from_readers_with_bigram_info (dictionary/builder.rs:111-148): Raw connector,
    // or the Dual connector (DualConnector::from_readers, dual_connector.rs:155-213) when dual_connector is set
    static Dictionary from_bigram(std::string_view lex_csv, std::string_view bigram_right, std::string_view bigram_left,
                                  std::string_view bigram_cost, std::string_view char_def, std::string_view unk_def,
                                  bool dual_connector = false);
    // Dictionary::read (dictionary.rs:173-197): the zstd-decoded "VibratoTokenizer 0.5\n" stream.
    static Dictionary read(const uint8_t* p, size_t n);
    // Dictionary::write (dictionary.rs:142-150)
    void write(std::vector<uint8_t>& out) const;
    // Dictionary::reset_user_lexicon_from_reader (dictionary.rs:209-229); nullopt clears.
    void reset_user_lexicon(std::optional<std::string_view> csv);
    // Dictionary::map_connection_ids_from_iter (dictionary.rs:245-259): lmap/rmap list OLD ids in their
    // NEW order (ConnIdMapper::parse, mapper.rs:49-80).
    void map_connection_ids(const std::vector<uint16_t>& lmap, const std::vector<uint16_t>& rmap);

    WordParam word_param(uint32_t word_idx) const;         // dictionary.rs:98-104
    std::string_view word_feature(uint32_t word_idx) const;  // dictionary.rs:108-114

   private:
    void finish_build(std::string_view lex_csv, std::string_view char_def, std::string_view unk_def);
};

// utils::parse_csv_row (utils.rs:41-61): the fields of one CSV row
std::vector<std::string> parse_csv_row(std::string_view row);
// BufRead::lines(): next line without its "\n" / "\r\n"; false at the end of the text
bool next_line(std::string_view text, size_t& pos, std::string_view& line);

// UTF-8 helpers
bool utf8_valid(const uint8_t* s, size_t n);
std::u32string utf8_to_u32(std::string_view s);

// zstd frame decoding through the runtime libzstd.so.1 (no headers in this image).
std::vector<uint8_t> zstd_decompress_file(const char* path);
// zstd::Encoder::new(File::create(path), level) + write_all + finish (compile/src/main.rs:98-100): one frame that
// carries its content size.  Fails with kIo and removes the partly written file.
void zstd_compress_to_file(const std::vector<uint8_t>& data, const char* path, int level);

}  // namespace vbt
