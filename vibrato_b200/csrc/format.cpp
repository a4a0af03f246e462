// Compiler of the MeCab-style format strings (format.hpp).
#include "format.hpp"

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "host_dict.hpp"

namespace vbt {

namespace {

class Compiler {
   public:
    Compiler(FormatProgram& p, bool marginals, bool lattice_text, bool sample_text)
        : p_(p), marginals_(marginals), lattice_text_(lattice_text), sample_text_(sample_text) {}

    // Appends the ops of one format string as section `sec`; `tokens` = false admits only what BOS / EOS can print.
    void section(uint32_t sec, const char* name, const char* s, size_t n, bool tokens) {
        name_ = name;
        open_lit_ = false;
        p_.sec[sec][0] = uint16_t(p_.n_ops);
        for (size_t i = 0; i < n;) {
            const size_t at = i;
            const char c = s[i];
            if (c == '\\') {
                lit_byte(escape(s, n, i), at);
                continue;
            }
            if (c != '%') {
                lit_byte(uint8_t(c), at);
                ++i;
                continue;
            }
            ++i;
            if (i >= n) fail(at, "'%' at the end of the string");
            const char d = s[i++];
            if (d == '%') {
                lit_byte('%', at);
                continue;
            }
            if (d == 'S') {
                op(kOpSentence, at);
                continue;
            }
            if (d == 'L') {
                op(kOpSentLen, at);
                continue;
            }
            std::string dir = std::string("%") + d;
            if (d == 'p') {
                if (i >= n) fail(at, "unknown directive %p");
                dir += s[i++];
                if (dir == "%ph" && i < n && (s[i] == 'l' || s[i] == 'r')) dir += s[i++];
            }
            if (sample_text_ && (dir == "%pP" || dir == "%pb"))
                fail(at, dir + " has no value in sample text (option \"sample_text\" = 1): a sampled token has no " +
                             (dir == "%pP" ? "marginal" : "best-path flag"));
            if (dir == "%pP" && marginals_) {
                if (!tokens) fail(at, dir + " is not allowed here (only literals, %%, %S and %L)");
                op(kOpProb, at);
                p_.uses |= kUsesProb;
                continue;
            }
            if (dir == "%pb" && lattice_text_) {
                if (!tokens) fail(at, dir + " is not allowed here (only literals, %%, %S and %L)");
                op(kOpBest, at);
                p_.uses |= kUsesBest;
                continue;
            }
            if (lattice_text_ && (dir == "%M" || dir == "%pS" || dir == "%pn" || dir == "%pC" || dir == "%pL"))
                fail(at, dir + " has no value in lattice text (option \"lattice\" = 2): a node has no previous token");
            static const char* const kNoValue[] = {"%h", "%t", "%P", "%pP", "%pA", "%pB", "%pi", "%pb", "%pp"};
            for (const char* nv : kNoValue)
                if (dir == nv) fail(at, dir + " has no value for the tokens of the best path");
            struct Simple {
                const char* dir;
                uint8_t kind;
                uint32_t uses;
            };
            static const Simple kSimple[] = {
                {"%m", kOpSurface, 0},           {"%M", kOpSurfaceWs, kUsesPrev},  {"%pS", kOpWs, kUsesPrev},
                {"%H", kOpFeature, kUsesFeature}, {"%c", kOpWordCost, kUsesParams}, {"%pw", kOpWordCost, kUsesParams},
                {"%pc", kOpTotalCost, 0},         {"%pn", kOpCostDiff, kUsesPrev},  {"%pC", kOpConnCost, kUsesPrev | kUsesParams},
                {"%ps", kOpStart, 0},             {"%pe", kOpEnd, 0},               {"%pl", kOpSurfLen, 0},
                {"%pL", kOpSurfLenWs, kUsesPrev}, {"%phl", kOpLeftId, kUsesParams}, {"%phr", kOpRightId, kUsesParams},
                {"%s", kOpStat, 0},
            };
            bool done = false;
            for (const Simple& k : kSimple) {
                if (dir != k.dir) continue;
                if (!tokens) fail(at, dir + " is not allowed here (only literals, %%, %S and %L)");
                op(k.kind, at);
                p_.uses |= k.uses;
                done = true;
                break;
            }
            if (done) continue;
            if (dir == "%f" || dir == "%F") {
                if (!tokens) fail(at, dir + " is not allowed here (only literals, %%, %S and %L)");
                uint8_t sep = '\t';
                if (d == 'F') {
                    if (i >= n) fail(at, "malformed %F: a separator and a field list must follow");
                    if (s[i] == '\\')
                        sep = escape(s, n, i);
                    else
                        sep = uint8_t(s[i++]);
                }
                fields(at, dir, s, n, i, sep);
                continue;
            }
            fail(at, "unknown directive " + dir);
        }
        p_.sec[sec][1] = uint16_t(p_.n_ops);
        open_lit_ = false;
    }

    // The field indices referenced, sorted: slot[] then holds positions in that list.
    void finish() {
        std::vector<uint32_t> idx(raw_.begin(), raw_.end());
        std::sort(idx.begin(), idx.end());
        p_.n_fields = uint32_t(idx.size());
        for (size_t k = 0; k < idx.size(); ++k) p_.fields[k] = uint8_t(idx[k]);
        for (uint32_t k = 0; k < p_.n_slots; ++k)
            p_.slot[k] = uint8_t(std::lower_bound(idx.begin(), idx.end(), p_.slot[k]) - idx.begin());
        if (p_.n_fields) p_.uses |= kUsesFields;
    }

   private:
    [[noreturn]] void fail(size_t at, const std::string& what) const {
        throw Error(kInvalidArgument, std::string(name_) + " format, byte " + std::to_string(at) + ": " + what);
    }

    uint8_t escape(const char* s, size_t n, size_t& i) const {
        const size_t at = i;
        if (i + 1 >= n) fail(at, "'\\' at the end of the string");
        const char e = s[i + 1];
        i += 2;
        switch (e) {
            case '0': return 0;
            case 'a': return '\a';
            case 'b': return '\b';
            case 't': return '\t';
            case 'n': return '\n';
            case 'v': return '\v';
            case 'f': return '\f';
            case 'r': return '\r';
            case 's': return ' ';
            case '\\': return '\\';
            default: fail(at, std::string("unknown escape \\") + e);
        }
    }

    void lit_byte(uint8_t b, size_t at) {
        if (p_.n_lit >= kFmtMaxLit) fail(at, "the literals of the format exceed 2048 bytes");
        if (!open_lit_) {
            op(kOpLit, at);
            p_.ops[p_.n_ops - 1].at = p_.n_lit;
            open_lit_ = true;
        }
        p_.lit[p_.n_lit++] = b;
        ++p_.ops[p_.n_ops - 1].n;
    }

    void op(uint8_t kind, size_t at) {
        if (p_.n_ops >= kFmtMaxOps) fail(at, "the format has more than 256 pieces");
        p_.ops[p_.n_ops++] = FormatOp{kind, 0, 0, 0};
        open_lit_ = false;
    }

    // `[N1,N2,..]` at s[i]
    void fields(size_t at, const std::string& dir, const char* s, size_t n, size_t& i, uint8_t sep) {
        if (i >= n || s[i] != '[') fail(at, "malformed " + dir + ": '[' expected");
        ++i;
        op(kOpFields, at);
        FormatOp& o = p_.ops[p_.n_ops - 1];
        o.sep = sep;
        o.at = p_.n_slots;
        for (;;) {
            if (i >= n || s[i] < '0' || s[i] > '9') fail(at, "malformed " + dir + ": a field index expected");
            uint32_t v = 0;
            while (i < n && s[i] >= '0' && s[i] <= '9') {
                v = v * 10 + uint32_t(s[i++] - '0');
                if (v > kFmtMaxFieldIndex) fail(at, dir + ": field index above 255");
            }
            if (p_.n_slots >= kFmtMaxSlots) fail(at, "the format lists more than 256 fields");
            p_.slot[p_.n_slots++] = uint8_t(v);
            ++o.n;
            if (std::find(raw_.begin(), raw_.end(), v) == raw_.end()) {
                if (raw_.size() == kFmtMaxFields) fail(at, dir + ": more than 16 distinct feature fields are referenced");
                raw_.push_back(v);
            }
            if (i < n && s[i] == ',') {
                ++i;
                continue;
            }
            if (i < n && s[i] == ']') {
                ++i;
                return;
            }
            fail(at, "malformed " + dir + ": ',' or ']' expected");
        }
    }

    FormatProgram& p_;
    const char* name_ = "";
    bool marginals_ = false;
    bool lattice_text_ = false;
    bool sample_text_ = false;
    bool open_lit_ = false;
    std::vector<uint32_t> raw_;
};

// Bytes the ops [a, b) write whatever the sentence: literals, and at most 10 digits per %L.
uint32_t fixed_bytes(const FormatProgram& p, uint32_t a, uint32_t b) {
    uint32_t n = 0;
    for (uint32_t k = a; k < b; ++k) n += p.ops[k].kind == kOpLit ? p.ops[k].n : p.ops[k].kind == kOpSentLen ? 10 : 0;
    return n;
}

}  // namespace

FormatProgram compile_format(FormatText node, FormatText unk, FormatText bos, FormatText eos, bool marginals,
                             bool lattice_text, bool sample_text) {
    FormatProgram p;
    std::memset(&p, 0, sizeof p);
    Compiler c(p, marginals, lattice_text, sample_text);
    if (!node.ptr) throw Error(kInvalidArgument, "format: the node format must be given");
    c.section(kSecNode, "node", node.ptr, node.len, true);
    if (unk.ptr) {
        c.section(kSecUnk, "unk", unk.ptr, unk.len, true);
    } else {
        p.sec[kSecUnk][0] = p.sec[kSecNode][0];
        p.sec[kSecUnk][1] = p.sec[kSecNode][1];
    }
    if (bos.ptr) c.section(kSecBos, "bos", bos.ptr, bos.len, false);
    else p.sec[kSecBos][0] = p.sec[kSecBos][1] = uint16_t(p.n_ops);
    static const char kEos[] = "EOS\n";
    if (eos.ptr) c.section(kSecEos, "eos", eos.ptr, eos.len, false);
    else c.section(kSecEos, "eos", kEos, 4, false);
    c.finish();
    p.per_sentence = std::max<uint32_t>(4, fixed_bytes(p, p.sec[kSecBos][0], p.sec[kSecBos][1]) +
                                               fixed_bytes(p, p.sec[kSecEos][0], p.sec[kSecEos][1]));
    return p;
}

}  // namespace vbt
