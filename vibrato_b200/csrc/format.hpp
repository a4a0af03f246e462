// MeCab-style output formats (node / unk / BOS / EOS format strings), compiled on the host into one compact program
// that the output stage (kernels.cu, mode kOutFormat) interprets on the device.
//
// Directives per token ("prev" = the previous token of the sentence, or BOS with cost 0 and end byte 0):
//   %m surface   %M prev's end byte .. end byte   %pS prev's end byte .. start byte   %H the raw feature string
//   %f[N,..] feature fields (csv-core split, unquoted) joined by TAB   %F<c>[N,..] the same joined by <c>
//   (a field whose text begins with '*', or that the feature does not have, is left out with its separator)
//   %c %pw word cost   %pc total cost   %pn total - prev's total   %pC total - prev's total - word cost (wrapping i32)
//   %ps %pe %pl %pL start byte, end byte, surface bytes, end byte - prev's end byte   %phl %phr left / right id
//   %s 0 for System / User words, 1 for Unknown   %S %L the whole sentence, its byte length   %% '%'
//   %pP the token's marginal probability as d.dddddd (only while marginals are on)
//   %pb '*' for a node of the best path, ' ' otherwise (only in lattice text, option "lattice" = 2, where the "prev"
//   directives %M %pS %pn %pC %pL are refused: a node has no previous token)
// Sample text ("sample_text" = 1) renders each sampled path like a sentence's tokens: "prev" is the previous record of
// the same sample, and %pP / %pb are refused (a sampled record has no marginal and no best-path flag).
// Escapes \0 \a \b \t \n \v \f \r \s(space) \\ are replaced by the compiler.  BOS / EOS take literals, %%, %S, %L.
#pragma once

#include <cstddef>
#include <cstdint>

namespace vbt {

enum FormatOpKind : uint8_t {
    kOpLit = 0,      // lit[at .. at + n)
    kOpSurface,      // %m
    kOpSurfaceWs,    // %M
    kOpWs,           // %pS
    kOpFeature,      // %H
    kOpFields,       // %f / %F: field positions slot[at .. at + n) joined by `sep`
    kOpWordCost,     // %c, %pw
    kOpTotalCost,    // %pc
    kOpCostDiff,     // %pn
    kOpConnCost,     // %pC
    kOpStart,        // %ps
    kOpEnd,          // %pe
    kOpSurfLen,      // %pl
    kOpSurfLenWs,    // %pL
    kOpLeftId,       // %phl
    kOpRightId,      // %phr
    kOpStat,         // %s
    kOpSentence,     // %S
    kOpSentLen,      // %L
    kOpProb,         // %pP
    kOpBest,         // %pb (lattice text)
};

struct FormatOp {
    uint8_t kind;
    uint8_t sep;  // kOpFields: the separator byte
    uint16_t n;
    uint32_t at;
};

constexpr uint32_t kFmtMaxOps = 256, kFmtMaxSlots = 256, kFmtMaxLit = 2048, kFmtMaxFields = 16, kFmtMaxFieldIndex = 255;
enum : uint32_t { kSecNode = 0, kSecUnk = 1, kSecBos = 2, kSecEos = 3 };
// what a token's values must be loaded for (FormatProgram::uses)
enum : uint32_t { kUsesPrev = 1u, kUsesParams = 2u, kUsesFeature = 4u, kUsesFields = 8u, kUsesProb = 16u, kUsesBest = 32u };

// Laid out so that the used part is a prefix of each array: the kernels stage the header, ops[0 .. n_ops),
// slot[0 .. n_slots) and lit[0 .. n_lit) in shared memory.
struct FormatProgram {
    uint16_t sec[4][2];  // [first, end) op of the node, unk, bos and eos sections
    uint32_t n_ops, n_slots, n_lit, n_fields;
    uint32_t uses;
    uint32_t per_sentence;  // text bytes bos + eos give a sentence besides copies of it (sizing of the text buffers)
    uint8_t fields[kFmtMaxFields];  // the feature-field indices referenced, sorted and distinct
    FormatOp ops[kFmtMaxOps];
    uint8_t slot[kFmtMaxSlots];  // kOpFields: positions in fields[] (= in the field table) of the listed fields
    uint8_t lit[kFmtMaxLit];
};
constexpr uint32_t kFmtHeaderBytes = offsetof(FormatProgram, ops);

#ifndef __CUDACC__
struct FormatText {  // one format string: ptr == nullptr means "not given"
    const char* ptr;
    size_t len;
};
// Compiles node / unk / bos / eos (unk not given = node, bos = "", eos = "EOS\n").  Throws
// Error(kInvalidArgument, "<which> format, byte <pos>: ...") naming the offending directive or escape.
// `marginals`: the tokenizer computes marginal probabilities, so %pP has a value (otherwise it is refused).
// `lattice_text`: the text renders lattice nodes ("lattice" = 2), so %pb has a value and the "prev" directives do not.
// `sample_text`: the text renders the samples ("sample_text" = 1), so neither %pP nor %pb has a value.
FormatProgram compile_format(FormatText node, FormatText unk, FormatText bos, FormatText eos, bool marginals = false,
                             bool lattice_text = false, bool sample_text = false);
#endif

}  // namespace vbt
