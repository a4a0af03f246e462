// Device engine: owns the dictionary image in HBM, the per-batch workspace and the launch sequence.
#pragma once

#include <array>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "format.hpp"
#include "host_dict.hpp"

namespace vbt {

// ---- the outputs of a batch ------------------------------------------------------------------------
// A batch produces up to twenty-one arrays in six ragged groups.  A group's offsets index its records: entries
// off[i] .. off[i + 1] belong to sentence i (to sample j of sentence i at i * n_samp + j for the samples), and the
// group's total is the number of its records.  path_prob, entropy and log_path_prob have one entry per sentence and no
// offsets.  The positions group has one record per character position 0..n of every sentence: its offsets are the
// slot offsets and its total is the batch's slot count.  The posterior group holds each sentence's posterior path.
enum Group { kGroupTokens, kGroupText, kGroupLattice, kGroupSamples, kGroupPositions, kGroupPosterior, kNumGroups };
enum Array {
    kTokOff, kTokens, kTokenProb, kPathProb,  // vbt_token (or vbt_token16) records; marginals (set_marginals)
    kEntropy, kLogPathProb,                   // uncertainty ("uncertainty" >= 1): float64 per sentence
    kTextOff, kText,                          // output stage ("output_mode" or a format): the text `tokenize` prints
    kNodeOff, kNodes, kLinks, kNodeProb,      // lattice ("lattice" >= 1): vbt_token nodes, vbt_lattice_link, marginals
    kNodeMargin,                              // near-best lattice ("lattice_margin" >= 0): each kept node's margin (int64)
    kSampleOff, kSamples,                     // sampling (set_sampling): vbt_token records of every sampled path
    kPosOff, kBoundaryProb,                   // uncertainty 2: float32 boundary probability of every character position
    kPostOff, kPostTokens, kPostProb,         // posterior decoding (set_posterior): vbt_token records and their marginals
    kPostGain,                                // ... and each sentence's total gain (float64)
    kNumArrays
};
enum ArrayKind { kOffsets, kRecords, kPerSentence };
struct ArrayInfo {
    Group group;
    ArrayKind kind;
    uint32_t bytes;  // per element; 0 = the token record size
};
constexpr ArrayInfo kArrays[kNumArrays] = {
    {kGroupTokens, kOffsets, 8},   {kGroupTokens, kRecords, 0},  {kGroupTokens, kRecords, 4},   {kGroupTokens, kPerSentence, 4},
    {kGroupTokens, kPerSentence, 8}, {kGroupTokens, kPerSentence, 8},
    {kGroupText, kOffsets, 8},     {kGroupText, kRecords, 1},    {kGroupLattice, kOffsets, 8},  {kGroupLattice, kRecords, 24},
    {kGroupLattice, kRecords, 8},  {kGroupLattice, kRecords, 4}, {kGroupLattice, kRecords, 8},  {kGroupSamples, kOffsets, 8},
    {kGroupSamples, kRecords, 24}, {kGroupPositions, kOffsets, 8}, {kGroupPositions, kRecords, 4},
    {kGroupPosterior, kOffsets, 8}, {kGroupPosterior, kRecords, 24}, {kGroupPosterior, kRecords, 4},
    {kGroupPosterior, kPerSentence, 8},
};
constexpr Array kOffsetsOf[kNumGroups] = {kTokOff, kTextOff, kNodeOff, kSampleOff, kPosOff, kPostOff};

using Totals = std::array<uint64_t, kNumGroups>;  // one count per group

// Which arrays a batch carries, decided by its output options, and where a piece of the batch goes in each.
struct Outputs {
    uint32_t token_bytes = 24;  // 24, or 16 with "compact_tokens"
    uint32_t n_samp = 0;        // sampled paths per sentence, 0 = sampling off
    bool marg = false, text = false, lat = false;
    bool margin = false;  // "lattice_margin" >= 0: the lattice keeps the near-best nodes and carries their margins
    uint32_t unc = 0;     // "uncertainty": 1 entropy and log_path_prob, 2 also the boundary probabilities
    bool post = false;    // posterior decoding (set_posterior)

    bool has(int a) const {
        switch (a) {
            case kTokenProb:
            case kPathProb: return marg;
            case kEntropy:
            case kLogPathProb: return marg && unc >= 1;
            case kPosOff:
            case kBoundaryProb: return marg && unc >= 2;
            case kTextOff:
            case kText: return text;
            case kNodeOff:
            case kNodes:
            case kLinks: return lat;
            case kNodeProb: return lat && marg;
            case kNodeMargin: return lat && margin;
            case kSampleOff:
            case kSamples: return n_samp != 0;
            case kPostOff:
            case kPostTokens:
            case kPostProb:
            case kPostGain: return marg && post;
            default: return true;
        }
    }
    uint64_t elem_bytes(int a) const { return kArrays[a].bytes ? kArrays[a].bytes : token_bytes; }
    uint64_t stride(int a) const { return kArrays[a].kind == kOffsets && kArrays[a].group == kGroupSamples ? n_samp : 1; }
    // Bytes of array a in a piece of n sentences whose groups hold `count` records; `last`: the piece that ends the
    // batch also brings the closing offset.
    uint64_t bytes(int a, uint64_t n, const Totals& count, bool last) const {
        if (kArrays[a].kind == kRecords) return count[kArrays[a].group] * elem_bytes(a);
        return (n * stride(a) + (kArrays[a].kind == kOffsets && last ? 1 : 0)) * elem_bytes(a);
    }
    // Byte position of that piece in the batch's array: it starts at sentence s0, its records after `base` others.
    uint64_t at(int a, uint64_t s0, const Totals& base) const {
        return (kArrays[a].kind == kRecords ? base[kArrays[a].group] : s0 * stride(a)) * elem_bytes(a);
    }
};

// Pinned host memory, freed with the buffer.
struct PinnedBuf {
    void* p = nullptr;
    size_t cap = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf();
    void ensure(size_t bytes);                   // room for `bytes`; the contents are not kept
    void grow(size_t bytes, size_t keep_bytes);  // room for `bytes`, keeping the first keep_bytes
};

// Device memory that grows on demand (engine.cu, multi_engine.cu).
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    void ensure(size_t bytes, double slack = 1.0);  // room for `bytes` (times slack when it grows); contents not kept
    void release();
    template <typename T>
    T* as() const {
        return static_cast<T*>(p);
    }
};

// What the last run_device (on a shard engine: run_shard) left in device memory, valid until the next call.
struct DeviceOutputs {
    Outputs made{};                  // the arrays it produced
    Totals total{};                  // records per group
    uint64_t addr[kNumArrays] = {};  // device address of array a, 0 when !made.has(a)
};

struct HostResult {  // one batch's outputs in pinned host memory
    uint64_t n_sent = 0;
    Outputs out;
    Totals total{};
    PinnedBuf buf[kNumArrays];  // buf[a] holds array a when out.has(a)
    template <typename T>
    T* ptr(int a) const {
        return static_cast<T*>(buf[a].p);
    }
};

// Pooled host results, reused across calls.
class ResultPool {
   public:
    // A result for n_sent sentences carrying `out`, with room for `total` records per group.
    HostResult* acquire(const Outputs& out, uint64_t n_sent, const Totals& total);
    void release(HostResult* r) {
        if (r) free_.push_back(r);
    }

   private:
    std::vector<std::unique_ptr<HostResult>> all_;
    std::vector<HostResult*> free_;
};

// Required tokens of a batch (vbt_tokenize_batch_spans): sentence i's spans are rec[off[i] .. off[i+1]), three words
// {start_byte, end_byte, pattern} each, in host or device memory like the boundaries they travel with; the compiled
// patterns (kernels.cuh SpanArgs) are always in host memory: pat_off[n_pat + 1] into pf, whose fields index pat_bytes.
struct Spans {
    const uint64_t* off = nullptr;  // n_sent + 1; nullptr = no spans
    const uint32_t* rec = nullptr;
    uint64_t n = 0;
    const uint32_t* pat_off = nullptr;
    const uint32_t* pf = nullptr;  // 3 words per field: {field index, first byte, length}
    const uint8_t* pat_bytes = nullptr;
    uint32_t n_pat = 0;
    uint64_t n_pat_bytes = 0;
};
// Required token boundaries of a batch (vbt_tokenize_batch_bounded): sentence i's boundaries are the
// sentence-relative byte offsets bnd[off[i] .. off[i+1]), and bnd holds n entries.  Host or device addresses, as the
// call that takes them says.  A null pointer to Bounds = an unbounded batch.
// With spans, off may be nullptr (no explicit boundary) and the batch is still bounded: the span ends are boundaries.
struct Bounds {
    const uint64_t* off = nullptr;  // n_sent + 1
    const uint32_t* bnd = nullptr;
    uint64_t n = 0;
    Spans spans;
};

// The input errors a batch can hold, in the order it reports them: a batch with several reports the first of these,
// whichever sentences hold them (the multi-device engine keeps that order across its shards).
constexpr const char* kBadOffsetsMsg = "byte_offsets must be non-decreasing and end within the input buffer";
constexpr const char* kBadUtf8Msg = "stream did not contain valid UTF-8";  // what `stdin.lines()` reports
constexpr const char* kBadBoundsMsg =
    "required boundaries must be non-decreasing, at most the sentence's byte length and on a UTF-8 lead byte, "
    "and their offsets non-decreasing and within the boundary array";
constexpr const char* kBadSpansMsg =
    "required tokens (spans) must have start < end <= the sentence's byte length, both on a UTF-8 lead byte or at the "
    "end, be sorted and non-overlapping, name VBT_SPAN_ANY or a pattern of the call, hold no explicit boundary "
    "inside, not start at a space when ignore_space is on, and their offsets must be non-decreasing and within the "
    "span array";
struct InputError {
    uint32_t flag;  // the kernels' batch flag (kernels.cuh kFlag*)
    Status status;
    const char* msg;
};
constexpr int kNumInputErrors = 4;
extern const InputError kInputErrors[kNumInputErrors];  // engine.cu: the four above, in that order

// Why a call ran an attempt again: its candidate pool, its per-character slots or (chunked host batches) the output
// text of a chunk outgrew the size learned from earlier batches.  An attempt with several counts under each.
enum Rerun { kRerunPool, kRerunSlots, kRerunText, kNumReruns };
using Reruns = std::array<uint64_t, kNumReruns>;
// describe()'s "last_reruns" entry: the attempts the last call re-ran, by reason.
inline std::string reruns_json(const Reruns& r) {
    return "\"last_reruns\": {\"pool\": " + std::to_string(r[kRerunPool]) + ", \"slots\": " + std::to_string(r[kRerunSlots]) +
           ", \"text\": " + std::to_string(r[kRerunText]) + "}";
}

constexpr int kNumStages = 9;
extern const char* const kStageNames;  // comma-separated, kNumStages entries
// A call on the k_small_batch route ("small_batch" option) runs every stage in one kernel: its whole time is booked
// under "viterbi" and the other stages read 0.
constexpr int kSmallBatchStage = 5;

class Engine {
   public:
    // host_blob: packed dictionary image (device_blob.hpp) to upload; or d_blob: an image already
    // resident on `device` (not owned).
    static std::unique_ptr<Engine> create(int device, const uint8_t* host_blob, uint64_t d_blob, uint64_t n_bytes,
                                          bool ignore_space, uint64_t max_grouping_len);
    // One tokenizer over several devices of this node (multi_engine.cu): the image is uploaded to devices[0] and
    // broadcast (NCCL when libnccl.so.2 loads, peer copies otherwise); batches are split by bytes.
    static std::unique_ptr<Engine> create_multi(const std::vector<int>& devices, const uint8_t* host_blob, uint64_t n_bytes,
                                                bool ignore_space, uint64_t max_grouping_len);
    virtual ~Engine() = default;

    // Inputs/outputs in device memory; outputs owned by the engine until the next call, described by last_device().
    // With bnd: a bounded batch, its boundary arrays in device memory too.  Bounded batches refuse "counting".
    virtual void run_device(uint64_t d_utf8, uint64_t d_byte_off, uint64_t n_sent, uint64_t n_bytes, const Bounds* bnd = nullptr) = 0;
    // The arrays the last run_device (or run_shard) left in device memory.  After a run_device that failed, `made`
    // holds no optional array; run_host leaves the record alone.
    virtual const DeviceOutputs& last_device() const = 0;
    // Inputs/outputs in host memory (copies inside); bnd in host memory.
    virtual HostResult* run_host(const char* utf8, const uint64_t* byte_off, uint64_t n_sent, const Bounds* bnd = nullptr) = 0;
    virtual void release(HostResult* r) = 0;

    // Building blocks of the multi-device engine (multi_engine.cu); a single-device caller never needs them.
    // run_shard: host sentences in, outputs left in this device's memory; returns their record counts per group
    // (synchronises).  With src_device >= 0 `utf8` is a DEVICE address on that device (peer copy over NVLink) while
    // byte_off is still a host array.  first_sentence is the caller's index of the shard's first sentence (the i of the
    // sampling draws), so that a shard draws what the whole batch would.  With with_text the shard's output text is
    // formatted too, when an output mode or format is set.  bnd (host memory, may be null) holds the shard's
    // n_sent + 1 boundary offsets.  last_device() then describes the shard's arrays.
    virtual Totals run_shard(const char* utf8, const uint64_t* byte_off, uint64_t n_sent, int src_device,
                             uint64_t first_sentence, bool with_text, const Bounds* bnd = nullptr) = 0;
    // rebase_shard: adds base[g] to the last shard's offsets of every group g it produced, on the device.
    virtual void rebase_shard(const Totals& base) = 0;
    // fetch_shard: rebases the last shard like rebase_shard, then copies every array r carries into r at the shard's
    // place: sentence first_sentence and records after base[g] others (the closing offsets too when `last`).
    virtual void fetch_shard(HostResult* r, uint64_t first_sentence, const Totals& base, bool last) = 0;
    virtual int device() const = 0;
    virtual uint32_t token_bytes() const = 0;  // 24, or 16 with the "compact_tokens" option
    virtual std::string describe() const = 0;  // JSON: devices, how the dictionary travelled, ...
    virtual Reruns last_reruns() const = 0;    // the attempts the last call re-ran (a multi-device one: over its shards)

    virtual void set_counting(bool on) = 0;
    // Knobs: "lanes_per_sentence" (4/8/16/32), "sort_by_length" (0/1), "counting" (0/1), "chunk_sentences",
    // "dual_stream", "connid_counting", "output_mode" (0 none, 1 mecab, 2 wakati, 3 detail: run_host also
    // produces the text arrays, on every host route; run_device stays token-only), "small_batch" (N > 0: run_host
    // takes k_small_batch for batches of at most N sentences and 16 KiB without counting; run_device and the shards
    // of a multi-device engine keep the usual route), "lattice" (0 off, 1 results also carry every lattice node,
    // 2 the same and the output text renders the nodes in place of the tokens), "lattice_margin" (-1 off; D in
    // 0 .. 2^62: the lattice keeps only the nodes within cost D of the best path, kernels.cuh MarginArgs),
    // "uncertainty" (0 off; with marginals on, 1 results also carry kEntropy / kLogPathProb, 2 also kPosOff /
    // kBoundaryProb, kernels.cuh UncertaintyArgs; k_small_batch and the eager small-batch copies step aside),
    // "posterior_text" (0 off; 1 with posterior decoding on: the output text renders the posterior path in place of
    // the best path; excludes lattice text and sample text).
    virtual void set_option(const std::string& name, long long value) = 0;
    // An output format (format.hpp) in place of "output_mode" 1-3, on every host route; nullptr switches it off.
    // Setting "output_mode" replaces it.  Builds the format's field table on the device.
    virtual void set_format(const FormatProgram* p) = 0;
    // The arrays a host result carries under the current options.
    virtual Outputs outputs() const = 0;
    // Marginal probabilities (kernels.cuh MargArgs) at temperature theta > 0 on every route except k_small_batch,
    // which steps aside while they are on; 0 switches them off.  Results then carry kTokenProb / kPathProb (and
    // kNodeProb with the lattice), and run_device leaves them in device memory (last_device).
    virtual void set_marginals(double theta) = 0;
    virtual double marginals() const = 0;
    virtual int lattice() const = 0;  // the option "lattice"
    // Segmentation sampling (kernels.cuh SampleArgs): n (1..1024) paths per sentence drawn from P(path) at temperature
    // theta (> 0, finite; the marginals' theta when they are on), with Philox keyed by seed; n = 0 switches it off.
    // On every route except k_small_batch, which steps aside.  Results then carry kSampleOff / kSamples, and
    // run_device leaves them in device memory (last_device).
    virtual void set_sampling(uint32_t n, double theta, uint64_t seed) = 0;
    virtual uint32_t sampling() const = 0;  // n, 0 when off
    // Posterior decoding (kernels.cuh PosteriorArgs) with weight gamma (>= 0, finite), which needs marginals on; off
    // switches it off.  On every route except k_small_batch and the eager small-batch copies, which step aside.
    // Results then carry kPostOff / kPostTokens / kPostProb / kPostGain, and run_device leaves them in device memory.
    virtual void set_posterior(bool on, double gamma) = 0;
    virtual bool posterior() const = 0;
    // Launch on a caller-owned CUDA stream (0 restores the engine's own stream).
    virtual void set_stream(uint64_t stream) = 0;
    virtual const float* stage_ms() const = 0;
    virtual uint64_t launch_count() const = 0;
    virtual const uint64_t* counters() const = 0;  // 10 entries, valid after a counted batch
    // ConnIdCounter (mapper.rs:87-104) accumulated since "connid_counting" was switched on, in the
    // dictionary's own connection ids: lid[num_left], rid[num_right].
    virtual void connid_counts(uint64_t* lid, uint64_t* rid, uint32_t* num_left, uint32_t* num_right) = 0;
};

// Restricts the calling thread to the CPUs of the NUMA node `device` is attached to (never beyond the process's
// own affinity mask); a no-op where sysfs does not say.
void pin_thread_to_device_numa_node(int device);

void* pinned_alloc(size_t n);
void pinned_free(void* p);

}  // namespace vbt
