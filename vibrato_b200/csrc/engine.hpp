// Device engine: owns the dictionary image in HBM, the per-batch workspace and the launch sequence.
#pragma once

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "format.hpp"
#include "host_dict.hpp"

namespace vbt {

struct HostResult {  // pinned host memory holding one batch's tokens
    uint64_t n_sent = 0, n_tokens = 0;
    uint64_t* tok_off = nullptr;  // n_sent + 1
    void* tokens = nullptr;       // vbt_token[n_tokens], or vbt_token16[n_tokens] when token_bytes == 16
    uint32_t token_bytes = 24;
    size_t cap_off = 0, cap_tok = 0;
    // output stage ("output_mode" option): the text `tokenize` prints for the batch and where each sentence's
    // part starts (n_sent + 1 offsets); text == nullptr when the stage is off
    uint64_t text_bytes = 0;
    uint64_t* text_off = nullptr;
    char* text = nullptr;
    size_t cap_text_off = 0, cap_text = 0;
    bool has_text = false;
    // marginals (set_marginals): per token and per sentence, has_marg == false when they are off
    float* token_prob = nullptr;  // n_tokens
    float* path_prob = nullptr;   // n_sent
    size_t cap_tprob = 0, cap_pprob = 0;
    bool has_marg = false;
    // lattice output (option "lattice" >= 1): every node of each sentence's lattice, has_lat == false when it is off.
    // node_off[i] .. node_off[i + 1] index sentence i's nodes (kernels.cuh LatticeArgs).
    uint64_t n_nodes = 0;
    uint64_t* node_off = nullptr;  // n_sent + 1
    void* nodes = nullptr;         // vbt_token[n_nodes], always 24 bytes
    void* links = nullptr;         // vbt_lattice_link[n_nodes]
    float* node_prob = nullptr;    // n_nodes, with marginals only (has_marg)
    size_t cap_node_off = 0, cap_nodes = 0, cap_links = 0, cap_nprob = 0;
    bool has_lat = false;
    // segmentation sampling (set_sampling): n_samp paths per sentence, has_samp == false when it is off.
    // sample_off[i * n_samp + j] .. sample_off[i * n_samp + j + 1] index sample j of sentence i (kernels.cuh SampleArgs).
    uint32_t n_samp = 0;
    uint64_t n_sample_tokens = 0;
    uint64_t* sample_off = nullptr;  // n_sent * n_samp + 1
    void* samples = nullptr;         // vbt_token[n_sample_tokens], always 24 bytes
    size_t cap_sample_off = 0, cap_samples = 0;
    bool has_samp = false;
};

// Required token boundaries of a batch (vbt_tokenize_batch_bounded): sentence i's boundaries are the
// sentence-relative byte offsets bnd[off[i] .. off[i+1]), and bnd holds n entries.  Host or device addresses, as the
// call that takes them says.  A null pointer to Bounds = an unbounded batch.
struct Bounds {
    const uint64_t* off = nullptr;  // n_sent + 1
    const uint32_t* bnd = nullptr;
    uint64_t n = 0;
};

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

    // Inputs/outputs in device memory; outputs owned by the engine until the next call.
    // With bnd: a bounded batch, its boundary arrays in device memory too.  Bounded batches refuse "counting".
    virtual void run_device(uint64_t d_utf8, uint64_t d_byte_off, uint64_t n_sent, uint64_t n_bytes,
                            uint64_t* d_tok_off, uint64_t* d_tokens, uint64_t* n_tokens, const Bounds* bnd = nullptr) = 0;
    // Inputs/outputs in host memory (copies inside); bnd in host memory.
    virtual HostResult* run_host(const char* utf8, const uint64_t* byte_off, uint64_t n_sent, const Bounds* bnd = nullptr) = 0;
    virtual void release(HostResult* r) = 0;

    // Building blocks of the multi-device engine (multi_engine.cu); a single-device caller never needs them.
    // run_shard: host sentences in, tokens left in this device's memory; returns their number (synchronises).
    // With src_device >= 0 `utf8` is a DEVICE address on that device (peer copy over NVLink) while byte_off is
    // still a host array.  With text_bytes != nullptr the shard's output text is formatted too ("output_mode";
    // *text_bytes = its size, 0 when the option is off).
    // bnd (host memory, may be null) holds the shard's n_sent + 1 boundary offsets.
    virtual uint64_t run_shard(const char* utf8, const uint64_t* byte_off, uint64_t n_sent, int src_device,
                               uint64_t* text_bytes, const Bounds* bnd = nullptr) = 0;
    // fetch_shard: the last shard's token offsets (+ tok_base, n_sent entries, one more when `last`) and token
    // records into host memory (pinned, or it is slow); with h_text_off != nullptr also its text offsets
    // (+ text_base, same count) and text, which run_shard must have formatted; with h_token_prob != nullptr also its
    // marginals (n_tokens and n_sent floats), which it must have computed.
    virtual void fetch_shard(uint64_t* h_tok_off, void* h_tokens, uint64_t tok_base, bool last, uint64_t* h_text_off,
                             char* h_text, uint64_t text_base, float* h_token_prob = nullptr, float* h_path_prob = nullptr) = 0;
    // Device addresses of the last shard's token offsets (uint64[n_sent + 1], already + tok_base after
    // rebase_shard) and token records.
    virtual void rebase_shard(uint64_t tok_base) = 0;
    virtual void shard_outputs(uint64_t* d_tok_off, uint64_t* d_tokens) const = 0;
    // Device addresses of the last shard's marginals: float token_prob[n_tokens], path_prob[n_sent].
    virtual void shard_marginals(uint64_t* d_token_prob, uint64_t* d_path_prob) const = 0;
    // The last shard's lattice (option "lattice"): its node count; fetch_shard_lattice copies its node offsets
    // (+ node_base, n_sent entries, one more when `last`), nodes, links and, with h_node_prob != nullptr, node marginals
    // into host memory; rebase_shard_lattice adds node_base to the offsets on the device and shard_lattice gives the
    // device addresses of the four arrays.
    virtual uint64_t shard_nodes() const = 0;
    virtual void fetch_shard_lattice(uint64_t* h_node_off, void* h_nodes, void* h_links, float* h_node_prob,
                                     uint64_t node_base, bool last) = 0;
    virtual void rebase_shard_lattice(uint64_t node_base) = 0;
    virtual void shard_lattice(uint64_t* d_node_off, uint64_t* d_nodes, uint64_t* d_links, uint64_t* d_node_prob) const = 0;
    // Sampling: set_sample_base gives the caller's index of the next run's first sentence (the i of the draws), so
    // that a shard draws what the whole batch would.  The last shard's sample-token count; fetch_shard_samples copies
    // its sample offsets (+ sample_base, n_sent * n entries, one more when `last`) and records into host memory;
    // rebase_shard_samples adds sample_base on the device and shard_samples_dev gives the two device addresses.
    virtual void set_sample_base(uint64_t first_sentence) = 0;
    virtual uint64_t shard_samples() const = 0;
    virtual void fetch_shard_samples(uint64_t* h_sample_off, void* h_samples, uint64_t sample_base, bool last) = 0;
    virtual void rebase_shard_samples(uint64_t sample_base) = 0;
    virtual void shard_samples_dev(uint64_t* d_sample_off, uint64_t* d_samples) const = 0;
    virtual int device() const = 0;
    virtual uint32_t token_bytes() const = 0;  // 24, or 16 with the "compact_tokens" option
    virtual std::string describe() const = 0;  // JSON: devices, how the dictionary travelled, ...

    virtual void set_counting(bool on) = 0;
    // Knobs: "lanes_per_sentence" (4/8/16/32), "sort_by_length" (0/1), "counting" (0/1), "chunk_sentences",
    // "dual_stream", "connid_counting", "output_mode" (0 none, 1 mecab, 2 wakati, 3 detail: run_host also
    // produces HostResult::text, on every host route; run_device stays token-only), "small_batch" (N > 0: run_host
    // takes k_small_batch for batches of at most N sentences and 16 KiB without counting; run_device and the shards
    // of a multi-device engine keep the usual route), "lattice" (0 off, 1 results also carry every lattice node,
    // 2 the same and the output text renders the nodes in place of the tokens).
    virtual void set_option(const std::string& name, long long value) = 0;
    // An output format (format.hpp) in place of "output_mode" 1-3, on every host route; nullptr switches it off.
    // Setting "output_mode" replaces it.  Builds the format's field table on the device.
    virtual void set_format(const FormatProgram* p) = 0;
    // Marginal probabilities (kernels.cuh MargArgs) at temperature theta > 0 on every route except k_small_batch,
    // which steps aside while they are on; 0 switches them off.  Results then carry HostResult::token_prob /
    // path_prob, and run_device leaves them in device memory (device_marginals).
    virtual void set_marginals(double theta) = 0;
    virtual double marginals() const = 0;
    virtual int lattice() const = 0;  // the option "lattice"
    // Segmentation sampling (kernels.cuh SampleArgs): n (1..1024) paths per sentence drawn from P(path) at temperature
    // theta (> 0, finite; the marginals' theta when they are on), with Philox keyed by seed; n = 0 switches it off.
    // On every route except k_small_batch, which steps aside.  Results then carry HostResult::sample_off / samples,
    // and run_device leaves them in device memory (device_samples).
    virtual void set_sampling(uint32_t n, double theta, uint64_t seed) = 0;
    virtual uint32_t sampling() const = 0;  // n, 0 when off
    // Device addresses of the last run_device's uint64 sample_off[n_sent * n + 1] and vbt_token samples[n_tokens];
    // valid until the next call.  Throws when that call ran without sampling.
    virtual void device_samples(uint64_t* d_sample_off, uint64_t* d_samples, uint64_t* n_tokens) const = 0;
    // Device addresses of the last run_device's float token_prob[n_tokens] and path_prob[n_sent]; valid until the
    // next call.  Throws when that call ran without marginals.
    virtual void device_marginals(uint64_t* d_token_prob, uint64_t* d_path_prob) const = 0;
    // Device addresses of the last run_device's lattice (option "lattice" >= 1): uint64 node_off[n_sent + 1],
    // vbt_token nodes[n_nodes], vbt_lattice_link links[n_nodes] and float node_prob[n_nodes] (0 without marginals);
    // valid until the next call.  Throws when that call ran without the lattice.
    virtual void device_lattice(uint64_t* d_node_off, uint64_t* d_nodes, uint64_t* d_links, uint64_t* d_node_prob,
                                uint64_t* n_nodes) const = 0;
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
