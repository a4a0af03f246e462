// Device engine of the batched Viterbi tokenizer: HBM workspace + launch sequence (one stream).
#include "engine.hpp"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include <algorithm>
#include <cmath>
#include <iterator>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "device_blob.hpp"
#include "kernels.cuh"

namespace vbt {

const char* const kStageNames =
    "count_chars,scan_slots,decode,candidates,scan_ends,viterbi,backtrack_count,scan_tokens,backtrack_write";

const InputError kInputErrors[kNumInputErrors] = {
    {kFlagBadOffsets, kInvalidArgument, kBadOffsetsMsg},
    {kFlagUtf8Error, kUtf8, kBadUtf8Msg},
    {kFlagBadBoundary, kInvalidArgument, kBadBoundsMsg},
    {kFlagBadSpan, kInvalidArgument, kBadSpansMsg},
};

namespace {

void cuda_check(cudaError_t e, const char* what) {
    if (e != cudaSuccess) {
        Status st = (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInvalidDevice) ? kNoDevice : kCuda;
        throw Error(st, std::string(what) + ": " + cudaGetErrorString(e));
    }
}
#define CK(x) cuda_check((x), #x)

// Throws the first input error (kInputErrors) that the flags of a finished attempt hold.
void throw_input_error(uint32_t flags) {
    for (const InputError& e : kInputErrors)
        if (flags & e.flag) throw Error(e.status, e.msg);
}

// The flag of each re-run reason (Rerun), and what a call reports when it persists.
constexpr uint32_t kRerunFlags[kNumReruns] = {kFlagPoolOverflow, kFlagSlotsOverflow, kFlagTextOverflow};
const char* const kRerunPersists[kNumReruns] = {"candidate pool overflow persists", "slot overflow persists",
                                                "text buffer overflow persists"};
// The flags that end an attempt without a result: an input error (kInputErrors) or a re-run reason.
constexpr uint32_t kFlagsEndAttempt = kFlagBadOffsets | kFlagUtf8Error | kFlagBadBoundary | kFlagBadSpan | kFlagPoolOverflow |
                                      kFlagSlotsOverflow | kFlagTextOverflow;

// A pooled host result that goes back to its pool unless release() hands it to the caller: an attempt that throws or
// runs again does not keep it.
struct ReturnTo {
    ResultPool* pool;
    void operator()(HostResult* r) const { pool->release(r); }
};
using PooledResult = std::unique_ptr<HostResult, ReturnTo>;

struct Control {  // one small block zeroed per batch and read back once
    unsigned long long pool_ctr;  // candidates
    unsigned long long seg_ctr;   // segments of the candidate pool
    unsigned long long counters[kNumCounters];
    unsigned long long total[kNumGroups];  // records of each output group in the batch (or chunk)
    uint32_t flags;
    uint32_t total_slots;
    uint32_t tickets[2];  // tile tickets of k_front and k_backtrack (TileScan)
};

// Entries the workspace must hold per batch: the segment pool and the lattice rows are sized from one learned count,
// and a batch needs it to cover both its candidates and its segments (almost always fewer).
static uint64_t pool_need(const Control& c) { return std::max<uint64_t>(c.pool_ctr, c.seg_ctr); }

static Totals totals(const Control& c) {
    Totals t;
    for (int g = 0; g < kNumGroups; ++g) t[g] = c.total[g];
    return t;
}

// Output iterator for the row-offset scan: writes {offset, offset} (an empty row) into the 8-byte row metadata so that
// no separate initialisation pass is needed.
struct RowMetaOut {
    uint2* p;
    struct Ref {
        uint2* q;
        __host__ __device__ Ref& operator=(uint32_t v) {
            *q = make_uint2(v, v);
            return *this;
        }
    };
    using iterator_category = std::random_access_iterator_tag;
    using value_type = uint32_t;
    using difference_type = ptrdiff_t;
    using pointer = void;
    using reference = Ref;
    __host__ __device__ Ref operator[](difference_type i) const { return Ref{p + i}; }
    __host__ __device__ Ref operator*() const { return Ref{p}; }
    __host__ __device__ RowMetaOut operator+(difference_type i) const { return RowMetaOut{p + i}; }
};

// A theta as an error message prints it: the shortest form that reads back as the same double.
static std::string num(double v) {
    char buf[32];
    for (int prec = 1; prec <= 17; ++prec) {
        std::snprintf(buf, sizeof buf, "%.*g", prec, v);
        if (std::strtod(buf, nullptr) == v) break;
    }
    return buf;
}

struct CastU64 {
    __host__ __device__ unsigned long long operator()(uint32_t v) const { return v; }
};
using CountsU64 = cub::TransformInputIterator<unsigned long long, CastU64, const uint32_t*>;  // u32 counts read as u64

__global__ void k_iota(uint32_t* v, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = i;
}

// Sentence order for K3: inside every tile of kOrderTile consecutive sentences, longest first.  K3 walks the
// sentences of a warp (and block) in lockstep, so neighbours of similar length waste fewer steps, while a tile
// stays small enough that the text and lattice rows of its sentences remain neighbours in memory (a global sort
// by length was measured to lose more through scattered accesses than it gained).
constexpr int kOrderTile = 256;
__global__ void __launch_bounds__(kOrderTile) k_local_order(const uint32_t* __restrict__ n_slots, uint32_t n_sent,
                                                          uint32_t* __restrict__ order) {
    __shared__ unsigned long long key[kOrderTile];
    const uint32_t i = blockIdx.x * kOrderTile + threadIdx.x;
    // descending length, ties by index: key = (~len) << 32 | index, sorted ascending; padding sorts last
    key[threadIdx.x] = i < n_sent ? ((unsigned long long)(~n_slots[i]) << 32) | i : ~0ull;
    __syncthreads();
    for (uint32_t k = 2; k <= kOrderTile; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            const uint32_t t = threadIdx.x, p = t ^ j;
            if (p > t) {
                const unsigned long long a = key[t], c = key[p];
                const bool up = (t & k) == 0;
                if ((a > c) == up) {
                    key[t] = c;
                    key[p] = a;
                }
            }
            __syncthreads();
        }
    }
    if (i < n_sent) order[i] = uint32_t(key[threadIdx.x]);  // the tile's valid entries come first
}

// ConnIdCounter totals += the counts of one finished attempt (see EngineImpl::connid_begin / connid_commit).
__global__ void k_add_u64(unsigned long long* dst, const unsigned long long* src, size_t n) {
    size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) dst[i] += src[i];
}

__global__ void k_publish_totals(const uint32_t* slot_off, const unsigned long long* tok_off, uint32_t n_sent, Control* c) {
    c->total_slots = slot_off[n_sent];
    c->total[kGroupTokens] = tok_off[n_sent];
}

// Chunked host batches: a group's offsets of a chunk become global by adding the group's records of all earlier
// chunks (kept in a device-resident running total so the host never has to wait for it).
__global__ void k_add_base(unsigned long long* tok_off, uint32_t n_plus_1, const unsigned long long* base) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_plus_1) tok_off[i] += *base;
}
__global__ void k_bump_base(unsigned long long* base, const unsigned long long* by) { *base += *by; }
__global__ void k_add_value(unsigned long long* tok_off, uint32_t n_plus_1, unsigned long long base) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_plus_1) tok_off[i] += base;
}

struct Workspace {  // every per-(chunk of a)-batch device array; two of them let consecutive chunks overlap
    DevBuf n_slots, slot_off, eos, n_tok, code_sys, code_usr, cinfo, groupable, byte_pos, info, info_ex, ends_cnt,
        ends_meta, seg, ends_hot, ends_cold, scan_tmp, stats, iota, sort_keys, order, tiles;
    DevBuf bnd_dist;  // bounded batches only: Batch::bnd_dist
    DevBuf span_tag;  // span batches only: SpanArgs::tag
    DevBuf m_fill, m_ncand, m_cand_entry, m_R, m_ab, m_r_eos, m_a_eos;  // marginals only: MargArgs
    DevBuf l_row_base, l_n_nodes;  // lattice output only: LatticeArgs
    DevBuf g_G, g_keep;            // near-best lattice only: MarginArgs::G / keep
    DevBuf m_lw, s_cnt, s_total;   // sampling only: MargArgs::lw, SampleArgs::cnt / total
    DevBuf p_V, p_A, p_cnt, p_total;  // posterior decoding only: PosteriorArgs (MargArgs::lw too)
    cudaStream_t stream = nullptr;
    void release() {
        for (DevBuf* b : {&n_slots, &slot_off, &eos, &n_tok, &code_sys, &code_usr, &cinfo, &groupable, &byte_pos, &info,
                          &info_ex, &ends_cnt, &ends_meta, &seg, &ends_hot, &ends_cold, &scan_tmp, &stats, &iota,
                          &sort_keys, &order, &tiles, &bnd_dist, &span_tag, &m_fill, &m_ncand, &m_cand_entry, &m_R, &m_ab, &m_r_eos, &m_a_eos,
                          &l_row_base, &l_n_nodes, &g_G, &g_keep, &m_lw, &s_cnt, &s_total, &p_V, &p_A, &p_cnt, &p_total})
            b->release();
    }
};

// The required boundaries of a batch (or chunk) in device memory: bnd_off[n_sent + 1] into bnd[n]; off == nullptr
// for an unbounded batch.
// A span batch also has the span records (span_off[n_sent + 1] into span_rec[n_spans]) and the compiled pattern table
// (shared by every chunk); its off is never nullptr (all zero without explicit boundaries).
struct DevBounds {
    const unsigned long long* off = nullptr;
    const uint32_t* bnd = nullptr;
    uint64_t n = 0;
    const unsigned long long* span_off = nullptr;
    const uint3* span_rec = nullptr;
    uint64_t n_spans = 0;
    const uint32_t* pat_off = nullptr;
    const uint3* pf = nullptr;
    const uint8_t* pat_bytes = nullptr;
    uint32_t n_pat = 0;
};

// What the output text renders in place of the tokens (options "lattice" = 2, "sample_text", "posterior_text"): at most
// one source replaces the best path.  Per source its name and option in the refusals, its offsets, records and their
// marginals (%pP), and the row of learned text ratios it sizes its text from.
enum TextSrc { kTextBest, kTextNodes, kTextPosterior, kTextSamples, kNumTextSrcs };
struct TextSrcInfo {
    const char *name, *off, *on;  // "<name> text", and how its option switches it off and on
    Array tok_off, tokens, prob;  // prob: kNumArrays = none (sample text refuses %pP)
    int ratio;                    // posterior text renders a path like the best one: it shares that ratio
};
constexpr TextSrcInfo kTextSrcs[kNumTextSrcs] = {
    {nullptr, nullptr, nullptr, kTokOff, kTokens, kTokenProb, 0},
    {"lattice", "\"lattice\" below 2", "lattice = 2", kNodeOff, kNodes, kNodeProb, 1},
    {"posterior", "\"posterior_text\" to 0", "posterior_text = 1", kPostOff, kPostTokens, kPostProb, 0},
    {"sample", "\"sample_text\" to 0", "sample_text = 1", kSampleOff, kSamples, kNumArrays, 2},
};
// Output text bytes expected per input byte (beyond text_per_sent_ per sentence) by [TextSrcInfo::ratio][output mode],
// before any is learned: the best path, lattice text (~17 nodes per token) and sample text (per rendering of a sentence).
constexpr int kTextRatios = 3;
using TextRatios = std::array<std::array<double, 5>, kTextRatios>;
constexpr TextRatios kTextPerByte = {{{0.0, 8.0, 2.0, 16.0, 8.0},
                                      {0.0, 8.0 * 17, 2.0 * 17, 16.0 * 17, 8.0 * 17},
                                      {0.0, 8.0, 2.0, 16.0, 8.0}}};

// The passes a batch runs between K3 and K4 and the host routes it may take, derived from the options (plan()).
struct PassPlan {
    FwdKind fwd;
    BwdKind bwd;                    // kBwdNone <=> marginals off
    bool bprob, margin, lat, post;  // k_boundary_probs (uncertainty 2), k_margin_backward, the lattice, posterior kernels
    uint32_t samp;                  // sampled paths per sentence, 0 = no sampling kernels
    bool small, eager;              // a small host batch may take k_small_batch / queue its copies behind the kernels
};

struct OutSlot {  // where one (chunk of a) batch leaves its results; two of them alternate in chunked runs
    DevBuf buf[kNumArrays];  // the output arrays; path_prob is written by the forward pass of sampling too
    DevBuf ctrl, sent_len;   // sent_len: output stage (k_format_*)
    DevBuf walk_off;         // sample text: where each walk's text starts (n_sent * n + 1)
    Outputs made;            // the arrays the (chunk of a) batch in this slot produced
    Control* h_ctrl = nullptr;
    cudaEvent_t ev[kNumStages + 1];
    cudaEvent_t done = nullptr, drained = nullptr;
    uint64_t launches = 0;
    uint32_t route = kRouteNone;  // ViterbiRoute as launched; resolved against h_ctrl->flags once `done`
};

class EngineImpl final : public Engine {
   public:
    EngineImpl(int device, const uint8_t* host_blob, uint64_t d_blob, uint64_t n_bytes, bool ignore_space,
               uint64_t max_grouping_len)
        : device_(device) {
        int count = 0;
        cudaError_t e = cudaGetDeviceCount(&count);
        if (e != cudaSuccess || count == 0)
            throw Error(kNoDevice, "no CUDA device available: the tokenizer has no CPU fallback");
        if (device < 0 || device >= count) throw Error(kInvalidArgument, "device ordinal out of range");
        CK(cudaSetDevice(device));
        CK(cudaStreamCreateWithFlags(&own_stream_, cudaStreamNonBlocking));
        stream_ = own_stream_;
        CK(cudaStreamCreateWithFlags(&in_stream_, cudaStreamNonBlocking));
        CK(cudaStreamCreateWithFlags(&out_stream_, cudaStreamNonBlocking));
        for (auto& o : out_) {
            for (auto& ev : o.ev) CK(cudaEventCreate(&ev));
            CK(cudaEventCreateWithFlags(&o.done, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&o.drained, cudaEventDisableTiming));
            o.ctrl.ensure(sizeof(Control));
            o.h_ctrl = static_cast<Control*>(pinned_alloc(sizeof(Control)));
        }
        CK(cudaEventCreateWithFlags(&in_done_, cudaEventDisableTiming));
        CK(cudaStreamCreateWithFlags(&aux_stream_, cudaStreamNonBlocking));
        for (auto& e : base_ready_) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        base_.ensure(kNumGroups * 8);
        BlobHeader h;
        if (host_blob) {
            if (n_bytes < sizeof(BlobHeader)) throw Error(kInvalidArgument, "dictionary image too small");
            std::memcpy(&h, host_blob, sizeof(h));
        } else {
            if (!d_blob || n_bytes < sizeof(BlobHeader)) throw Error(kInvalidArgument, "dictionary image too small");
            CK(cudaMemcpyAsync(&h, reinterpret_cast<const void*>(d_blob), sizeof(h), cudaMemcpyDeviceToHost, stream_));
            CK(cudaStreamSynchronize(stream_));
        }
        if (h.magic != kBlobMagic || h.total_bytes != n_bytes) throw Error(kInvalidArgument, "not a vibrato_b200 dictionary image");
        // k_viterbi2 addresses the connection matrix with a fixed high address word: the matrix must not cross a
        // 4 GiB boundary.  Where the allocation happens to straddle one, the image is placed again, shifted so that
        // the matrix starts on the boundary (at most one extra matrix of padding).
        const uint64_t m_bytes = h.connector_kind == 0 ? uint64_t(h.num_left) * h.num_right * 2 : 0;
        auto crosses = [&](uint64_t base) {
            return m_bytes && ((base + h.off_matrix) >> 32) != ((base + h.off_matrix + m_bytes - 1) >> 32);
        };
        const bool fits_window = m_bytes <= (1ull << 32);
        uint64_t shift = 0;
        if (host_blob || (fits_window && crosses(d_blob))) {
            blob_own_.ensure(n_bytes);
            if (fits_window && crosses(reinterpret_cast<uint64_t>(blob_own_.p))) {
                blob_own_.release();
                blob_own_.ensure(n_bytes + m_bytes + 512);
                const uint64_t base = reinterpret_cast<uint64_t>(blob_own_.p);
                if (crosses(base)) {  // the boundary lies inside the matrix: less than m_bytes ahead of its start
                    const uint64_t boundary = ((base + h.off_matrix) | 0xFFFFFFFFull) + 1;  // next multiple of 4 GiB
                    shift = (boundary - (base + h.off_matrix) + 255) & ~255ull;  // off_matrix is 256-byte aligned
                }
            }
            uint8_t* dst = static_cast<uint8_t*>(blob_own_.p) + shift;
            if (host_blob)
                CK(cudaMemcpyAsync(dst, host_blob, n_bytes, cudaMemcpyHostToDevice, stream_));
            else
                CK(cudaMemcpyAsync(dst, reinterpret_cast<const void*>(d_blob), n_bytes, cudaMemcpyDeviceToDevice, stream_));
            blob_ = dst;
        } else {
            blob_ = reinterpret_cast<const uint8_t*>(d_blob);
        }
        CK(cudaStreamSynchronize(stream_));
        dv_.matrix_window = (m_bytes && fits_window && !crosses(reinterpret_cast<uint64_t>(blob_))) ? 1 : 0;
        dv_.chr2inf = reinterpret_cast<const uint32_t*>(blob_ + h.off_chr2inf);
        dv_.chr2inf_len = h.chr2inf_len;
        dv_.sys_table = reinterpret_cast<const uint32_t*>(blob_ + h.off_sys_table);
        dv_.sys_table_len = h.sys_table_len;
        dv_.sys_nodes = reinterpret_cast<const uint4*>(blob_ + h.off_sys_nodes);
        dv_.sys_num_nodes = h.sys_num_nodes;
        dv_.sys_post = reinterpret_cast<const uint4*>(blob_ + h.off_sys_post);
        if (h.has_user) {
            dv_.usr_table = reinterpret_cast<const uint32_t*>(blob_ + h.off_usr_table);
            dv_.usr_table_len = h.usr_table_len;
            dv_.usr_nodes = reinterpret_cast<const uint4*>(blob_ + h.off_usr_nodes);
            dv_.usr_num_nodes = h.usr_num_nodes;
            dv_.usr_post = reinterpret_cast<const uint4*>(blob_ + h.off_usr_post);
        } else {
            dv_.usr_table = nullptr;
            dv_.usr_table_len = 0;
            dv_.usr_nodes = nullptr;
            dv_.usr_num_nodes = 0;
            dv_.usr_post = nullptr;
        }
        dv_.unk_off = reinterpret_cast<const uint32_t*>(blob_ + h.off_unk_off);
        dv_.unk_ent = reinterpret_cast<const uint2*>(blob_ + h.off_unk_ent);
        dv_.matrix = reinterpret_cast<const int16_t*>(blob_ + h.off_matrix);
        dv_.num_right = h.num_right;
        dv_.conn_stride_left = h.matrix_transposed ? 1 : h.num_right;
        dv_.conn_stride_right = h.matrix_transposed ? h.num_left : 1;
        dv_.connector_kind = h.connector_kind;
        for (int li = 0; li < 3; ++li) {
            dv_.feat_off[li] = reinterpret_cast<const uint32_t*>(blob_ + h.off_feat_off[li]);
            dv_.feat[li] = blob_ + h.off_feat[li];
            dv_.params[li] = reinterpret_cast<const uint2*>(blob_ + h.off_params[li]);
            dv_.n_words[li] = h.n_words[li];
        }
        dv_.right_conn = dv_.left_conn = nullptr;
        if (h.connector_kind == 1 || h.connector_kind == 2) {
            dv_.right_feats = reinterpret_cast<const uint32_t*>(blob_ + h.off_right_feats);
            dv_.left_feats = reinterpret_cast<const uint32_t*>(blob_ + h.off_left_feats);
            dv_.feat_T = h.feat_T;
            dv_.sc_bases = reinterpret_cast<const uint32_t*>(blob_ + h.off_bases);
            dv_.sc_checks = reinterpret_cast<const uint32_t*>(blob_ + h.off_checks);
            dv_.sc_costs = reinterpret_cast<const int32_t*>(blob_ + h.off_costs);
            dv_.n_bases = h.n_bases;
            dv_.n_checks = h.n_checks;
            if (h.connector_kind == 2) {
                if (h.feat_T != 8) throw Error(kDecode, "dual connector image: the raw term must be 8 lanes wide");
                dv_.num_right = h.m_num_right;
                dv_.right_conn = reinterpret_cast<const uint16_t*>(blob_ + h.off_right_conn);
                dv_.left_conn = reinterpret_cast<const uint16_t*>(blob_ + h.off_left_conn);
            }
        } else if (h.connector_kind != 0) {
            throw Error(kUnsupported, "dictionary image with an unknown connector kind");
        }
        num_left_ = h.num_left;
        num_right_ = h.num_right;
        left_ids_.resize(h.num_left);
        right_ids_.resize(h.num_right);
        CK(cudaMemcpy(left_ids_.data(), blob_ + h.off_left_ids, size_t(h.num_left) * 2, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(right_ids_.data(), blob_ + h.off_right_ids, size_t(h.num_right) * 2, cudaMemcpyDeviceToHost));
        if (ignore_space) {  // Tokenizer::ignore_space tokenizer.rs:42-55
            if (h.space_cate_id < 0)
                throw Error(kInvalidArgument, "dict: SPACE is not defined in the input dictionary (i.e., char.def).");
            dv_.space_mask = 1u << (h.space_cate_id & 31);  // release-build `1 << id`
        } else {
            dv_.space_mask = 0;
        }
        dv_.max_grouping = max_grouping_len ? max_grouping_len : ~0ull;  // tokenizer.rs:67-74
        std::memset(stage_ms_, 0, sizeof(stage_ms_));
        std::memset(counters_, 0, sizeof(counters_));
    }

    ~EngineImpl() override {
        cudaSetDevice(device_);
        cudaStreamSynchronize(stream_);
        cudaStreamSynchronize(in_stream_);
        cudaStreamSynchronize(out_stream_);
        for (auto& o : out_) {
            for (DevBuf& b : o.buf) b.release();
            o.ctrl.release();
            o.sent_len.release();
            o.walk_off.release();
            pinned_free(o.h_ctrl);
            for (auto& ev : o.ev) cudaEventDestroy(ev);
            cudaEventDestroy(o.done);
            cudaEventDestroy(o.drained);
        }
        for (int i = 0; i < kRingSlots; ++i) {
            if (ring_[i]) pinned_free(ring_[i]);
            if (ring_ev_[i]) cudaEventDestroy(ring_ev_[i]);
        }
        cudaEventDestroy(in_done_);
        cudaStreamDestroy(in_stream_);
        cudaStreamDestroy(out_stream_);
        base_.release();
        for (DevBuf* b : {&fmt_prog_, &ft_keep_, &ft_off_, &ft_bytes_}) b->release();
        for (auto* b : {&blob_own_, &in_utf8_, &in_off_, &in_bnd_off_, &in_bnd_, &in_span_off_, &in_span_, &in_pat_, &connid_,
                        &connid_try_})
            b->release();
        for (auto& w : ws_) w.release();
        ws_small_.release();
        small_in_.release();
        small_out_.release();
        pinned_free(small_in_h_);
        pinned_free(small_out_h_);
        pinned_free(bnd_stage_);
        cudaStreamSynchronize(aux_stream_);
        cudaStreamDestroy(aux_stream_);
        for (auto& e : base_ready_) cudaEventDestroy(e);
        cudaStreamDestroy(own_stream_);
    }

    void set_counting(bool on) override { counting_ = on; }
    void set_option(const std::string& name, long long value) override {
        if (name == "lanes_per_sentence") {
            if (value != 4 && value != 8 && value != 16 && value != 32)
                throw Error(kInvalidArgument, "lanes_per_sentence must be 4, 8, 16 or 32");
            lanes_ = int(value);
        } else if (name == "sort_by_length") {
            if (value < 0 || value > 2) throw Error(kInvalidArgument, "sort_by_length must be 0 (off), 1 (whole batch) or 2 (tiles)");
            order_mode_ = int(value);
        } else if (name == "connid_counting") {
            // Worker::init_connid_counter (worker.rs:77-83) when switched on; every batch tokenised
            // while it is on is followed by update_connid_counts (worker.rs:90-93)
            cudaStreamSynchronize(stream_);
            connid_on_ = value != 0;
            if (connid_on_) {
                connid_.ensure((size_t(num_left_) + num_right_) * 8);
                connid_try_.ensure((size_t(num_left_) + num_right_) * 8);
                CK(cudaMemset(connid_.p, 0, (size_t(num_left_) + num_right_) * 8));
            }
        } else if (name == "compact_tokens") {
            // 16-byte token records {start_byte, end_byte, word_idx, total_cost}: a third less to bring back over PCIe;
            // the character range of a token is recomputed by the caller from its own UTF-8 (vbt_result_view_compact)
            if (value != 0 && output_mode_ != kOutNone) throw Error(kInvalidArgument, "compact_tokens and output_mode exclude each other");
            cudaStreamSynchronize(stream_);
            tok_bytes_ = value ? 16 : 24;
        } else if (name == "output_mode") {
            if (value < 0 || value > 3) throw Error(kInvalidArgument, "output_mode must be 0 (off), 1 mecab, 2 wakati or 3 detail");
            if (value != 0 && tok_bytes_ != 24) throw Error(kInvalidArgument, "compact_tokens and output_mode exclude each other");
            clear_format();  // a fixed mode replaces an output format
            output_mode_ = uint32_t(value);
        } else if (name == "dual_stream") {
            dual_stream_ = value != 0;
        } else if (name == "chunk_sentences") {
            if (value < 0 || value > 0x7FFFFFFF) throw Error(kInvalidArgument, "chunk_sentences out of range");
            chunk_sentences_ = uint32_t(value);  // 0 disables the chunked host pipeline
        } else if (name == "pool_estimate_permille") {
            // candidates expected per input byte (x 1000): the pool of segments and the candidate rows are both
            // sized from it (the larger of the two counts is learned), and a batch that overflows either is re-run
            // with the exact size.  Tests set it low to walk that path.
            if (value < 1 || value > 1000000) throw Error(kInvalidArgument, "pool_estimate_permille out of range");
            cand_per_byte_ = double(value) / 1000.0;
        } else if (name == "chars_estimate_permille") {
            // characters expected per input byte (x 1000) for sizing the per-character launches; tests set it low
            if (value < 1 || value > 1000) throw Error(kInvalidArgument, "chars_estimate_permille out of range");
            chars_per_byte_ = double(value) / 1000.0;
        } else if (name == "viterbi_kernel") {
            if (value < 0 || value > 2) throw Error(kInvalidArgument, "viterbi_kernel must be 0, 1 or 2");
            viterbi_kernel_ = int(value);
        } else if (name == "counting") {
            counting_ = value != 0;
        } else if (name == "lattice") {
            // every lattice node next to the tokens (1), and in place of them in the output text (2)
            if (value < 0 || value > 2) throw Error(kInvalidArgument, "lattice must be 0 (off), 1 (nodes) or 2 (nodes, and the text renders them)");
            set_text(kTextNodes, value == 2);
            lattice_ = value != 0;
        } else if (name == "lattice_margin") {
            // the lattice keeps the nodes of the paths within cost D of the best one (-1: every node)
            if (value < -1 || value > kMaxLatticeMargin)
                throw Error(kInvalidArgument, "lattice_margin must be -1 (off) or a cost margin between 0 and 2^62");
            cudaStreamSynchronize(stream_);
            lat_margin_ = value;
        } else if (name == "uncertainty") {
            // each sentence's path entropy and best-path log-probability (1), and each position's boundary probability (2)
            if (value < 0 || value > 2)
                throw Error(kInvalidArgument, "uncertainty must be 0 (off), 1 (entropy and log_path_prob) or 2 (also boundary probabilities)");
            if (value != 0 && theta_ == 0)
                throw Error(kInvalidArgument, "uncertainty needs marginals: switch them on with set_marginals before setting it");
            cudaStreamSynchronize(stream_);
            unc_ = uint32_t(value);
        } else if (name == "sample_text") {
            // the output text renders each sentence's samples in place of its best path
            if (value < 0 || value > 1) throw Error(kInvalidArgument, "sample_text must be 0 (off) or 1 (the text renders the samples)");
            set_text(kTextSamples, value != 0);
        } else if (name == "posterior_text") {
            // the output text renders each sentence's posterior path in place of its best path
            if (value < 0 || value > 1) throw Error(kInvalidArgument, "posterior_text must be 0 (off) or 1 (the text renders the posterior path)");
            set_text(kTextPosterior, value != 0);
        } else if (name == "sample_base") {
            // the sentence index of the draws starts here: a caller that splits a corpus over calls keeps its draws
            if (value < 0 || value > kMaxSampleBase) throw Error(kInvalidArgument, "sample_base must be between 0 and 2^32");
            sample_base_ = uint64_t(value);
        } else if (name == "small_batch") {
            // host batches of at most `value` sentences and kEagerBytes bytes take k_small_batch (0 = never)
            if (value < 0 || value > kSmallBatchMax) throw Error(kInvalidArgument, "small_batch must be between 0 and 65536");
            small_batch_ = uint32_t(value);
        } else {
            throw Error(kInvalidArgument, "unknown option: " + name);
        }
    }
    void set_format(const FormatProgram* p) override {
        CK(cudaSetDevice(device_));
        clear_format();
        if (!p) return;
        if (tok_bytes_ != 24) throw Error(kInvalidArgument, "compact_tokens and output formats exclude each other");
        if ((p->uses & kUsesProb) && theta_ == 0)
            throw Error(kInvalidArgument, "%pP needs marginals: switch them on before setting the format");
        if ((p->uses & kUsesBest) && text_src_ != kTextNodes)
            throw Error(kInvalidArgument, "%pb needs lattice text: set the option \"lattice\" to 2 before setting the format");
        if ((p->uses & kUsesPrev) && text_src_ == kTextNodes)  // compile_format names the directive; this guards other callers
            throw Error(kInvalidArgument, "lattice text has no previous token: the format may not print %M %pS %pn %pC %pL");
        if ((p->uses & (kUsesProb | kUsesBest)) && text_src_ == kTextSamples)  // the same
            throw Error(kInvalidArgument, "sample text has no marginals or best-path flags: the format may not print %pP or %pb");
        try {
            fmt_prog_.ensure(sizeof(FormatProgram));
            CK(cudaMemcpy(fmt_prog_.p, p, sizeof(FormatProgram), cudaMemcpyHostToDevice));
            if (p->n_fields) build_field_table(*p);
        } catch (...) {
            clear_format();
            throw;
        }
        output_mode_ = kOutFormat;
        fmt_uses_ = p->uses;
        text_per_sent_ = p->per_sentence;
        for (int s = 0; s < kTextRatios; ++s) text_per_byte_[s][kOutFormat] = kTextPerByte[s][kOutFormat];  // learned anew
    }
    void set_marginals(double theta) override {
        if (!(theta >= 0) || !std::isfinite(theta))
            throw Error(kInvalidArgument, "the marginals' theta must be a finite number >= 0 (0 switches them off)");
        if (theta == 0 && output_mode_ == kOutFormat && (fmt_uses_ & kUsesProb))
            throw Error(kInvalidArgument, "the output format prints %pP: change the format before switching marginals off");
        if (theta == 0 && unc_)
            throw Error(kInvalidArgument, "uncertainty needs marginals: set the option \"uncertainty\" to 0 before switching marginals off");
        if (theta == 0 && post_)
            throw Error(kInvalidArgument, "posterior decoding needs marginals: switch it off with set_posterior before switching marginals off");
        if (theta > 0 && samp_n_ && theta != samp_theta_)
            throw Error(kInvalidArgument, "marginals and sampling share one forward pass: the marginals' theta " + num(theta) +
                                              " differs from the sampling theta " + num(samp_theta_));
        cudaStreamSynchronize(stream_);
        theta_ = theta;
    }
    void set_sampling(uint32_t n, double theta, uint64_t seed) override {
        if (n > kMaxSamples) throw Error(kInvalidArgument, "sampling: n must be between 0 (off) and 1024");
        if (n && (!(theta > 0) || !std::isfinite(theta)))
            throw Error(kInvalidArgument, "sampling: theta must be a finite number > 0");
        if (n && theta_ > 0 && theta != theta_)
            throw Error(kInvalidArgument, "marginals and sampling share one forward pass: the sampling theta " + num(theta) +
                                              " differs from the marginals' theta " + num(theta_));
        if (!n && text_src_ == kTextSamples)
            throw Error(kInvalidArgument, "the output text renders the samples: set \"sample_text\" to 0 before switching sampling off");
        cudaStreamSynchronize(stream_);
        samp_n_ = n;
        samp_theta_ = n ? theta : 0.0;
        samp_seed_ = seed;
    }
    uint32_t sampling() const override { return samp_n_; }
    void set_posterior(bool on, double gamma) override {
        if (on && (!(gamma >= 0) || !std::isfinite(gamma)))
            throw Error(kInvalidArgument, "posterior decoding: gamma must be a finite number >= 0");
        if (on && theta_ == 0)
            throw Error(kInvalidArgument, "posterior decoding needs marginals: switch them on with set_marginals first");
        if (!on && text_src_ == kTextPosterior)
            throw Error(kInvalidArgument, "the output text renders the posterior path: set \"posterior_text\" to 0 before switching posterior decoding off");
        cudaStreamSynchronize(stream_);
        post_ = on;
        post_g1_ = on ? gamma + 1.0 : 0.0;
    }
    bool posterior() const override { return post_; }
    double marginals() const override { return theta_; }
    int lattice() const override { return text_src_ == kTextNodes ? 2 : lattice_; }
    Outputs outputs() const override {
        return Outputs{tok_bytes_, samp_n_, theta_ > 0, output_mode_ != kOutNone, lattice_ != 0, lat_margin_ >= 0, unc_, post_};
    }
    const DeviceOutputs& last_device() const override { return last_; }
    void set_stream(uint64_t stream) override {
        cudaStreamSynchronize(stream_);
        stream_ = stream ? reinterpret_cast<cudaStream_t>(stream) : own_stream_;
    }
    const float* stage_ms() const override { return stage_ms_; }
    uint64_t launch_count() const override { return launches_; }
    const uint64_t* counters() const override { return counters_; }
    void connid_counts(uint64_t* lid, uint64_t* rid, uint32_t* num_left, uint32_t* num_right) override {
        if (num_left) *num_left = num_left_;
        if (num_right) *num_right = num_right_;
        if (!lid || !rid) return;
        if (!connid_.p) throw Error(kInvalidArgument, "connid counting was never switched on");
        CK(cudaSetDevice(device_));
        std::vector<unsigned long long> raw(size_t(num_left_) + num_right_);
        CK(cudaMemcpy(raw.data(), connid_.p, raw.size() * 8, cudaMemcpyDeviceToHost));
        for (uint32_t i = 0; i < num_left_; ++i) lid[left_ids_[i]] = raw[i];
        for (uint32_t i = 0; i < num_right_; ++i) rid[right_ids_[i]] = raw[num_left_ + i];
    }

    void run_device(uint64_t d_utf8, uint64_t d_byte_off, uint64_t n_sent, uint64_t n_bytes, const Bounds* bnd) override {
        last_ = DeviceOutputs{};
        reruns_ = Reruns{};
        CK(cudaSetDevice(device_));
        check_size(n_sent, n_bytes);
        check_bounded(bnd);
        Bounds nb;
        if (bnd) {  // no boundary and no span at all: the unbounded kernels
            nb = *bnd;
            if (nb.spans.off && nb.spans.n == 0 && device_offsets_zero(nb.spans.off, n_sent)) nb.spans = Spans{};
            if (nb.off && nb.n == 0 && device_offsets_zero(nb.off, n_sent)) nb.off = nullptr;
            bnd = (nb.off || nb.spans.off) ? &nb : nullptr;
        }
        DevBounds bd;
        if (bnd) {
            if (bnd->off)
                bd = DevBounds{reinterpret_cast<const unsigned long long*>(bnd->off), bnd->bnd, bnd->n};
            else
                bd.off = zero_offsets(uint32_t(n_sent), stream_);
            if (bnd->spans.off) {
                bd.span_off = reinterpret_cast<const unsigned long long*>(bnd->spans.off);
                bd.span_rec = reinterpret_cast<const uint3*>(bnd->spans.rec);
                bd.n_spans = bnd->spans.n;
                upload_patterns(bnd->spans, bd, stream_);
            }
        }
        run_whole(reinterpret_cast<const uint8_t*>(d_utf8), reinterpret_cast<const unsigned long long*>(d_byte_off),
                  uint32_t(n_sent), n_bytes, bd);
        keep_device_outputs();
    }

    // Host path.  Large batches are cut into chunks that flow through three streams: the H2D copy of
    // chunk i+1 and the D2H copy of chunk i-1 overlap the kernels of chunk i (PCIe is full duplex).
    HostResult* run_host(const char* utf8, const uint64_t* byte_off, uint64_t n_sent64, const Bounds* bnd) override {
        reruns_ = Reruns{};
        CK(cudaSetDevice(device_));
        Bounds nb;
        const HostWindow hw = host_window(byte_off, n_sent64, bnd, nb);
        const uint64_t first = hw.first, n_bytes = hw.n_bytes;
        const uint64_t* off = hw.off;
        bnd = hw.bnd;
        const uint32_t n_sent = uint32_t(n_sent64);
        const uint8_t* d_utf8 = in_utf8_.as<uint8_t>();
        const unsigned long long* d_off = in_off_.as<unsigned long long>();
        const bool utf8_pinned = n_bytes == 0 || is_pinned(utf8 + first);
        const bool off_pinned = off != byte_off || is_pinned(byte_off);  // rebased_ is ours (pageable, small)
        const uint32_t chunk = chunk_sentences_;
        const bool chunked = chunk > 0 && n_sent > chunk + chunk / 2;
        const bool fmt = output_mode_ != kOutNone;
        const PassPlan p = plan();
        if (p.small && n_sent <= small_batch_ && !chunked && n_bytes <= kEagerBytes &&
            (!bnd || (!bnd->spans.off && small_bounds_fit(*bnd, n_sent)))) {  // k_small_batch has no span rules
            if (HostResult* r = run_small(utf8 + first, off, n_sent, n_bytes, bnd)) return r;
            // the batch outgrew the scratch of k_small_batch: it runs again on the route below
        }
        const DevBounds bd = bnd ? upload_bounds(*bnd, n_sent, stream_) : DevBounds{};
        for (int attempt = 0;; ++attempt) {
            if (!chunked) {
                h2d(in_off_.p, off, (size_t(n_sent) + 1) * 8, stream_, off_pinned && off == byte_off);
                h2d(in_utf8_.p, utf8 + first, n_bytes, stream_, utf8_pinned);
                if (p.eager && n_bytes <= kEagerBytes) {
                    // Small batches (a per-sentence Worker loop ends up here) are all latency: the result copies are
                    // queued behind the kernels with an upper bound for the token count (a token spans >= 1 byte), so
                    // that the call makes ONE host synchronisation instead of two.
                    PooledResult r(pool_.acquire(outputs(), n_sent, Totals{n_bytes, 0, 0, 0}), ReturnTo{&pool_});
                    run_whole(d_utf8, d_off, n_sent, n_bytes, bd, 0, r.get());
                    r->total[kGroupTokens] = out_[0].h_ctrl->total[kGroupTokens];
                    return r.release();
                }
                run_whole(d_utf8, d_off, n_sent, n_bytes, bd);
                if (fmt) format_whole(d_utf8, d_off, n_sent);
                OutSlot& o = out_[0];
                PooledResult r(pool_.acquire(outputs(), n_sent, totals(*o.h_ctrl)), ReturnTo{&pool_});
                place(o, r.get(), 0, n_sent, r->total, Totals{}, true, stream_);
                CK(cudaStreamSynchronize(stream_));
                return r.release();
            }
            // ---- chunked, pipelined -------------------------------------------------------------
            // Chunk plan: a small first chunk (its H2D copy is the pipeline's fill), then halving sizes
            // down to a small last chunk (its D2H copy is the drain); big middle chunks keep the
            // kernels efficient.
            std::vector<uint32_t> bounds{0};
            {
                const uint32_t lo = std::max<uint32_t>(1024, chunk / 2);
                bounds.push_back(std::min(n_sent, lo));
                while (bounds.back() < n_sent) {
                    uint32_t rest = n_sent - bounds.back();
                    uint32_t take = rest <= lo + lo / 2 ? rest : std::max(lo, rest / 2);
                    bounds.push_back(bounds.back() + take);
                }
            }
            const uint32_t n_chunks = uint32_t(bounds.size()) - 1;
            uint64_t max_chunk_bytes = 0;
            uint32_t max_chunk_sent = 0;
            for (uint32_t c = 0; c < n_chunks; ++c) {
                max_chunk_bytes = std::max(max_chunk_bytes, off[bounds[c + 1]] - off[bounds[c]]);
                max_chunk_sent = std::max(max_chunk_sent, bounds[c + 1] - bounds[c]);
            }
            ws_[0].stream = stream_;
            ws_[1].stream = aux_stream_;
            // sized once: no cudaMalloc in the pipeline
            const size_t cands = want_cand(max_chunk_bytes);
            const uint32_t n_ws = dual_stream_ ? 2 : 1;
            for (uint32_t i = 0; i < n_ws; ++i)
                ensure_workspace(ws_[i], max_chunk_sent, max_chunk_bytes, cands, bd.off != nullptr, bd.span_off != nullptr);
            for (int i = 0; i < 2; ++i) {  // chunk c runs in slot c & 1 and workspace c & 1 (dual_stream) or 0
                ensure_out(out_[i], max_chunk_sent, max_chunk_bytes);
                ensure_entries(ws_[dual_stream_ ? i : 0], out_[i], cands + max_chunk_sent + 1);
            }
            // output stage: each slot's text buffer holds the text a chunk is expected to produce (at most 4 bytes per
            // sentence plus the learned ratio per input byte); a chunk with more text flags itself and the batch is
            // re-run with the ratio it measured
            // (sample text: n renderings per sentence, the ratio learned per rendering)
            const uint32_t renders = text_view(out_[0]).units;
            const double text_ratio = text_ratio_ref() * renders;
            const uint64_t per_sent = uint64_t(text_per_sent_) * renders;
            if (fmt)
                for (int i = 0; i < 2; ++i) {
                    ensure_format(out_[i], ws_[dual_stream_ ? i : 0], max_chunk_sent);
                    out_[i].buf[kText].ensure(size_t(double(max_chunk_bytes) * text_ratio) + size_t(max_chunk_sent) * per_sent + 4096);
                }
            // a pinned result sized from the learned ratios per input byte (grown below if short)
            PooledResult pr(pool_.acquire(outputs(), n_sent,
                                          Totals{uint64_t(double(n_bytes) * tok_per_byte_) + 1024,
                                                 uint64_t(double(n_bytes) * text_ratio) + uint64_t(n_sent) * per_sent + 1024,
                                                 uint64_t(double(n_bytes) * node_per_byte_) + 1024,
                                                 uint64_t(double(n_bytes) * tok_per_byte_ * samp_n_) + 1024,
                                                 uint64_t(double(n_bytes) * chars_per_byte_) + n_sent + 1024,
                                                 uint64_t(double(n_bytes) * tok_per_byte_) + 1024}),
                            ReturnTo{&pool_});
            HostResult* r = pr.get();
            CK(cudaMemsetAsync(base_.p, 0, kNumGroups * 8, stream_));
            connid_begin(stream_);
            h2d(in_off_.p, off, (size_t(n_sent) + 1) * 8, stream_, off_pinned && off == byte_off);
            CK(cudaEventRecord(in_done_, stream_));
            CK(cudaStreamWaitEvent(in_stream_, in_done_, 0));
            CK(cudaStreamWaitEvent(aux_stream_, in_done_, 0));
            clear_stats();
            Totals sum{};  // records per group of the chunks drained so far
            double text_need = 0;  // text bytes per input byte beyond per_sent per sentence, largest over the sound chunks
            uint32_t route = kRouteNone;
            uint32_t seen = 0;       // the flags of the chunks drained so far
            uint64_t pool_most = 0;  // pool_need of the largest chunk
            uint64_t slots_seen = 0;
            batch_total_bytes_ = n_bytes;
            std::vector<cudaEvent_t>& h2d_ev = h2d_events(n_chunks);
            auto issue_h2d = [&](uint32_t c) {
                uint32_t s0 = bounds[c], s1 = bounds[c + 1];
                uint64_t b0 = off[s0], b1 = off[s1];
                h2d(in_utf8_.as<uint8_t>() + b0, utf8 + first + b0, b1 - b0, in_stream_, utf8_pinned);
                CK(cudaEventRecord(h2d_ev[c], in_stream_));
            };
            // pinned input: every H2D copy is queued up front on its own stream.  Pageable input is staged by
            // this thread, one chunk ahead of the kernels (the staging of chunk c + 1 overlaps the kernels of c).
            if (utf8_pinned)
                for (uint32_t c = 0; c < n_chunks; ++c) issue_h2d(c);
            else
                issue_h2d(0);
            auto drain = [&](uint32_t c) {  // wait for chunk c's kernels, then queue its D2H copies
                OutSlot& o = out_[c & 1];
                uint32_t s0 = bounds[c], s1 = bounds[c + 1];
                CK(cudaEventSynchronize(o.done));
                seen |= o.h_ctrl->flags;
                slots_seen += o.h_ctrl->total_slots;
                // chunks share one static route; a chunk holding a very long sentence takes the unpruned twin
                route = std::max(route, add_stats(o));
                pool_most = std::max<uint64_t>(pool_most, pool_need(*o.h_ctrl));
                const Totals count = totals(*o.h_ctrl);
                if (fmt && !(o.h_ctrl->flags & (kFlagsStandDown | kFlagUtf8Error | kFlagPoolOverflow)))
                    text_need = std::max(text_need, (double(count[kGroupText]) - double(per_sent) * (s1 - s0)) /
                                                        double(std::max<uint64_t>(1, off[s1] - off[s0])));
                if (!(seen & kFlagsEndAttempt)) {  // else nothing of the attempt is kept: it throws or runs again
                    // offsets are global already (base_); a record array that is short grows (rare), keeping what it
                    // holds once the copies into it have landed
                    for (int a = 0; a < kNumArrays; ++a) {
                        if (!r->out.has(a) || kArrays[a].kind != kRecords) continue;
                        const uint64_t keep = r->out.at(a, 0, sum), need = keep + r->out.bytes(a, 0, count, false);
                        if (need <= r->buf[a].cap) continue;
                        CK(cudaStreamSynchronize(out_stream_));
                        r->buf[a].grow(need, keep);
                    }
                    place(o, r, s0, s1 - s0, count, sum, s1 == n_sent, out_stream_);
                }
                CK(cudaEventRecord(o.drained, out_stream_));
                for (int g = 0; g < kNumGroups; ++g) sum[g] += count[g];
            };
            for (uint32_t c = 0; c < n_chunks; ++c) {
                OutSlot& o = out_[c & 1];
                uint32_t s0 = bounds[c], s1 = bounds[c + 1];
                // "dual_stream": chunks alternate between two workspaces / compute streams so that the head
                // of chunk c+1 can fill SMs left idle by the tail of chunk c; off by default, since the
                // concurrent kernels contend for the same L1/L2
                Workspace& w = ws_[dual_stream_ ? (c & 1) : 0];
                CK(cudaStreamWaitEvent(w.stream, h2d_ev[c], 0));
                if (c >= 2) CK(cudaStreamWaitEvent(w.stream, o.drained, 0));  // slot reused: its D2H must be done
                DevBounds cb = bd;  // the chunk's slice of the boundary offsets (they index the whole bnd array)
                if (cb.off) cb.off += s0;
                if (cb.span_off) cb.span_off += s0;
                enqueue(w, d_utf8, d_off + s0, s1 - s0, off[s1] - off[s0], o, base_.as<unsigned long long>(),
                        c >= 1 ? base_ready_[(c - 1) & 1] : nullptr, base_ready_[c & 1], cb, s0);
                if (!utf8_pinned && c + 1 < n_chunks) issue_h2d(c + 1);
                if (c >= 1) drain(c - 1);
            }
            drain(n_chunks - 1);
            CK(cudaStreamSynchronize(out_stream_));
            CK(cudaStreamSynchronize(in_stream_));
            CK(cudaStreamSynchronize(aux_stream_));
            CK(cudaStreamSynchronize(stream_));
            throw_input_error(seen);
            if (rerun(seen, attempt)) {
                if (seen & kFlagSlotsOverflow) chars_per_byte_ = 1.0;
                if (seen & (kFlagPoolOverflow | kFlagSlotsOverflow))
                    cand_per_byte_ = std::max(cand_per_byte_ * 1.5, double(pool_most) / double(std::max<uint64_t>(1, max_chunk_bytes)) * 1.2);
                if (seen & kFlagTextOverflow) text_ratio_ref() = std::max(text_ratio * 1.5, text_need * 1.05) / renders;
                continue;
            }
            if (max_chunk_bytes)
                cand_per_byte_ = std::max(0.25, double(pool_most) / double(max_chunk_bytes) * 1.25);
            if (n_bytes) tok_per_byte_ = std::max(0.02, double(sum[kGroupTokens]) / double(n_bytes) * 1.1);
            if (n_bytes) chars_per_byte_ = std::min(1.0, double(slots_seen - n_sent) / double(n_bytes) * 1.10);
            if (fmt) text_ratio_ref() = std::max(0.5, text_need * 1.25 / renders);
            if (n_bytes && lattice_) node_per_byte_ = std::max(0.1, double(sum[kGroupLattice]) / double(n_bytes) * 1.1);
            connid_commit(stream_);
            last_route_ = route;
            r->total = sum;
            return pr.release();
        }
    }

    void release(HostResult* r) override { pool_.release(r); }

    // ---- shard-level entry points (multi_engine.cu) -------------------------------------------------
    Totals run_shard(const char* utf8, const uint64_t* byte_off, uint64_t n_sent64, int src_device, uint64_t first_sentence,
                     bool with_text, const Bounds* bnd) override {
        last_ = DeviceOutputs{};
        reruns_ = Reruns{};
        CK(cudaSetDevice(device_));
        Bounds nb;
        const HostWindow hw = host_window(byte_off, n_sent64, bnd, nb);
        const uint64_t first = hw.first, n_bytes = hw.n_bytes;
        const uint32_t n_sent = uint32_t(n_sent64);
        const DevBounds bd = hw.bnd ? upload_bounds(*hw.bnd, n_sent, stream_) : DevBounds{};
        h2d(in_off_.p, hw.off, (size_t(n_sent) + 1) * 8, stream_, hw.off == byte_off && is_pinned(byte_off));
        if (n_bytes) {
            if (src_device >= 0 && src_device != device_)
                CK(cudaMemcpyPeerAsync(in_utf8_.p, device_, utf8 + first, src_device, n_bytes, stream_));
            else if (src_device >= 0)
                CK(cudaMemcpyAsync(in_utf8_.p, utf8 + first, n_bytes, cudaMemcpyDeviceToDevice, stream_));
            else
                h2d(in_utf8_.p, utf8 + first, n_bytes, stream_, is_pinned(utf8 + first));
        }
        run_whole(in_utf8_.as<uint8_t>(), in_off_.as<unsigned long long>(), n_sent, n_bytes, bd, first_sentence);
        shard_n_sent_ = n_sent;
        if (with_text && output_mode_ != kOutNone) format_whole(in_utf8_.as<uint8_t>(), in_off_.as<unsigned long long>(), n_sent);
        keep_device_outputs();
        return last_.total;
    }
    void rebase_shard(const Totals& base) override {
        CK(cudaSetDevice(device_));
        add_bases(base);
        CK(cudaStreamSynchronize(stream_));
    }
    void fetch_shard(HostResult* r, uint64_t first_sentence, const Totals& base, bool last) override {
        CK(cudaSetDevice(device_));
        add_bases(base);
        place(out_[0], r, first_sentence, shard_n_sent_, totals(*out_[0].h_ctrl), base, last, stream_);
        CK(cudaStreamSynchronize(stream_));
    }
    int device() const override { return device_; }
    uint32_t token_bytes() const override { return tok_bytes_; }
    std::string describe() const override {
        static const char* const kRouteNames[] = {"none", "k_viterbi", "k_viterbi2", "k_viterbi2_unpruned", "k_small_batch"};
        std::string ft;
        if (output_mode_ == kOutFormat)  // the field table of the output format: device bytes and build time
            ft = ", \"field_table\": {\"bytes\": " + std::to_string(ft_size_) + ", \"build_ms\": " + std::to_string(ft_ms_) + "}";
        return "{\"devices\": [" + std::to_string(device_) + "], \"dictionary_transport\": \"single device\", \"token_gather\": \"none\", " +
               "\"last_viterbi\": \"" + kRouteNames[last_route_] + "\"" + ft + ", " + reruns_json(reruns_) + "}";
    }
    Reruns last_reruns() const override { return reruns_; }

   private:
    // Host -> device copy of caller memory.  Pinned (page-locked) memory goes straight to the copy engine; pageable
    // memory is staged through a small ring of pinned buffers owned by the engine, so that the copy stays
    // asynchronous and runs at PCIe speed instead of falling back to the driver's synchronous bounce path.
    static bool is_pinned(const void* p) {
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
    }
    void h2d(void* dst, const void* src, size_t bytes, cudaStream_t st, bool src_pinned) {
        if (!bytes) return;
        if (src_pinned) {
            CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st));
            return;
        }
        if (!ring_[0]) {
            for (int i = 0; i < kRingSlots; ++i) {
                ring_[i] = static_cast<uint8_t*>(pinned_alloc(kRingBytes));
                CK(cudaEventCreateWithFlags(&ring_ev_[i], cudaEventDisableTiming));
            }
        }
        for (size_t o = 0; o < bytes; o += kRingBytes) {
            const size_t len = std::min(kRingBytes, bytes - o);
            const int slot = ring_next_;
            ring_next_ = (ring_next_ + 1) % kRingSlots;
            CK(cudaEventSynchronize(ring_ev_[slot]));  // the copy that last used this slot has left it
            std::memcpy(ring_[slot], static_cast<const uint8_t*>(src) + o, len);
            CK(cudaMemcpyAsync(static_cast<uint8_t*>(dst) + o, ring_[slot], len, cudaMemcpyHostToDevice, st));
            CK(cudaEventRecord(ring_ev_[slot], st));
        }
    }

    // One attempt at a batch = connid_begin, its enqueue(s), then connid_commit once it is known to have succeeded.
    void connid_begin(cudaStream_t st) {
        if (connid_on_) CK(cudaMemsetAsync(connid_try_.p, 0, (size_t(num_left_) + num_right_) * 8, st));
    }
    void connid_commit(cudaStream_t st) {
        if (!connid_on_) return;
        const size_t n = size_t(num_left_) + num_right_;
        k_add_u64<<<unsigned((n + 255) / 256), 256, 0, st>>>(connid_.as<unsigned long long>(),
                                                                connid_try_.as<unsigned long long>(), n);
        CK(cudaStreamSynchronize(st));
    }

    void check_size(uint64_t n_sent, uint64_t n_bytes) const {
        // warp-per-sentence kernels derive the sentence from a 32-bit global thread index (>> 5): 2^27 is the bound
        if (n_sent >= 0x07FFFFFFull || n_bytes + n_sent >= 0xFFFFFF00ull)
            throw Error(kInvalidArgument, "batch too large: split it (at most 2^27 sentences / 2^32 characters per call)");
        if (n_sent * samp_n_ >= 0xFFFFFFFFull)
            throw Error(kInvalidArgument, "sampling: n_sent * n must stay below 2^32: split the batch or draw fewer samples");
        if (sample_base_ + n_sent > kMaxSampleBase)
            throw Error(kInvalidArgument, "sampling: sample_base + n_sent exceeds 2^32, the range of the draws' sentence index");
    }

    void check_bounded(const Bounds* bnd) const {
        if (bnd && counting_)
            throw Error(kInvalidArgument, "the \"counting\" hook measures the unconstrained lattice: it refuses bounded batches");
    }

    // A batch whose boundary lists are all empty (every offset the same) runs the unbounded kernels.  Broken offsets
    // are not empty: they take the bounded route, which reports them after the errors that take precedence.
    static bool host_lists_empty(const uint64_t* off, uint64_t n_sent) {
        for (uint64_t i = 0; i < n_sent; ++i)
            if (off[i + 1] != off[0]) return false;
        return true;
    }
    // bnd without its empty boundary or span lists (in nb), or nullptr when both are empty.
    static const Bounds* drop_empty(const Bounds* bnd, uint64_t n_sent, Bounds& nb) {
        if (!bnd) return nullptr;
        nb = *bnd;
        if (nb.spans.off && host_lists_empty(nb.spans.off, n_sent)) nb.spans = Spans{};
        if (nb.off && host_lists_empty(nb.off, n_sent)) nb.off = nullptr;
        return (nb.off || nb.spans.off) ? &nb : nullptr;
    }
    // The window of the caller's buffer a host batch uses (its offsets may start anywhere in it; only the window is
    // copied): the checks of the call, its offsets rebased to the window's first byte (into rebased_ unless that is
    // 0), its bounds without empty lists (drop_empty, into nb) and in_utf8_ / in_off_ sized for it.
    struct HostWindow {
        uint64_t first, n_bytes;
        const uint64_t* off;
        const Bounds* bnd;
    };
    HostWindow host_window(const uint64_t* byte_off, uint64_t n_sent, const Bounds* bnd, Bounds& nb) {
        const uint64_t first = n_sent ? byte_off[0] : 0;
        HostWindow w{first, n_sent ? byte_off[n_sent] - first : 0, byte_off, nullptr};
        check_size(n_sent, w.n_bytes);
        check_bounded(bnd);
        w.bnd = drop_empty(bnd, n_sent, nb);  // no boundary and no span at all: the unbounded kernels
        in_utf8_.ensure(w.n_bytes + 16, 1.25);
        in_off_.ensure((size_t(n_sent) + 1) * 8, 1.25);
        if (first != 0) {
            rebased_.resize(size_t(n_sent) + 1);
            for (uint64_t i = 0; i <= n_sent; ++i) rebased_[i] = byte_off[i] - first;
            w.off = rebased_.data();
        }
        return w;
    }
    // n_sent + 1 zero offsets on the device (in_bnd_off_): a span batch without explicit boundaries.
    const unsigned long long* zero_offsets(uint32_t n_sent, cudaStream_t st) {
        in_bnd_off_.ensure((size_t(n_sent) + 1) * 8, 1.25);
        CK(cudaMemsetAsync(in_bnd_off_.p, 0, (size_t(n_sent) + 1) * 8, st));
        return in_bnd_off_.as<unsigned long long>();
    }
    // The compiled patterns of s (host) -> one device block [pat_off | pf | bytes] (in_pat_).
    void upload_patterns(const Spans& s, DevBounds& d, cudaStream_t st) {
        const size_t n_off = size_t(s.n_pat) + 1, n_pf = s.pat_off[s.n_pat];
        const size_t at_pf = (n_off * 4 + 15) & ~size_t(15), at_bytes = at_pf + n_pf * 12;
        in_pat_.ensure(at_bytes + s.n_pat_bytes + 16, 1.25);
        uint8_t* p = in_pat_.as<uint8_t>();
        h2d(p, s.pat_off, n_off * 4, st, false);
        if (n_pf) h2d(p + at_pf, s.pf, n_pf * 12, st, false);
        if (s.n_pat_bytes) h2d(p + at_bytes, s.pat_bytes, s.n_pat_bytes, st, false);
        d.pat_off = reinterpret_cast<const uint32_t*>(p);
        d.pf = reinterpret_cast<const uint3*>(p + at_pf);
        d.pat_bytes = p + at_bytes;
        d.n_pat = s.n_pat;
    }
    // The same for device-resident lists with n_bnd == 0: valid offsets are then all 0 (one copy of them to the host).
    bool device_offsets_zero(const uint64_t* d_off, uint64_t n_sent) {
        const size_t bytes = (size_t(n_sent) + 1) * 8;
        if (bnd_stage_cap_ < bytes) {
            pinned_free(bnd_stage_);
            bnd_stage_ = static_cast<uint64_t*>(pinned_alloc(bytes));
            bnd_stage_cap_ = bytes;
        }
        CK(cudaMemcpyAsync(bnd_stage_, d_off, bytes, cudaMemcpyDeviceToHost, stream_));
        CK(cudaStreamSynchronize(stream_));
        for (uint64_t i = 0; i <= n_sent; ++i)
            if (bnd_stage_[i] != 0) return false;
        return true;
    }

    // Host boundary lists -> in_bnd_off_ / in_bnd_ on `st`.  The offsets are rebased to the window that is copied,
    // bnd[off[0] .. off[n_sent]).  A list whose window is inverted or leaves bnd ships no boundaries and keeps
    // offsets that k_mark_bounds refuses (some sentence's end offset then lies below its start or beyond 0).
    DevBounds upload_bounds(const Bounds& hb, uint32_t n_sent, cudaStream_t st) {
        DevBounds d = hb.off ? upload_list(hb.off, hb.bnd, hb.n, n_sent, st) : DevBounds{zero_offsets(n_sent, st)};
        if (hb.spans.off) {  // the same for the span records (12 bytes each) into in_span_off_ / in_span_
            const DevBounds s = upload_list(hb.spans.off, hb.spans.rec, hb.spans.n, n_sent, st, 12);
            d.span_off = s.off;
            d.span_rec = reinterpret_cast<const uint3*>(s.bnd);
            d.n_spans = s.n;
            upload_patterns(hb.spans, d, st);
        }
        return d;
    }
    DevBounds upload_list(const uint64_t* hoff, const void* hrec, uint64_t hn, uint32_t n_sent, cudaStream_t st,
                          size_t rec_bytes = 4) {
        const bool spans = rec_bytes != 4;
        std::vector<uint64_t>& rebased = spans ? span_rebased_ : bnd_rebased_;
        DevBuf& d_off = spans ? in_span_off_ : in_bnd_off_;
        DevBuf& d_rec = spans ? in_span_ : in_bnd_;
        const uint64_t first = hoff[0], last = hoff[n_sent];
        const bool sound = first <= last && last <= hn;
        const uint64_t lo = sound ? first : 0, n = sound ? last - first : 0;
        rebased.resize(size_t(n_sent) + 1);
        for (uint32_t i = 0; i <= n_sent; ++i) rebased[i] = hoff[i] - lo;  // wraps for a broken list: refused
        d_off.ensure((size_t(n_sent) + 1) * 8, 1.25);
        d_rec.ensure(n * rec_bytes + 16, 1.25);
        h2d(d_off.p, rebased.data(), (size_t(n_sent) + 1) * 8, st, false);
        const uint8_t* src = static_cast<const uint8_t*>(hrec) + lo * rec_bytes;
        if (n) h2d(d_rec.p, src, n * rec_bytes, st, is_pinned(src));
        return DevBounds{d_off.as<unsigned long long>(), d_rec.as<uint32_t>(), n};
    }

    std::vector<cudaEvent_t>& h2d_events(uint32_t n) {
        while (h2d_ev_.size() < n) {
            cudaEvent_t e;
            CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            h2d_ev_.push_back(e);
        }
        return h2d_ev_;
    }

    // last_ = the arrays a whole batch or shard left in out_[0].
    void keep_device_outputs() {
        const OutSlot& o = out_[0];
        last_.made = o.made;
        last_.total = totals(*o.h_ctrl);
        for (int a = 0; a < kNumArrays; ++a) last_.addr[a] = o.made.has(a) ? reinterpret_cast<uint64_t>(o.buf[a].p) : 0;
    }

    // Switches text source src on (it replaces the best path in the output text) or off (back to the best path when
    // it was the source): the rules of every source, in the order they are reported.
    void set_text(TextSrc src, bool on) {
        const uint32_t uses = output_mode_ == kOutFormat ? fmt_uses_ : 0;
        if (on) {
            if (src == kTextSamples && !samp_n_)
                throw Error(kInvalidArgument, "sample_text needs sampling: switch it on with set_sampling first");
            if (src == kTextPosterior && !post_)
                throw Error(kInvalidArgument, "posterior_text needs posterior decoding: switch it on with set_posterior first");
            if (src == kTextNodes && (uses & kUsesPrev))
                throw Error(kInvalidArgument,
                            "the output format prints a \"prev\" directive (%M %pS %pn %pC %pL), which lattice text has no value for: "
                            "change the format before setting lattice = 2");
            if (text_src_ != kTextBest && text_src_ != src)
                throw Error(kInvalidArgument, std::string(kTextSrcs[std::min(text_src_, src)].name) + " text and " +
                                                  kTextSrcs[std::max(text_src_, src)].name + " text both replace the output text: set " +
                                                  kTextSrcs[text_src_].off + " before setting " + kTextSrcs[src].on);
            if (src == kTextSamples && (uses & (kUsesProb | kUsesBest)))  // capi names the directive
                throw Error(kInvalidArgument, "the output format prints %pP or %pb, which sample text has no value for: change the format before setting sample_text = 1");
        } else if (src == kTextNodes && (uses & kUsesBest)) {
            throw Error(kInvalidArgument, "the output format prints %pb, which only lattice text has: change the format before setting lattice below 2");
        }
        cudaStreamSynchronize(stream_);
        if (on || text_src_ == src) text_src_ = on ? src : kTextBest;
    }

    PassPlan plan() const {
        const bool marg = theta_ > 0, margin = lattice_ && lat_margin_ >= 0;
        const FwdKind fwd = (samp_n_ || post_) ? kFwdLseLw : marg ? kFwdLse : margin ? kFwdR : kFwdNone;
        return PassPlan{fwd, !marg ? kBwdNone : unc_ ? kBwdUnc : kBwdPlain, marg && unc_ >= 2, margin, lattice_, post_, samp_n_,
                        // k_small_batch runs none of the passes and counts nothing
                        small_batch_ && fwd == kFwdNone && !lattice_ && !counting_ && !connid_on_,
                        // the eager copies are sized by the token bound alone
                        output_mode_ == kOutNone && !lattice_ && !samp_n_ && !unc_ && !post_};
    }

    // What the output stage renders from slot o (text_src_): offsets, records and the marginals %pP prints, the
    // renderings per sentence (each of its samples in sample text), and the nodes' links when lattice text prints %pb.
    struct TextView { const DevBuf *tok_off, *tokens; const float* prob; uint32_t units; const int2* links; };
    TextView text_view(const OutSlot& o) const {
        const TextSrcInfo& t = kTextSrcs[text_src_];
        const bool prob = o.made.marg && output_mode_ == kOutFormat && (fmt_uses_ & kUsesProb) && t.prob != kNumArrays;
        const bool links = text_src_ == kTextNodes && output_mode_ == kOutFormat && (fmt_uses_ & kUsesBest);
        return TextView{&o.buf[t.tok_off], &o.buf[t.tokens], prob ? o.buf[t.prob].as<float>() : nullptr,
                        text_src_ == kTextSamples ? samp_n_ : 1, links ? o.buf[kLinks].as<int2>() : nullptr};
    }

    // D2H on `st` of every array r carries, from slot `o` holding n sentences and `count` records per group: to
    // sentence s0 of r and after `base` records per group; `last` brings the closing offsets too.
    void place(const OutSlot& o, HostResult* r, uint64_t s0, uint64_t n, const Totals& count, const Totals& base, bool last,
               cudaStream_t st) {
        for (int a = 0; a < kNumArrays; ++a) {
            if (!r->out.has(a)) continue;
            if (!o.made.has(a)) throw Error(kInternal, "the batch was run without an output its result carries");
            const uint64_t bytes = r->out.bytes(a, n, count, last);
            if (bytes)
                CK(cudaMemcpyAsync(r->ptr<uint8_t>(a) + r->out.at(a, s0, base), o.buf[a].p, bytes, cudaMemcpyDeviceToHost, st));
        }
    }

    // Adds base[g] to the last shard's offsets of every group g it produced, on stream_.
    void add_bases(const Totals& base) {
        const OutSlot& o = out_[0];
        for (int g = 0; g < kNumGroups; ++g) {
            const int a = kOffsetsOf[g];
            if (!o.made.has(a) || !base[g]) continue;
            const uint64_t n = uint64_t(shard_n_sent_) * o.made.stride(a) + 1;
            k_add_value<<<unsigned((n + 255) / 256), 256, 0, stream_>>>(o.buf[a].as<unsigned long long>(), uint32_t(n), base[g]);
        }
    }

    // Device outputs of slot `o` for (chunks of) up to n_sent sentences and n_bytes bytes, except the text (sized by
    // the output stage), the sample records (sized by enqueue from the scanned total) and the lattice records (one
    // per lattice entry: ensure_entries).
    void ensure_out(OutSlot& o, uint32_t n_sent, uint64_t n_bytes) {
        const Outputs out = outputs();
        const PassPlan p = plan();
        Totals most{};  // records per group: a token spans >= 1 character >= 1 byte, and a slot is a character or a sentinel
        most[kGroupTokens] = most[kGroupPosterior] = n_bytes + 1;
        most[kGroupPositions] = n_bytes + n_sent + 1;
        for (int a = 0; a < kNumArrays; ++a) {
            const ArrayInfo& k = kArrays[a];
            // sampling without marginals: the forward pass still writes path_prob
            const bool need = out.has(a) || (a == kPathProb && p.fwd >= kFwdLse);
            if (!need || k.group == kGroupText || (k.kind == kRecords && !most[k.group])) continue;
            const uint64_t rows = k.kind == kRecords ? most[k.group] : uint64_t(n_sent) * out.stride(a) + 1;
            o.buf[a].ensure(rows * out.elem_bytes(a), 1.25);
        }
    }

    double& text_ratio_ref() { return text_per_byte_[kTextSrcs[text_src_].ratio][output_mode_]; }

    // Output stage buffers of slot `o` and scan storage of `w` for (chunks of) up to n_sent sentences.
    void ensure_format(OutSlot& o, Workspace& w, uint32_t n_sent) {
        const size_t units = size_t(n_sent) * text_view(o).units + 1;
        o.sent_len.ensure(units * 8, 1.25);
        if (text_src_ == kTextSamples) o.walk_off.ensure(units * 8, 1.25);
        o.buf[kTextOff].ensure((size_t(n_sent) + 1) * 8, 1.25);
        size_t tmp = 0;
        CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp, static_cast<unsigned long long*>(nullptr),
                                         static_cast<unsigned long long*>(nullptr), units, w.stream));
        w.scan_tmp.ensure(tmp + 1024, 1.5);
    }

    // Output stage, pass 1 and the scan on w.stream: the text offsets of `o` = where each sentence's text starts in its
    // text (n_sent + 1 entries, relative to the batch or chunk in `o`).  Returns the arguments of pass 2.  Sample text
    // renders the walks of the samples instead: its offsets per walk go to o.walk_off, and pass 2 (format_write)
    // takes those of each sentence's first walk into the text offsets.
    FormatArgs format_offsets(Workspace& w, const uint8_t* d_utf8, const unsigned long long* d_off, uint32_t n_sent, OutSlot& o) {
        const TextView t = text_view(o);
        FormatArgs f{};
        f.utf8 = d_utf8;
        f.byte_off = d_off;
        f.n_sent = n_sent;
        f.tok_off = t.tok_off->as<unsigned long long>();
        f.tokens = t.tokens->as<uint2>();
        f.token_prob = t.prob;
        f.sent_len = o.sent_len.as<unsigned long long>();
        f.text_off = (text_src_ == kTextSamples ? o.walk_off : o.buf[kTextOff]).as<unsigned long long>();
        f.text = o.buf[kText].as<uint8_t>();
        f.text_cap = o.buf[kText].cap;
        Control* dc = o.ctrl.as<Control>();
        f.flags = &dc->flags;
        f.text_total = &dc->total[kGroupText];
        set_mode(f);
        const size_t units = size_t(n_sent) * t.units;
        CK(cudaMemsetAsync(f.sent_len + units, 0, 8, w.stream));
        if (text_src_ == kTextSamples) {
            if (!n_sent) CK(cudaMemsetAsync(o.buf[kTextOff].p, 0, 8, w.stream));  // no walk writes it
            launch_format_len_samples(dv_, f, samp_n_, w.stream);
        } else {
            launch_format_len(dv_, f, w.stream, t.links);
        }
        exclusive_scan(w, f.sent_len, f.text_off, units + 1);
        return f;
    }

    // Output stage, pass 2 on `st`, after format_offsets.
    void format_write(const FormatArgs& f, OutSlot& o, cudaStream_t st) {
        if (text_src_ == kTextSamples)
            launch_format_write_samples(dv_, f, samp_n_, o.buf[kTextOff].as<unsigned long long>(), st);
        else
            launch_format_write(dv_, f, st, text_view(o).links);
    }

    // Output stage of a whole batch (or shard) that run_whole left in out_[0]: the text buffer is sized from the
    // exact total, read back with one synchronisation, which out_[0] records with the text arrays.
    void format_whole(const uint8_t* d_utf8, const unsigned long long* d_off, uint32_t n_sent) {
        OutSlot& o = out_[0];
        ensure_format(o, ws_[0], n_sent);
        FormatArgs f = format_offsets(ws_[0], d_utf8, d_off, n_sent, o);
        unsigned long long total = 0;
        const size_t units = size_t(n_sent) * text_view(o).units;  // the scan's last entry is the total
        CK(cudaMemcpyAsync(&total, f.text_off + units, 8, cudaMemcpyDeviceToHost, stream_));
        CK(cudaStreamSynchronize(stream_));
        o.buf[kText].ensure(total + 16, 1.25);
        f.text = o.buf[kText].as<uint8_t>();
        f.text_cap = o.buf[kText].cap;
        format_write(f, o, stream_);
        launches_ += 2;
        o.h_ctrl->total[kGroupText] = total;
        o.made.text = true;
    }

    // ---- k_small_batch route -------------------------------------------------------------------------------
    // Its scratch is sized once for the largest batch the route accepts: per-slot arrays for the hard bound of
    // kEagerBytes + small_batch_ + 1 slots and a pool of kSmallCands candidates (about 5 MiB with the lattice rows,
    // so it stays in L2).  A batch with more candidates, or more text than kSmallText, flags itself and is run again
    // on the usual route; nothing grows on the device.  Input and output each travel in ONE copy: offsets + text up
    // through a pinned staging block, and the output region [SmallBatchOut | tok_off | text_off | tokens | text] back
    // into another, from which the result is copied into the pooled HostResult.
    static constexpr uint32_t kSmallCands = 131072;
    static constexpr size_t kSmallText = size_t(2) << 20;
    static constexpr long long kSmallBatchMax = 65536;
    static constexpr size_t kSmallHead = 64;  // SmallBatchOut, padded
    static constexpr uint64_t kSmallBounds = 16384;  // boundaries a bounded batch may bring (more take the usual route)

    // A bounded host batch takes k_small_batch when its boundaries fit the upload; a broken list is left to the usual
    // route, which reports it.
    bool small_bounds_fit(const Bounds& hb, uint32_t n_sent) const {
        const uint64_t first = hb.off[0], last = hb.off[n_sent];
        return first <= last && last <= hb.n && last - first <= kSmallBounds;
    }

    void ensure_small() {
        Workspace& w = ws_small_;
        const size_t ns = size_t(small_batch_) + 1, ms = kEagerBytes + ns;
        w.n_slots.ensure(ns * 4);
        w.slot_off.ensure(ns * 4);
        w.eos.ensure(ns * 16);
        w.n_tok.ensure(ns * 4);
        w.stats.ensure(ns * 8);  // sent_len of the output stage
        w.code_sys.ensure(ms * 4);
        if (dv_.usr_table) w.code_usr.ensure(ms * 4);
        w.cinfo.ensure(ms * 4);
        w.groupable.ensure(ms * 4);
        w.byte_pos.ensure(ms * 4);
        w.info.ensure(ms * 8);
        w.info_ex.ensure(ms * 8);
        w.ends_cnt.ensure(ms * 4);
        w.ends_meta.ensure(ms * 8);
        w.bnd_dist.ensure(ms * 4);
        // Segments outnumber candidates only through move segments (an end slot more than 32 767 away); 16 KiB of
        // text keeps every move shorter, so each segment holds a candidate here.
        w.seg.ensure(size_t(kSmallCands) * 8);
        w.ends_hot.ensure((kSmallCands + ns) * 8);
        w.ends_cold.ensure((kSmallCands + ns) * 16);
        const size_t in_cap = ns * 8 + kEagerBytes + 8 + ns * 8 + kSmallBounds * 4;  // [off | utf8 | bnd_off | bnd]
        const size_t out_cap = kSmallHead + 2 * ns * 8 + 16 + kEagerBytes * 24 + kSmallText;
        small_in_.ensure(in_cap);
        small_out_.ensure(out_cap);
        if (small_in_cap_ < in_cap) {
            pinned_free(small_in_h_);
            small_in_h_ = static_cast<uint8_t*>(pinned_alloc(in_cap));
            small_in_cap_ = in_cap;
        }
        if (small_out_cap_ < out_cap) {
            pinned_free(small_out_h_);
            small_out_h_ = static_cast<uint8_t*>(pinned_alloc(out_cap));
            small_out_cap_ = out_cap;
        }
    }

    // One host batch through k_small_batch: one copy up, one launch, one copy down, one synchronisation (a second
    // copy only when the text outgrew the part of the region the first one brought back).  Returns nullptr when the
    // batch overflowed the scratch; input errors throw like on the usual route.
    HostResult* run_small(const char* utf8, const uint64_t* off, uint32_t n_sent, uint64_t n_bytes, const Bounds* bnd) {
        ensure_small();
        const size_t off_bytes = (size_t(n_sent) + 1) * 8;
        std::memcpy(small_in_h_, off, off_bytes);
        if (n_bytes) std::memcpy(small_in_h_ + off_bytes, utf8, n_bytes);
        size_t in_bytes = off_bytes + n_bytes;
        const size_t at_bnd_off = (in_bytes + 7) & ~size_t(7), at_bnd = at_bnd_off + off_bytes;
        uint64_t n_bnd = 0;
        if (bnd) {  // the boundaries travel in the same copy, their offsets rebased to the part that is copied
            const uint64_t first = bnd->off[0];
            n_bnd = bnd->off[n_sent] - first;
            uint64_t* o = reinterpret_cast<uint64_t*>(small_in_h_ + at_bnd_off);
            for (uint32_t i = 0; i <= n_sent; ++i) o[i] = bnd->off[i] - first;
            if (n_bnd) std::memcpy(small_in_h_ + at_bnd, bnd->bnd + first, n_bnd * 4);
            in_bytes = at_bnd + n_bnd * 4;
        }
        CK(cudaMemcpyAsync(small_in_.p, small_in_h_, in_bytes, cudaMemcpyHostToDevice, stream_));

        const bool fmt = output_mode_ != kOutNone;
        const size_t tb = tok_bytes_;
        const size_t at_tok_off = kSmallHead, at_text_off = at_tok_off + off_bytes;
        const size_t at_tokens = (at_text_off + (fmt ? off_bytes : 0) + 15) & ~size_t(15);
        const size_t at_text = at_tokens + n_bytes * tb;
        uint8_t* region = small_out_.as<uint8_t>();
        Workspace& w = ws_small_;
        Batch b{};
        b.utf8 = small_in_.as<uint8_t>() + off_bytes;
        b.byte_off = small_in_.as<unsigned long long>();
        b.total_bytes = n_bytes;
        b.n_sent = n_sent;
        b.n_slots = w.n_slots.as<uint32_t>();
        b.slot_off = w.slot_off.as<uint32_t>();
        b.eos = w.eos.as<uint4>();
        b.n_tok = w.n_tok.as<uint32_t>();
        b.tok_off = reinterpret_cast<unsigned long long*>(region + at_tok_off);
        b.code_sys = w.code_sys.as<uint32_t>();
        b.code_usr = w.code_usr.as<uint32_t>();
        b.cinfo = w.cinfo.as<uint32_t>();
        b.groupable = w.groupable.as<uint32_t>();
        b.byte_pos = w.byte_pos.as<uint32_t>();
        b.info = w.info.as<uint2>();
        b.info_ex = w.info_ex.as<uint2>();
        b.ends_cnt = w.ends_cnt.as<uint32_t>();
        b.ends_meta = w.ends_meta.as<uint2>();
        b.seg = w.seg.as<uint2>();
        b.seg_cap = kSmallCands;
        b.cand_cap = kSmallCands;
        b.ends_hot = w.ends_hot.as<int2>();
        b.ends_cold = w.ends_cold.as<uint4>();
        b.tokens = region + at_tokens;
        b.compact = tb == 16 ? 1u : 0u;
        if (bnd) {
            b.bnd_off = reinterpret_cast<const unsigned long long*>(small_in_.as<uint8_t>() + at_bnd_off);
            b.bnd = reinterpret_cast<const uint32_t*>(small_in_.as<uint8_t>() + at_bnd);
            b.n_bnd = n_bnd;
            b.bnd_dist = w.bnd_dist.as<uint32_t>();
        }
        FormatArgs f{};
        f.utf8 = b.utf8;
        f.byte_off = b.byte_off;
        f.n_sent = n_sent;
        f.tok_off = b.tok_off;
        f.tokens = static_cast<const uint2*>(b.tokens);
        f.sent_len = w.stats.as<unsigned long long>();
        f.text_off = reinterpret_cast<unsigned long long*>(region + at_text_off);
        f.text = region + at_text;
        f.text_cap = small_out_cap_ - at_text;  // the device region and its pinned twin have (at least) this size
        set_mode(f);

        // the first copy brings the text expected from the learned ratio; more comes in a second one
        const size_t text_guess = fmt ? std::min<size_t>(f.text_cap, size_t(double(n_bytes) * text_per_byte_[0][output_mode_]) +
                                                                         size_t(n_sent) * text_per_sent_ + 256)
                                      : 0;
        OutSlot& o = out_[0];
        CK(cudaEventRecord(o.ev[0], stream_));
        launch_small_batch(dv_, b, f, reinterpret_cast<SmallBatchOut*>(region), stream_);
        CK(cudaGetLastError());
        CK(cudaEventRecord(o.ev[1], stream_));
        CK(cudaMemcpyAsync(small_out_h_, region, at_text + text_guess, cudaMemcpyDeviceToHost, stream_));
        CK(cudaStreamSynchronize(stream_));
        SmallBatchOut h;
        std::memcpy(&h, small_out_h_, sizeof h);
        throw_input_error(h.flags);
        if (rerun(h.flags, 0)) return nullptr;
        if (fmt && h.text_bytes > text_guess) {
            CK(cudaMemcpyAsync(small_out_h_ + at_text + text_guess, region + at_text + text_guess, h.text_bytes - text_guess,
                               cudaMemcpyDeviceToHost, stream_));
            CK(cudaStreamSynchronize(stream_));
            if (n_bytes)
                text_per_byte_[0][output_mode_] = std::max(text_per_byte_[0][output_mode_] * 1.5, double(h.text_bytes) / double(n_bytes) * 1.25);
        }
        HostResult* r = pool_.acquire(outputs(), n_sent, Totals{h.n_tokens, fmt ? h.text_bytes : 0, 0, 0});
        std::memcpy(r->buf[kTokOff].p, small_out_h_ + at_tok_off, off_bytes);
        if (h.n_tokens) std::memcpy(r->buf[kTokens].p, small_out_h_ + at_tokens, h.n_tokens * tb);
        if (fmt) {
            std::memcpy(r->buf[kTextOff].p, small_out_h_ + at_text_off, off_bytes);
            if (h.text_bytes) std::memcpy(r->buf[kText].p, small_out_h_ + at_text, h.text_bytes);
        }
        clear_stats();
        CK(cudaEventElapsedTime(&stage_ms_[kSmallBatchStage], o.ev[0], o.ev[1]));
        launches_ = 1;
        last_route_ = kRouteSmallBatch;
        return r;
    }

    // The output mode of the stage, with the program and field table of an output format.
    void set_mode(FormatArgs& f) const {
        f.mode = output_mode_;
        f.prog = fmt_prog_.as<FormatProgram>();
        f.ft_keep = ft_keep_.as<uint32_t>();
        f.ft_off = ft_off_.as<uint32_t>();
        f.ft_bytes = ft_bytes_.as<uint8_t>();
    }

    void clear_format() {
        CK(cudaStreamSynchronize(stream_));
        for (DevBuf* b : {&fmt_prog_, &ft_keep_, &ft_off_, &ft_bytes_}) b->release();
        ft_size_ = 0;
        ft_ms_ = 0;
        fmt_uses_ = 0;
        text_per_sent_ = 4;
        if (output_mode_ == kOutFormat) output_mode_ = kOutNone;
    }

    // The field table of format `p` (FormatArgs::ft_*): per word of the three lexicons, the unquoted text of every
    // field p references, split on the device from the feature strings of the image (k_field_table_*).
    void build_field_table(const FormatProgram& p) {
        const uint64_t n_words = uint64_t(dv_.n_words[0]) + dv_.n_words[1] + dv_.n_words[2];
        const uint64_t n_entries = n_words * p.n_fields;
        uint64_t feat_bytes = 0;  // a field is part of its feature string: the table holds at most this many bytes
        for (int li = 0; li < 3; ++li) {
            uint32_t end = 0;
            if (dv_.n_words[li]) CK(cudaMemcpy(&end, dv_.feat_off[li] + dv_.n_words[li], 4, cudaMemcpyDeviceToHost));
            feat_bytes += end;
        }
        if (n_entries + 1 > 0xFFFFFFFFull || feat_bytes > 0xFFFFFFFFull)
            throw Error(kUnsupported, "the field table of this format exceeds 2^32 entries or bytes: reference fewer fields");
        FieldTableArgs a{};
        std::memset(a.slot_of, 0xFF, sizeof a.slot_of);
        for (uint32_t k = 0; k < p.n_fields; ++k) {
            a.slot_of[p.fields[k]] = uint8_t(k);
            a.fields[k] = p.fields[k];
        }
        a.n_fields = p.n_fields;
        a.n_words = uint32_t(n_words);
        DevBuf lens, tmp;
        cudaEvent_t ev[2] = {nullptr, nullptr};
        try {
            for (auto& e : ev) CK(cudaEventCreate(&e));
            CK(cudaEventRecord(ev[0], stream_));
            lens.ensure((n_entries + 1) * 4);
            ft_keep_.ensure(n_words * 4);
            ft_off_.ensure((n_entries + 1) * 4);
            a.lens = lens.as<uint32_t>();
            a.keep = ft_keep_.as<uint32_t>();
            launch_field_table_len(dv_, a, stream_);
            CK(cudaMemsetAsync(a.lens + n_entries, 0, 4, stream_));
            size_t tmp_bytes = 0;
            CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, a.lens, ft_off_.as<uint32_t>(), n_entries + 1, stream_));
            tmp.ensure(tmp_bytes);
            CK(cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, a.lens, ft_off_.as<uint32_t>(), n_entries + 1, stream_));
            uint32_t total = 0;
            CK(cudaMemcpyAsync(&total, ft_off_.as<uint32_t>() + n_entries, 4, cudaMemcpyDeviceToHost, stream_));
            CK(cudaStreamSynchronize(stream_));
            ft_bytes_.ensure(size_t(total) + 16);
            a.off = ft_off_.as<uint32_t>();
            a.bytes = ft_bytes_.as<uint8_t>();
            launch_field_table_write(dv_, a, stream_);
            CK(cudaGetLastError());
            CK(cudaEventRecord(ev[1], stream_));
            CK(cudaEventSynchronize(ev[1]));
            CK(cudaEventElapsedTime(&ft_ms_, ev[0], ev[1]));
            ft_size_ = ft_keep_.cap + ft_off_.cap + ft_bytes_.cap;
        } catch (...) {
            lens.release();
            tmp.release();
            for (auto& e : ev)
                if (e) cudaEventDestroy(e);
            throw;
        }
        lens.release();
        tmp.release();
        for (auto& e : ev) cudaEventDestroy(e);
    }

    template <typename In, typename Out>
    void exclusive_scan(Workspace& w, In in, Out out, size_t n) {
        size_t cap = w.scan_tmp.cap;  // sized by ensure_workspace
        CK(cub::DeviceScan::ExclusiveSum(w.scan_tmp.p, cap, in, out, n, w.stream));
    }
    // A ragged group's offsets on w.stream: off[0..n] = the exclusive scan of the n counts cnt (cnt[n], which the scan
    // reads, zeroed first), and the group's total off[n] into Control.
    void scan_group(Workspace& w, uint32_t* cnt, unsigned long long* off, size_t n, unsigned long long* total) {
        CK(cudaMemsetAsync(cnt + n, 0, 4, w.stream));
        exclusive_scan(w, CountsU64(cnt, CastU64()), off, n + 1);
        CK(cudaMemcpyAsync(total, off + n, 8, cudaMemcpyDeviceToDevice, w.stream));
    }

    // Candidates a batch (or chunk) of n_bytes bytes is given room for, from the ratio learned on earlier batches.
    size_t want_cand(uint64_t n_bytes) const {
        return std::min<size_t>(std::max<size_t>(1 << 16, size_t(double(n_bytes) * cand_per_byte_) + 4096), 0xFFFFFFF0ull);
    }

    // Every array indexed by lattice entry under the current options, with its bytes per entry: f(buffer, width) for
    // the rows of workspace w and the lattice records of slot o.  ensure_entries sizes them and enqueue bounds the
    // pool by them, both from this one list.
    template <typename F>
    void per_entry(Workspace& w, OutSlot& o, F&& f) const {
        const PassPlan p = plan();
        f(w.ends_hot, 8);
        f(w.ends_cold, 16);
        if (p.fwd != kFwdNone) {
            f(w.m_cand_entry, 4);
            f(w.m_R, 8);
        }
        if (p.fwd >= kFwdLse) f(w.m_ab, 16);
        if (p.fwd == kFwdLseLw) f(w.m_lw, 4);
        if (p.margin) {
            f(w.g_G, 8);
            f(w.g_keep, 4);
        }
        const Outputs out = outputs();  // a lattice node is a candidate placed in the pool
        for (int a = 0; a < kNumArrays; ++a)
            if (kArrays[a].group == kGroupLattice && kArrays[a].kind == kRecords && out.has(a)) f(o.buf[a], out.elem_bytes(a));
    }
    void ensure_entries(Workspace& w, OutSlot& o, size_t entries) {
        per_entry(w, o, [&](DevBuf& buf, size_t width) { buf.ensure(entries * width); });
    }

    // Sizes every workspace array but the per-entry ones (ensure_entries) for batches of up to n_sent sentences /
    // n_bytes bytes (upper bounds: characters <= bytes, one sentinel slot per sentence) and `cands` candidates.
    void ensure_workspace(Workspace& w, uint32_t n_sent, uint64_t n_bytes, size_t cands, bool bounded, bool spans) {
        const size_t ns = size_t(n_sent) + 1;
        w.n_slots.ensure(ns * 4, 1.25);
        w.slot_off.ensure(ns * 4, 1.25);
        w.eos.ensure(ns * 16, 1.25);
        w.n_tok.ensure(ns * 4, 1.25);
        w.tiles.ensure(size_t(scan_tiles(n_sent, kFrontTile) + scan_tiles(n_sent, kBackTileSmall)) * 8 + 8, 1.25);
        if (order_mode_ == 1) {
            w.iota.ensure(ns * 4, 1.25);
            w.sort_keys.ensure(ns * 4, 1.25);
        }
        if (order_mode_) w.order.ensure(ns * 4, 1.25);
        const size_t ms = size_t(n_bytes) + n_sent + 1;
        w.code_sys.ensure(ms * 4, 1.25);
        if (dv_.usr_table) w.code_usr.ensure(ms * 4, 1.25);
        w.cinfo.ensure(ms * 4, 1.25);
        w.groupable.ensure(ms * 4, 1.25);
        w.byte_pos.ensure(ms * 4, 1.25);
        w.info.ensure(ms * 8, 1.25);
        w.info_ex.ensure(ms * 8, 1.25);
        w.ends_cnt.ensure(ms * 4, 1.25);
        w.ends_meta.ensure(ms * 8, 1.25);
        if (bounded) w.bnd_dist.ensure(ms * 4, 1.25);
        if (spans) w.span_tag.ensure(ms * 8, 1.25);
        const PassPlan p = plan();
        if (p.fwd != kFwdNone) {
            w.m_fill.ensure(ms * 4, 1.25);
            w.m_ncand.ensure(ms * 4, 1.25);
            w.m_r_eos.ensure(ns * 8, 1.25);
        }
        if (p.fwd >= kFwdLse) w.m_a_eos.ensure(ns * 8, 1.25);
        if (p.lat) {
            w.l_row_base.ensure(ms * 4, 1.25);
            w.l_n_nodes.ensure(ns * 4, 1.25);
        }
        if (counting_) w.stats.ensure(ms * 16, 1.25);
        w.seg.ensure(cands * 8);  // sized like the candidates; move segments can outnumber them (overflow retry)
        const size_t walks = size_t(n_sent) * p.samp + 1;
        if (p.samp) {
            w.s_cnt.ensure(walks * 4, 1.25);
            w.s_total.ensure(walks * 4, 1.25);
        }
        if (p.post) {
            w.p_V.ensure(ms * 8, 1.25);
            w.p_A.ensure(ms * 4, 1.25);
            w.p_cnt.ensure(ns * 4, 1.25);
            w.p_total.ensure(ns * 4, 1.25);
        }
        size_t tmp = 0;  // cub temp storage for the largest scan / sort of this size
        cub::DeviceScan::ExclusiveSum(nullptr, tmp, static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr), ms, w.stream);
        w.scan_tmp.ensure(tmp + 1024, 1.5);
        const size_t group = std::max(p.lat || p.post ? ns : 0, p.samp ? walks : 0);  // the longest scan_group
        if (group) {
            cub::DeviceScan::ExclusiveSum(nullptr, tmp, CountsU64(nullptr, CastU64()), static_cast<unsigned long long*>(nullptr), group, w.stream);
            w.scan_tmp.ensure(tmp + 1024, 1.5);
        }
        if (order_mode_ == 1) {
            cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp, static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                                      static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr), int(ns), 0,
                                                      32, w.stream);
            w.scan_tmp.ensure(tmp + 1024, 1.5);
        }
    }

    // One whole batch from device-resident input into out_[0]; synchronises, retries on pool overflow.
    // sent_base: the caller's index of the first sentence (a shard's place in the batch), for the sampling draws.
    // sink (small host batches): a result the outputs are copied into right behind the kernels (enqueue).
    void run_whole(const uint8_t* d_utf8, const unsigned long long* d_off, uint32_t n_sent, uint64_t n_bytes,
                   const DevBounds& bd, uint64_t sent_base = 0, HostResult* sink = nullptr) {
        OutSlot& o = out_[0];
        ws_[0].stream = stream_;
        batch_total_bytes_ = n_bytes;
        for (int attempt = 0;; ++attempt) {
            const size_t cands = want_cand(n_bytes);
            ensure_workspace(ws_[0], n_sent, n_bytes, cands, bd.off != nullptr, bd.span_off != nullptr);
            ensure_out(o, n_sent, n_bytes);
            ensure_entries(ws_[0], o, cands + n_sent + 1);
            connid_begin(stream_);
            enqueue(ws_[0], d_utf8, d_off, n_sent, n_bytes, o, nullptr, nullptr, nullptr, bd, sent_base, sink);
            CK(cudaEventSynchronize(o.done));
            CK(cudaGetLastError());
            throw_input_error(o.h_ctrl->flags);
            // more characters per byte than any batch before: the next attempt takes the hard bound, and only then
            // counts its candidates in full
            const uint32_t why = o.h_ctrl->flags & kFlagSlotsOverflow ? kFlagSlotsOverflow : o.h_ctrl->flags;
            const double need = double(pool_need(*o.h_ctrl));
            if ((why & kFlagPoolOverflow) && need * 1.05 + 4096 >= double(0xFFFFFFF0ull))
                throw Error(kInvalidArgument, "batch produces more than 2^32 lattice nodes: split it");
            if (rerun(why, attempt)) {
                if (why & kFlagSlotsOverflow) chars_per_byte_ = 1.0;
                if (why & kFlagPoolOverflow) cand_per_byte_ = need / double(std::max<uint64_t>(1, n_bytes)) * 1.05 + 1e-3;
                continue;
            }
            if (n_bytes) cand_per_byte_ = std::max(0.25, need / double(n_bytes) * 1.15);
            if (n_bytes) chars_per_byte_ = std::min(1.0, double(o.h_ctrl->total_slots - n_sent) / double(n_bytes) * 1.10);
            connid_commit(stream_);
            break;
        }
        clear_stats();
        last_route_ = add_stats(o);
    }

    // Ends an attempt that finished with `flags` and no input error: books each re-run reason they hold in reruns_ and
    // says whether to run again.  An overflow that persists after three re-runs throws.
    bool rerun(uint32_t flags, int attempt) {
        bool again = false;
        for (int k = 0; k < kNumReruns; ++k) {
            if (!(flags & kRerunFlags[k])) continue;
            if (attempt >= 3) throw Error(kInternal, kRerunPersists[k]);
            ++reruns_[k];
            again = true;
        }
        return again;
    }

    // The statistics of a call: zeroed once per attempt, then each finished slot (a whole batch, or every chunk) adds
    // its stage times, launches and counters.  add_stats returns the slot's Viterbi route as resolved by its flags.
    void clear_stats() {
        std::memset(stage_ms_, 0, sizeof(stage_ms_));
        std::memset(counters_, 0, sizeof(counters_));
        launches_ = 0;
    }
    uint32_t add_stats(const OutSlot& o) {
        for (int i = 0; i < kNumStages; ++i) {
            float ms = 0;
            CK(cudaEventElapsedTime(&ms, o.ev[i], o.ev[i + 1]));
            stage_ms_[i] += ms;
        }
        launches_ += o.launches;
        if (counting_)
            for (int i = 0; i < kNumCounters; ++i) counters_[i] += o.h_ctrl->counters[i];
        return resolve_viterbi_route(o.route, o.h_ctrl->flags);
    }

    // Queues the whole kernel sequence for one (chunk of a) batch on stream_; no host synchronisation.
    // `base` (device, chunked runs only: one running total per group) makes the chunk's offsets global and is advanced
    // by its record counts.  A chunk with the output stage on is formatted into its text buffer up to its capacity
    // (kFlagTextOverflow beyond).
    void enqueue(Workspace& w, const uint8_t* d_utf8, const unsigned long long* d_off, uint32_t n_sent, uint64_t n_bytes,
                 OutSlot& o, unsigned long long* base, cudaEvent_t base_wait, cudaEvent_t base_signal, const DevBounds& bd,
                 uint64_t sent0, HostResult* sink = nullptr) {
        cudaStream_t st = w.stream;
        o.made = outputs();
        if (!base) o.made.text = false;  // whole batches and shards are formatted by format_whole
        // characters <= bytes is the hard bound; the per-character launches are sized from the ratio learned on
        // earlier batches (plus slack), and a batch that exceeds it flags itself and is re-run with the hard bound
        const uint32_t hard_slots = uint32_t(n_bytes + n_sent);
        const uint32_t max_slots = uint32_t(std::min<uint64_t>(hard_slots, uint64_t(double(n_bytes) * chars_per_byte_) + n_sent + 4096));
        // the candidates the pool may take: every per-entry array also holds one EOS entry per sentence
        size_t cap_all = 0xFFFFFFF0ull;
        per_entry(w, o, [&](const DevBuf& buf, size_t width) {
            const size_t rows = buf.cap / width;
            cap_all = std::min<size_t>(cap_all, rows > n_sent ? rows - n_sent - 1 : 0);
        });
        const uint32_t cand_cap = uint32_t(cap_all);
        const PassPlan p = plan();
        Batch b{};
        b.utf8 = d_utf8;
        b.byte_off = d_off;
        b.total_bytes = batch_total_bytes_;
        b.n_sent = n_sent;
        b.launch_slots = max_slots;
        b.n_slots = w.n_slots.as<uint32_t>();
        b.slot_off = w.slot_off.as<uint32_t>();
        b.order = (order_mode_ && n_sent > 1) ? w.order.as<uint32_t>() : nullptr;
        b.eos = w.eos.as<uint4>();
        b.n_tok = w.n_tok.as<uint32_t>();
        b.tok_off = o.buf[kTokOff].as<unsigned long long>();
        b.code_sys = w.code_sys.as<uint32_t>();
        b.code_usr = w.code_usr.as<uint32_t>();
        b.cinfo = w.cinfo.as<uint32_t>();
        b.groupable = w.groupable.as<uint32_t>();
        b.byte_pos = w.byte_pos.as<uint32_t>();
        b.info = w.info.as<uint2>();
        b.info_ex = w.info_ex.as<uint2>();
        b.ends_cnt = w.ends_cnt.as<uint32_t>();
        b.ends_meta = w.ends_meta.as<uint2>();
        b.seg = w.seg.as<uint2>();
        b.seg_cap = uint32_t(std::min<size_t>(w.seg.cap / 8, 0xFFFFFFF0ull));
        b.cand_cap = cand_cap;
        b.ends_hot = w.ends_hot.as<int2>();
        b.ends_cold = w.ends_cold.as<uint4>();
        b.tokens = o.buf[kTokens].p;
        b.compact = tok_bytes_ == 16 ? 1u : 0u;
        Control* dc = o.ctrl.as<Control>();
        b.pool_ctr = &dc->pool_ctr;
        b.seg_ctr = &dc->seg_ctr;
        b.flags = &dc->flags;
        b.counters = counting_ ? dc->counters : nullptr;
        // counts go to a per-attempt scratch: an attempt that ends in a pool overflow or an input error is re-run
        // or dropped, and must not leave its partial counts behind (lattice.rs:170-181 counts a lattice once)
        b.lid_count = connid_on_ ? connid_try_.as<unsigned long long>() : nullptr;
        b.rid_count = connid_on_ ? connid_try_.as<unsigned long long>() + num_left_ : nullptr;
        if (bd.off) {
            b.bnd_off = bd.off;
            b.bnd = bd.bnd;
            b.n_bnd = bd.n;
            b.bnd_dist = w.bnd_dist.as<uint32_t>();
        }
        SpanArgs sp{};
        if (bd.span_off) {
            sp = SpanArgs{bd.span_off, bd.span_rec, bd.n_spans, bd.pat_off, bd.pf, bd.pat_bytes, bd.n_pat, dv_.space_mask,
                          w.span_tag.as<uint2>()};
        }

        o.launches = 0;
        const TileScan ts{w.tiles.as<unsigned long long>(), dc->tickets};
        CK(cudaMemsetAsync(dc, 0, sizeof(Control), st));
        CK(cudaMemsetAsync(ts.state, 0, size_t(scan_tiles(n_sent, kFrontTile) + scan_tiles(n_sent, kBackTileSmall)) * 8, st));
        // count_chars and scan_slots are folded into k_front, which is booked under decode
        CK(cudaEventRecord(o.ev[0], st));
        CK(cudaEventRecord(o.ev[1], st));
        CK(cudaEventRecord(o.ev[2], st));
        if (n_sent) {
            launch_front(dv_, b, ts, st);
            // front, candidates, the row-offset scan (two cub kernels), backtrack, publish (+ viterbi below)
            o.launches += 6;
        } else {
            CK(cudaMemsetAsync(b.slot_off, 0, 4, st));
        }
        if (b.order && order_mode_ == 2) {
            k_local_order<<<(n_sent + kOrderTile - 1) / kOrderTile, kOrderTile, 0, st>>>(b.n_slots, n_sent, w.order.as<uint32_t>());
            ++o.launches;
        } else if (b.order) {
            // K3 walks several sentences per warp in lockstep: group sentences of similar length
            // (longest first, which also trims the tail of the launch)
            k_iota<<<(n_sent + 255) / 256, 256, 0, st>>>(w.iota.as<uint32_t>(), n_sent);
            size_t cap = w.scan_tmp.cap;
            CK(cub::DeviceRadixSort::SortPairsDescending(w.scan_tmp.p, cap, b.n_slots, w.sort_keys.as<uint32_t>(),
                                                         w.iota.as<uint32_t>(), w.order.as<uint32_t>(), int(n_sent), 0, 32,
                                                         st));
            ++o.launches;
        }
        if (b.bnd_dist && n_sent) {  // the bounded batch's boundaries (and spans), booked with the decode stage
            if (sp.off)
                launch_mark_spans(b, sp, st);
            else
                launch_mark_bounds(b, st);
            ++o.launches;
        }
        CK(cudaEventRecord(o.ev[3], st));
        launch_candidates(dv_, b, max_slots, st, sp.off ? &sp : nullptr);
        if (counting_) {
            launch_candidate_stats(dv_, b, max_slots, w.stats.as<uint4>(), st);
            ++o.launches;
        }
        CK(cudaEventRecord(o.ev[4], st));
        exclusive_scan(w, b.ends_cnt, RowMetaOut{b.ends_meta}, size_t(max_slots) + 1);
        CK(cudaEventRecord(o.ev[5], st));
        o.launches += launch_viterbi(dv_, b, counting_ ? w.stats.as<uint4>() : nullptr, lanes_, viterbi_kernel_, st, &o.route);
        MargArgs m{};
        UncertaintyArgs u{};
        MarginArgs g{};
        if (p.fwd != kFwdNone) {  // booked with the Viterbi stage; must run before K4 reuses ends_meta
            m.theta = theta_ > 0 ? theta_ : samp_theta_;  // equal when both are on (set_marginals / set_sampling)
            m.fill = w.m_fill.as<uint32_t>();
            m.ncand = w.m_ncand.as<uint32_t>();
            m.cand_entry = w.m_cand_entry.as<uint32_t>();
            m.R = w.m_R.as<long long>();
            m.ab = w.m_ab.as<double2>();
            m.r_eos = w.m_r_eos.as<long long>();
            m.a_eos = w.m_a_eos.as<double>();
            m.path_prob = o.buf[kPathProb].as<float>();
            m.token_prob = p.bwd != kBwdNone ? o.buf[kTokenProb].as<float>() : nullptr;
            m.lw = p.fwd == kFwdLseLw ? w.m_lw.as<uint32_t>() : nullptr;
            if (p.bwd == kBwdUnc) u = UncertaintyArgs{o.buf[kEntropy].as<double>(), o.buf[kLogPathProb].as<double>()};
            if (p.bprob) {
                u.pos_off = o.buf[kPosOff].as<unsigned long long>();
                u.boundary_prob = o.buf[kBoundaryProb].as<float>();
                if (n_sent == 0) CK(cudaMemsetAsync(u.pos_off, 0, 8, st));
                // the group's records: one per slot (the low word of a total zeroed with the rest of Control)
                CK(cudaMemcpyAsync(&dc->total[kGroupPositions], b.slot_off + n_sent, 4, cudaMemcpyDeviceToDevice, st));
            }
            if (p.margin)  // G of every entry, from the R of the forward pass
                g = MarginArgs{lat_margin_, w.g_G.as<long long>(), w.g_keep.as<uint32_t>(), o.buf[kNodeMargin].as<long long>()};
            launch_marginals(dv_, b, m, p.fwd, p.bwd, u, p.margin ? &g : nullptr, st);
            if (n_sent) o.launches += 1 + (p.bwd != kBwdNone) + p.bprob + p.margin;
        }
        if (p.lat) {  // booked with the Viterbi stage too, and also before K4
            LatticeArgs l{};
            l.row_base = w.l_row_base.as<uint32_t>();
            l.n_nodes = w.l_n_nodes.as<uint32_t>();
            l.node_off = o.buf[kNodeOff].as<unsigned long long>();
            l.nodes = o.buf[kNodes].as<uint2>();
            l.links = o.buf[kLinks].as<int2>();
            l.node_prob = p.bwd != kBwdNone ? o.buf[kNodeProb].as<float>() : nullptr;
            launch_lattice_count(b, l, m, p.margin ? &g : nullptr, st);
            scan_group(w, l.n_nodes, l.node_off, n_sent, &dc->total[kGroupLattice]);
            launch_lattice_write(b, l, m, p.margin ? &g : nullptr, st);
            if (n_sent) o.launches += 2;
        }
        if (p.samp) {  // booked with the Viterbi stage too, and also before K4
            SampleArgs sa{};
            sa.n = p.samp;
            sa.seed = samp_seed_;
            sa.sent_base = sample_base_ + sent0;
            sa.cnt = w.s_cnt.as<uint32_t>();
            sa.total = w.s_total.as<int32_t>();
            sa.off = o.buf[kSampleOff].as<unsigned long long>();
            const size_t walks = size_t(n_sent) * p.samp;
            launch_sample_count(dv_, b, m, sa, st);
            scan_group(w, sa.cnt, sa.off, walks, &dc->total[kGroupSamples]);
            // the records are sized from the scanned total: one wait for it here
            CK(cudaMemcpyAsync(&o.h_ctrl->total[kGroupSamples], sa.off + walks, 8, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            o.buf[kSamples].ensure(size_t(o.h_ctrl->total[kGroupSamples]) * 24 + 24, 1.25);
            sa.out = o.buf[kSamples].as<uint2>();
            launch_sample_write(dv_, b, m, sa, st);
            if (walks) o.launches += 2;
        }
        if (p.post) {  // booked with the Viterbi stage too, and also before K4; marginals are on (set_posterior)
            PosteriorArgs q{};
            q.g1 = post_g1_;
            q.V = w.p_V.as<double>();
            q.A = w.p_A.as<uint32_t>();
            q.cnt = w.p_cnt.as<uint32_t>();
            q.total = w.p_total.as<int32_t>();
            q.off = o.buf[kPostOff].as<unsigned long long>();
            q.out = o.buf[kPostTokens].as<uint2>();
            q.prob = o.buf[kPostProb].as<float>();
            q.gain = o.buf[kPostGain].as<double>();
            launch_posterior_sweep(dv_, b, m, q, st);
            scan_group(w, q.cnt, q.off, n_sent, &dc->total[kGroupPosterior]);
            launch_posterior_write(dv_, b, m, q, st);
            if (n_sent) o.launches += 2;
        }
        // backtrack_count and scan_tokens are folded into k_backtrack, which is booked under backtrack_write
        CK(cudaEventRecord(o.ev[6], st));
        CK(cudaEventRecord(o.ev[7], st));
        CK(cudaEventRecord(o.ev[8], st));
        if (n_sent)
            launch_backtrack(b, p.bwd != kBwdNone ? &m : nullptr, ts, st);
        else
            CK(cudaMemsetAsync(b.tok_off, 0, 8, st));
        k_publish_totals<<<1, 1, 0, st>>>(b.slot_off, b.tok_off, n_sent, dc);
        if (o.made.text) {  // output stage of a chunk: formatted while its token offsets are still chunk-local
            FormatArgs f = format_offsets(w, d_utf8, d_off, n_sent, o);
            format_write(f, o, st);
            o.launches += 2;
        }
        if (base) {
            if (base_wait) CK(cudaStreamWaitEvent(st, base_wait, 0));  // the previous chunk (other stream) bumped it
            for (int g = 0; g < kNumGroups; ++g) {
                const int a = kOffsetsOf[g];
                if (!o.made.has(a)) continue;
                const size_t n = size_t(n_sent) * o.made.stride(a) + 1;
                k_add_base<<<unsigned((n + 255) / 256), 256, 0, st>>>(o.buf[a].as<unsigned long long>(), uint32_t(n), base + g);
                k_bump_base<<<1, 1, 0, st>>>(base + g, &dc->total[g]);
                o.launches += 2;
            }
            if (base_signal) CK(cudaEventRecord(base_signal, st));
        }
        CK(cudaEventRecord(o.ev[9], st));
        CK(cudaMemcpyAsync(o.h_ctrl, dc, sizeof(Control), cudaMemcpyDeviceToHost, st));
        // small batch: results leave in the same breath (sized by their upper bound, a token per byte)
        if (sink) place(o, sink, 0, n_sent, Totals{n_bytes, 0, 0, 0}, Totals{}, true, st);
        CK(cudaEventRecord(o.done, st));
    }

    int device_;
    static constexpr int kRingSlots = 4;
    static constexpr size_t kRingBytes = size_t(4) << 20;
    uint8_t* ring_[kRingSlots] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ring_ev_[kRingSlots] = {nullptr, nullptr, nullptr, nullptr};
    int ring_next_ = 0;
    static constexpr uint64_t kEagerBytes = 16384;
    uint32_t small_batch_ = 0;  // "small_batch": the most sentences k_small_batch takes (0 = the route is off)
    Workspace ws_small_;        // scratch of k_small_batch (its stream is unused)
    DevBuf small_in_, small_out_;
    uint8_t* small_in_h_ = nullptr;  // pinned staging of the input / output region (ensure_small)
    uint8_t* small_out_h_ = nullptr;
    size_t small_in_cap_ = 0, small_out_cap_ = 0;
    uint32_t shard_n_sent_ = 0;
    cudaStream_t stream_ = nullptr, own_stream_ = nullptr, in_stream_ = nullptr, out_stream_ = nullptr;
    cudaEvent_t in_done_ = nullptr;
    std::vector<cudaEvent_t> h2d_ev_;
    OutSlot out_[2];
    DevBuf base_;  // chunked host batches: the running total of each group's records (enqueue)
    uint32_t chunk_sentences_ = 262144;
    double tok_per_byte_ = 0.2;
    DictView dv_{};
    const uint8_t* blob_ = nullptr;
    DevBuf blob_own_, in_utf8_, in_off_, connid_, connid_try_;
    DevBuf in_bnd_off_, in_bnd_;           // boundary lists of a bounded host batch (upload_bounds)
    DevBuf in_span_off_, in_span_, in_pat_;  // span lists of a host batch, and any span batch's compiled patterns
    std::vector<uint64_t> bnd_rebased_, span_rebased_;
    uint64_t* bnd_stage_ = nullptr;  // pinned: device-resident boundary offsets checked for emptiness
    size_t bnd_stage_cap_ = 0;
    bool connid_on_ = false;
    uint32_t num_left_ = 0, num_right_ = 0;
    std::vector<uint16_t> left_ids_, right_ids_;
    Workspace ws_[2];
    cudaStream_t aux_stream_ = nullptr;
    cudaEvent_t base_ready_[2] = {nullptr, nullptr};
    ResultPool pool_;
    std::vector<uint64_t> rebased_;
    double cand_per_byte_ = 4.0;
    double chars_per_byte_ = 1.0;  // learned; 1.0 = the hard bound (every byte a character)
    bool counting_ = false;
    int order_mode_ = 0;  // K3's sentence order: 0 input order, 1 whole batch by length, 2 by length inside tiles
    uint32_t output_mode_ = 0;
    uint64_t batch_total_bytes_ = 0;  // size of the input buffer of the batch in flight (bounds check in K1)
    TextRatios text_per_byte_ = kTextPerByte;  // sizes the text buffers of the chunked pipeline, learned like cand_per_byte_
    double node_per_byte_ = 2.0;  // lattice nodes per input byte: sizes the host result of the chunked pipeline
    uint32_t text_per_sent_ = 4;  // "EOS\n"; an output format: what its BOS and EOS print (FormatProgram::per_sentence)
    // output format (set_format): the compiled program and its field table, with the table's size and build time
    DevBuf fmt_prog_, ft_keep_, ft_off_, ft_bytes_;
    uint32_t fmt_uses_ = 0;  // FormatProgram::uses of the output format
    size_t ft_size_ = 0;
    float ft_ms_ = 0;
    bool dual_stream_ = false;
    int lanes_ = 16;  // fastest on H100 for ~40-character and 512-character sentences alike (DESIGN.md §4)
    uint32_t tok_bytes_ = 24;
    int viterbi_kernel_ = 1;  // 1 = k_viterbi2 with pruning (kernels.cuh)
    double theta_ = 0;        // marginals' theta, 0 = off (set_marginals)
    bool lattice_ = false;    // option "lattice" >= 1
    TextSrc text_src_ = kTextBest;  // what the output text renders (set_text)
    static constexpr long long kMaxLatticeMargin = 1ll << 62;
    long long lat_margin_ = -1;  // option "lattice_margin": the near-best lattice's D, -1 = off
    uint32_t unc_ = 0;           // option "uncertainty": 0 off, 1 entropy and log_path_prob, 2 also boundary probabilities
    static constexpr uint32_t kMaxSamples = 1024;
    uint32_t samp_n_ = 0;       // sampling: paths per sentence, 0 = off (set_sampling)
    double samp_theta_ = 0;
    uint64_t samp_seed_ = 0;
    bool post_ = false;         // posterior decoding (set_posterior)
    double post_g1_ = 0;        // its gamma + 1
    static constexpr long long kMaxSampleBase = 0x100000000ll;
    uint64_t sample_base_ = 0;  // option "sample_base": the draws' index of the call's first sentence
    DeviceOutputs last_;  // what the last run_device or run_shard left in out_[0] (last_device)
    float stage_ms_[kNumStages];
    uint64_t launches_ = 0;
    uint32_t last_route_ = kRouteNone;  // ViterbiRoute of the last successful call (describe())
    Reruns reruns_{};                    // the attempts the last call re-ran, by reason (describe())
    uint64_t counters_[kNumCounters];
};

}  // namespace

std::unique_ptr<Engine> Engine::create(int device, const uint8_t* host_blob, uint64_t d_blob, uint64_t n_bytes,
                                       bool ignore_space, uint64_t max_grouping_len) {
    return std::unique_ptr<Engine>(new EngineImpl(device, host_blob, d_blob, n_bytes, ignore_space, max_grouping_len));
}

void DevBuf::ensure(size_t bytes, double slack) {
    if (bytes <= cap) return;
    if (p) CK(cudaFree(p));
    p = nullptr;
    cap = 0;
    size_t want = size_t(double(bytes) * slack) + 256;
    CK(cudaMalloc(&p, want));
    cap = want;
}

void DevBuf::release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
}

PinnedBuf::~PinnedBuf() { pinned_free(p); }

void PinnedBuf::ensure(size_t bytes) {
    if (p && bytes <= cap) return;  // an array is allocated even when empty
    pinned_free(p);
    p = nullptr;
    cap = size_t(double(bytes) * 1.25) + 64;
    p = pinned_alloc(cap);
}

void PinnedBuf::grow(size_t bytes, size_t keep_bytes) {
    if (p && bytes <= cap) return;
    const size_t want = size_t(double(bytes) * 1.5) + 4096;
    void* bigger = pinned_alloc(want);
    if (keep_bytes) std::memcpy(bigger, p, keep_bytes);
    pinned_free(p);
    p = bigger;
    cap = want;
}

HostResult* ResultPool::acquire(const Outputs& out, uint64_t n_sent, const Totals& total) {
    if (free_.empty()) {
        all_.emplace_back(new HostResult());
        free_.push_back(all_.back().get());
    }
    HostResult* r = free_.back();
    free_.pop_back();
    r->n_sent = n_sent;
    r->out = out;
    r->total = total;
    for (int a = 0; a < kNumArrays; ++a) {
        if (!out.has(a)) continue;
        r->buf[a].ensure(out.bytes(a, n_sent, total, true));
        if (kArrays[a].kind == kOffsets && n_sent == 0) *r->ptr<uint64_t>(a) = 0;
    }
    return r;
}

void* pinned_alloc(size_t n) {
    void* p = nullptr;
    cuda_check(cudaHostAlloc(&p, n ? n : 1, cudaHostAllocDefault), "cudaHostAlloc");
    return p;
}

void pinned_free(void* p) {
    if (p) cudaFreeHost(p);
}

}  // namespace vbt
