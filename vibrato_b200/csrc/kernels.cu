// Hand-written sm_90a (H100) kernels of the batched Viterbi tokenizer.
//
//   K1  front           warp / sentence   UTF-8 validation + character count, slot offsets (look-back scan),
//                                         code points -> CharInfo, trie codes, c2b, groupable
//   K2  candidates      thread / char     common-prefix walks (user, system) + unknown words
//   K3  viterbi         warp / sentence   left-to-right min-plus DP over the lattice + EOS
//   K4  backtrack       thread / sentence best path, token offsets (look-back scan), then thread / token records
//
// Everything is integer gather / compare work: no tensor cores.  Citations are relative to
// /root/reference/vibrato/src/ and name the reference routine whose RESULT each step reproduces.
#include "kernels.cuh"

#include <climits>
#include <type_traits>

// Minimum resident blocks per SM asked of ptxas for k_viterbi (128 threads each): 16 -> 32 registers,
// 64 warps/SM.  The counting and Raw/Dual instantiations are not on the timed path and get 64 registers.
#ifndef VBT_K3_MIN_BLOCKS
#define VBT_K3_MIN_BLOCKS 16
#endif

namespace vbt {

namespace {

constexpr uint32_t kMask = 0x7FFFFFFFu;
constexpr uint32_t kFlag = 0x80000000u;
constexpr unsigned kFull = 0xFFFFFFFFu;

// A batch whose byte offsets k_front refused is not touched by any later kernel: the sizes derived from
// the offsets (slots, workspace bounds) cannot be trusted.
__device__ __forceinline__ bool stand_down(uint32_t batch_flags) { return batch_flags & kFlagsStandDown; }
// The lattice rows of a batch that overflowed its candidate pool (it is run again) cannot be read either: the
// boundary-probability, lattice and sampling kernels take nothing from such a batch or a refused one.
__device__ __forceinline__ bool rows_unreadable(uint32_t batch_flags) {
    return batch_flags & (kFlagsStandDown | kFlagPoolOverflow);
}

// CharInfo bit fields (dictionary/character.rs:10-24,72-94)
__device__ __forceinline__ uint32_t ci_cate(uint32_t ci) { return ci & 0x3FFFFu; }
__device__ __forceinline__ uint32_t ci_base(uint32_t ci) { return (ci >> 18) & 0xFFu; }
__device__ __forceinline__ bool ci_invoke(uint32_t ci) { return (ci >> 26) & 1u; }
__device__ __forceinline__ bool ci_group(uint32_t ci) { return (ci >> 27) & 1u; }
__device__ __forceinline__ uint32_t ci_length(uint32_t ci) { return ci >> 28; }

__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// ---------------------------------------------------------------------------------------------
// Characters per sentence + UTF-8 validity (what `&str` guarantees before worker.rs:34)
// ---------------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t utf8_len_checked(const uint8_t* p, unsigned long long i, unsigned long long len,
                                                     uint32_t c, bool& bad) {
    uint32_t L;
    if (c < 0x80) return 1;
    if (c >= 0xC2 && c <= 0xDF)
        L = 2;
    else if (c >= 0xE0 && c <= 0xEF)
        L = 3;
    else if (c >= 0xF0 && c <= 0xF4)
        L = 4;
    else {
        bad = true;
        return 1;
    }
    if (i + L > len) {
        bad = true;
        return 1;
    }
    uint32_t c1 = p[i + 1];
    if ((c1 & 0xC0) != 0x80) bad = true;
    if (L >= 3 && (p[i + 2] & 0xC0) != 0x80) bad = true;
    if (L == 4 && (p[i + 3] & 0xC0) != 0x80) bad = true;
    if (c == 0xE0 && c1 < 0xA0) bad = true;  // overlong
    if (c == 0xED && c1 > 0x9F) bad = true;  // surrogates
    if (c == 0xF0 && c1 < 0x90) bad = true;
    if (c == 0xF4 && c1 > 0x8F) bad = true;
    return L;
}

// Sentences per warp of the warp-per-sentence kernels (k_mark_bounds, the marginals): a warp walks a few consecutive sentences so
// that the grid has fewer, longer-lived blocks.
#ifndef VBT_SENT_PER_WARP
#define VBT_SENT_PER_WARP 4
#endif

// Characters of the sentence in p[0, len) (shared or global memory) with the validity rules of `&str`; lane 0 raises the
// batch flags, adds the counters and stores and returns the sentence's slots (characters + 1), 1 for invalid UTF-8.
__device__ __forceinline__ uint32_t count_chars_at(const Batch& b, const uint8_t* p, unsigned long long len, uint32_t* n_slots,
                                                   uint32_t lane) {
    unsigned long long nchar = 0, covered = 0;
    bool bad = false;
    for (unsigned long long i0 = 0; i0 < len; i0 += 32) {
        unsigned long long i = i0 + lane;
        if (i < len) {
            uint32_t c = p[i];
            if ((c & 0xC0) != 0x80) {
                covered += utf8_len_checked(p, i, len, c, bad);
                ++nchar;
            }
        }
    }
    nchar = warp_sum(nchar);
    covered = warp_sum(covered);
    bool any_bad = __any_sync(kFull, bad);
    if (lane == 0) {
        if (any_bad || covered != len || nchar >= 0xFFFFFFF0ull) {
            atomicOr(b.flags, kFlagUtf8Error);
            nchar = 0;  // keep the rest of the pipeline in bounds; the batch is rejected anyway
        }
        *n_slots = uint32_t(nchar) + 1;
        if (nchar > kPruneMaxChars) atomicOr(b.flags, kFlagLongSentence);
        if (b.counters) {
            atomicAdd(&b.counters[kCntU], len);
            atomicAdd(&b.counters[kCntC], nchar);
        }
    }
    return uint32_t(nchar) + 1;
}

__device__ __forceinline__ void count_chars_one(const Batch& b, uint32_t s, uint32_t lane) {
    unsigned long long bo = b.byte_off[s], len = b.byte_off[s + 1] - bo;
    if (b.byte_off[s + 1] < bo || b.byte_off[s + 1] > b.total_bytes) {  // caller error: nothing of this sentence is read
        if (lane == 0) {
            atomicOr(b.flags, kFlagBadOffsets);
            b.n_slots[s] = 1;
        }
        return;
    }
    count_chars_at(b, b.utf8 + bo, len, &b.n_slots[s], lane);
}

// ---------------------------------------------------------------------------------------------
// Sentence::compile (sentence.rs:34-71) for every sentence
// ---------------------------------------------------------------------------------------------

__device__ __forceinline__ void decode_one(const DictView& d, const Batch& b, uint32_t s, uint32_t lane) {
    unsigned long long bo = b.byte_off[s], len = b.byte_off[s + 1] - bo;
    const uint8_t* p = b.utf8 + bo;
    const uint32_t base = b.slot_off[s];
    const uint32_t n = b.slot_off[s + 1] - base - 1;
    if (n > 0) {  // n == 0 also covers a batch already flagged as invalid UTF-8
        uint32_t running = 0;
        for (unsigned long long i0 = 0; i0 < len; i0 += 32) {
            unsigned long long i = i0 + lane;
            uint32_t c = i < len ? p[i] : 0x80u;
            bool lead = (c & 0xC0) != 0x80;
            uint32_t m = __ballot_sync(kFull, lead);
            if (lead) {
                uint32_t idx = running + __popc(m & lanemask_lt());
                uint32_t c1 = i + 1 < len ? p[i + 1] : 0, c2 = i + 2 < len ? p[i + 2] : 0, c3 = i + 3 < len ? p[i + 3] : 0;
                uint32_t cp;  // compute_basic sentence.rs:40-46
                if (c < 0x80)
                    cp = c;
                else if (c < 0xE0)
                    cp = ((c & 0x1F) << 6) | (c1 & 0x3F);
                else if (c < 0xF0)
                    cp = ((c & 0x0F) << 12) | ((c1 & 0x3F) << 6) | (c2 & 0x3F);
                else
                    cp = ((c & 0x07) << 18) | ((c1 & 0x3F) << 12) | ((c2 & 0x3F) << 6) | (c3 & 0x3F);
                if (idx < n) {
                    uint32_t slot = base + idx;
                    b.byte_pos[slot] = uint32_t(i);
                    // CharProperty::char_info character.rs:112-116: out-of-table code points use entry 0
                    b.cinfo[slot] = __ldg(&d.chr2inf[cp < d.chr2inf_len ? cp : 0]);
                    b.code_sys[slot] = cp < d.sys_table_len ? __ldg(&d.sys_table[cp]) : kInvalidCode;
                    if (d.usr_table) b.code_usr[slot] = cp < d.usr_table_len ? __ldg(&d.usr_table[cp]) : kInvalidCode;
                    b.ends_cnt[slot] = idx == 0 ? 1u : 0u;  // BOS lives in ends[0] (lattice.rs:72-83)
                }
            }
            running += __popc(m);
        }
    }
    if (lane == 0) {  // sentinel slot == character position n
        uint32_t slot = base + n;
        b.byte_pos[slot] = uint32_t(len);
        b.cinfo[slot] = 0;
        b.groupable[slot] = 0;
        b.code_sys[slot] = kInvalidCode;
        if (d.usr_table) b.code_usr[slot] = kInvalidCode;
        b.ends_cnt[slot] = 0;
        b.info[slot] = make_uint2(0, 0);
    }
    __syncwarp();
    // compute_groupable sentence.rs:57-71: distance to the end of the run in which adjacent
    // characters share a category bit, solved per 32-character chunk from the right.
    uint32_t carry = 0;
    for (int k = int((n + 31) / 32) - 1; k >= 0; --k) {
        uint32_t c = uint32_t(k) * 32 + lane;
        bool valid = c < n;
        uint32_t ci = valid ? b.cinfo[base + c] : 0;
        uint32_t cn = (c + 1 < n) ? b.cinfo[base + c + 1] : 0;
        bool brk = valid && (c + 1 == n || (ci_cate(ci) & ci_cate(cn)) == 0);
        uint32_t bm = __ballot_sync(kFull, brk);
        uint32_t clen = min(32u, n - uint32_t(k) * 32);
        uint32_t m = bm >> lane;
        uint32_t g = m ? uint32_t(__ffs(m)) : (clen - lane) + carry;
        if (valid) b.groupable[base + c] = g;
        carry = __shfl_sync(kFull, g, 0);
    }
}

// decode_one for a sentence of n <= kFrontWarpChars characters in p[0, len) (shared or global memory), a lane per
// character: buf (the warp's, in shared memory) first maps characters to their lead bytes and then holds their CharInfo
// for groupable, so that every array is written 32 consecutive slots at a time and nothing is read back.
constexpr uint32_t kFrontWarpChars = 512;
__device__ __forceinline__ void decode_sentence_smem(const DictView& d, const Batch& b, const uint8_t* p,
                                                     unsigned long long len, uint32_t base, uint32_t n, uint32_t* buf,
                                                     uint32_t lane) {
    uint32_t running = 0;
    for (unsigned long long i0 = 0; n > 0 && i0 < len; i0 += 32) {
        const unsigned long long i = i0 + lane;
        const bool lead = i < len && (p[i] & 0xC0) != 0x80;
        const uint32_t m = __ballot_sync(kFull, lead);
        const uint32_t idx = running + __popc(m & lanemask_lt());
        if (lead && idx < n) buf[idx] = uint32_t(i);
        running += __popc(m);
    }
    __syncwarp();
    for (uint32_t idx = lane; idx < n; idx += 32) {
        const uint32_t i = buf[idx], slot = base + idx;
        const uint32_t c = p[i], c1 = i + 1 < len ? p[i + 1] : 0, c2 = i + 2 < len ? p[i + 2] : 0,
                       c3 = i + 3 < len ? p[i + 3] : 0;
        uint32_t cp;  // compute_basic sentence.rs:40-46
        if (c < 0x80)
            cp = c;
        else if (c < 0xE0)
            cp = ((c & 0x1F) << 6) | (c1 & 0x3F);
        else if (c < 0xF0)
            cp = ((c & 0x0F) << 12) | ((c1 & 0x3F) << 6) | (c2 & 0x3F);
        else
            cp = ((c & 0x07) << 18) | ((c1 & 0x3F) << 12) | ((c2 & 0x3F) << 6) | (c3 & 0x3F);
        b.byte_pos[slot] = i;
        // CharProperty::char_info character.rs:112-116: out-of-table code points use entry 0
        const uint32_t ci = __ldg(&d.chr2inf[cp < d.chr2inf_len ? cp : 0]);
        b.cinfo[slot] = ci;
        b.code_sys[slot] = cp < d.sys_table_len ? __ldg(&d.sys_table[cp]) : kInvalidCode;
        if (d.usr_table) b.code_usr[slot] = cp < d.usr_table_len ? __ldg(&d.usr_table[cp]) : kInvalidCode;
        b.ends_cnt[slot] = idx == 0 ? 1u : 0u;  // BOS lives in ends[0] (lattice.rs:72-83)
        buf[idx] = ci;
    }
    if (lane == 0) {  // sentinel slot == character position n
        const uint32_t slot = base + n;
        b.byte_pos[slot] = uint32_t(len);
        b.cinfo[slot] = 0;
        b.groupable[slot] = 0;
        b.code_sys[slot] = kInvalidCode;
        if (d.usr_table) b.code_usr[slot] = kInvalidCode;
        b.ends_cnt[slot] = 0;
        b.info[slot] = make_uint2(0, 0);
    }
    __syncwarp();
    uint32_t carry = 0;  // groupable as decode_one solves it
    for (int k = int((n + 31) / 32) - 1; k >= 0; --k) {
        const uint32_t c = uint32_t(k) * 32 + lane;
        const bool valid = c < n;
        const uint32_t ci = valid ? buf[c] : 0, cn = (c + 1 < n) ? buf[c + 1] : 0;
        const bool brk = valid && (c + 1 == n || (ci_cate(ci) & ci_cate(cn)) == 0);
        const uint32_t m = __ballot_sync(kFull, brk) >> lane;
        const uint32_t g = m ? uint32_t(__ffs(m)) : (min(32u, n - uint32_t(k) * 32) - lane) + carry;
        if (valid) b.groupable[base + c] = g;
        carry = __shfl_sync(kFull, g, 0);
    }
    __syncwarp();  // buf is the warp's next sentence's
}

// ---------------------------------------------------------------------------------------------
// Single-pass exclusive scans with decoupled look-back (k_front: slots per sentence, k_backtrack: tokens per sentence).
// A block takes its tile from a ticket counter, so every tile it waits for belongs to a block that is already running.
// Each tile has one word: its status in the top two bits (kTileAgg: the tile's own total is known, kTileIncl: the
// total of every tile up to and including it) and the value in the low 62 bits.
// ---------------------------------------------------------------------------------------------

constexpr unsigned long long kTileAgg = 1ull << 62, kTileIncl = 2ull << 62, kTileValue = kTileAgg - 1;

__device__ __forceinline__ uint32_t take_tile(uint32_t* ticket, uint32_t* s_tile) {
    if (threadIdx.x == 0) *s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    return *s_tile;
}

// Warp 0 of the block of `tile`, whose own total is `agg`: returns the total of the tiles before it (every lane) and
// publishes the inclusive total.  The fences order each tile's batch flags before its published values, so that a
// tile that has its prefix also sees the flags every tile before it raised.
__device__ unsigned long long tile_prefix(unsigned long long* state, uint32_t tile, unsigned long long agg, uint32_t lane) {
    if (lane == 0) {
        __threadfence();
        atomicExch(&state[tile], (tile == 0 ? kTileIncl : kTileAgg) | (agg & kTileValue));
    }
    unsigned long long excl = 0;
    for (long long j = (long long)tile - 1; j >= 0; j -= 32) {  // lane l looks at tile j - l
        const long long t = j - lane;
        unsigned long long w;
        do
            w = t >= 0 ? *reinterpret_cast<volatile unsigned long long*>(&state[t]) : (unsigned long long)kTileIncl;
        while (__any_sync(kFull, w < kTileAgg));
        const uint32_t incl = __ballot_sync(kFull, w >= kTileIncl);
        const uint32_t upto = incl ? uint32_t(__ffs(incl)) - 1 : 31u;  // the nearest inclusive total ends the walk
        excl += warp_sum(lane <= upto ? (w & kTileValue) : 0ull);
        if (incl) break;
    }
    __threadfence();
    if (lane == 0 && tile != 0) atomicExch(&state[tile], kTileIncl | ((excl + agg) & kTileValue));
    return excl;
}

// ---------------------------------------------------------------------------------------------
// K1: count_chars + slot-offset scan + Sentence::compile (sentence.rs:34-71), one pass over tiles of kFrontTile
// consecutive sentences (a warp per sentence).  The tile's text is staged in shared memory when it fits in
// kFrontStage bytes; otherwise, and for sentences outside the staged range (offsets out of order), it is read from
// global memory.  n_slots (the sort key of the K3 order) and slot_off are written for every sentence; a tile decodes
// only when no tile up to it has bad offsets, which could otherwise carry the slots past the arrays' n_bytes + n_sent.
// ---------------------------------------------------------------------------------------------

static_assert(kFrontTile == 32, "warp 0 scans the tile's counts");
constexpr uint32_t kFrontStage = 16384;

__global__ void __launch_bounds__(256) k_front(DictView d, Batch b, unsigned long long* tile_state, uint32_t* ticket) {
    __shared__ __align__(16) uint8_t s_text[kFrontStage + 32];
    __shared__ uint32_t s_buf[8][kFrontWarpChars];
    __shared__ uint32_t s_n[kFrontTile], s_off[kFrontTile];
    __shared__ uint32_t s_tile, s_stand;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t tile = take_tile(ticket, &s_tile);
    const uint32_t s0 = tile * kFrontTile, nt = min(kFrontTile, b.n_sent - s0);
    const unsigned long long lo = b.byte_off[s0], hi = b.byte_off[s0 + nt];
    const bool staged = lo <= hi && hi <= b.total_bytes && hi - lo <= kFrontStage;
    // s_text[head + x] = byte lo + x; 16-byte loads between the 16-byte boundaries, single bytes at either end
    const uint32_t head = uint32_t(reinterpret_cast<uintptr_t>(b.utf8 + lo) & 15u);
    if (staged) {
        const uint8_t* a0 = b.utf8 + lo - head;
        const uint32_t span = head + uint32_t(hi - lo);
        for (uint32_t c0 = threadIdx.x * 16; c0 < span; c0 += 256 * 16) {
            if (c0 >= head && c0 + 16 <= span) {
                *reinterpret_cast<uint4*>(s_text + c0) = __ldg(reinterpret_cast<const uint4*>(a0 + c0));
            } else {
                for (uint32_t q = max(c0, head); q < min(c0 + 16, span); ++q) s_text[q] = a0[q];
            }
        }
    }
    __syncthreads();
    auto text = [&](unsigned long long bo, unsigned long long eo) -> const uint8_t* {
        return staged && bo >= lo && eo <= hi ? s_text + head + (bo - lo) : b.utf8 + bo;
    };
    constexpr uint32_t kPerWarp = kFrontTile / 8;
#pragma unroll 1
    for (uint32_t r = 0; r < kPerWarp; ++r) {
        const uint32_t t = wid * kPerWarp + r;
        if (t >= nt) break;
        const uint32_t s = s0 + t;
        const unsigned long long bo = b.byte_off[s], eo = b.byte_off[s + 1];
        uint32_t ns = 1;
        if (eo < bo || eo > b.total_bytes) {  // caller error: nothing of this sentence is read
            if (lane == 0) {
                atomicOr(b.flags, kFlagBadOffsets);
                b.n_slots[s] = 1;
            }
        } else {
            ns = count_chars_at(b, text(bo, eo), eo - bo, &b.n_slots[s], lane);
        }
        if (lane == 0) s_n[t] = ns;
    }
    __syncthreads();
    if (wid == 0) {
        const uint32_t v = lane < nt ? s_n[lane] : 0u;
        uint32_t x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(kFull, x, o);
            if (lane >= uint32_t(o)) x += y;
        }
        const uint32_t agg = __shfl_sync(kFull, x, 31);
        // slot counts wrap like the u32 slot offsets; a batch where they could is rejected (kFlagBadOffsets)
        const uint32_t base = uint32_t(tile_prefix(tile_state, tile, agg, lane));
        if (lane < nt) {
            s_off[lane] = base + x - v;
            b.slot_off[s0 + lane] = base + x - v;
        }
        if (lane == 0) {
            // also the next tile's first offset (the same value), which decode_one reads for the tile's last sentence
            b.slot_off[s0 + nt] = base + agg;
            s_stand = stand_down(*reinterpret_cast<volatile uint32_t*>(b.flags));
        }
    }
    __syncthreads();
    if (s_stand) return;
#pragma unroll 1
    for (uint32_t r = 0; r < kPerWarp; ++r) {
        const uint32_t t = wid * kPerWarp + r;
        if (t >= nt) break;
        const unsigned long long bo = b.byte_off[s0 + t], eo = b.byte_off[s0 + t + 1];
        const uint32_t n = s_n[t] - 1;
        if (n <= kFrontWarpChars)
            decode_sentence_smem(d, b, text(bo, eo), eo - bo, s_off[t], n, s_buf[wid], lane);
        else
            decode_one(d, b, s0 + t, lane);
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------
// K2: lattice candidates per start position = Tokenizer::add_lattice_edges (tokenizer.rs:141-199)
// ---------------------------------------------------------------------------------------------

struct WalkStats {
    uint32_t m, t, p, w, walks;
};

// The candidate pool holds, per start position, its candidate SOURCES rather than the candidates: every candidate
// is one record of a postings list (trie hit) or of the unk.def entries of a character category (unknown-word span),
// and the candidates of one source are a contiguous run of it.  A segment (8 bytes) names such a run:
//   x = kind | index   kind: 0 system postings, kSegUser user postings (index = the key's header, the records follow
//                      it), kSegUnk unknown words (index = the first unk_ent entry)
//   y = delta << 16 | count   count: candidates in the run (< 2^16); delta (signed 16 bits): end slot of the run
//                      minus that of the segment before it, or minus the position's own slot for the first one.
// A source with 2^16 candidates or more becomes several segments; an end slot more than 32 767 away from the one
// before is reached through count-0 segments that only move it.  The segments of a position follow the candidate
// order of Tokenizer::add_lattice_edges (user, system, unknown; ascending length; CSV order inside a postings list),
// so candidate j of a position is found by walking its segments (cand_at).  The device image keeps both arrays
// below 2^30 entries, so that index + count never reaches the kind bits.
constexpr uint32_t kSegUser = 0x80000000u, kSegUnk = 0x40000000u, kSegIndex = 0x3FFFFFFFu;
constexpr int32_t kSegMaxDelta = 32767;

// Candidate j of segment s, whose run ends at slot `end`: {left | right << 16, cost word, word_idx, end slot}.
__device__ __forceinline__ uint4 seg_record(const DictView& d, uint2 s, uint32_t j, uint32_t end) {
    if (s.x & kSegUnk) {  // unknown.rs:133 `word_id as u16`, LexType::Unknown
        const uint32_t id = (s.x & kSegIndex) + j;
        const uint2 ue = __ldg(&d.unk_ent[id]);
        return make_uint4(ue.x, ue.y, (2u << 30) | (id & 0xFFFFu), end);
    }
    const uint4* __restrict__ post = (s.x & kSegUser) ? d.usr_post : d.sys_post;
    uint4 r = __ldg(&post[(s.x & kSegIndex) + 1 + j]);  // the candidate record, end slot still open
    r.w = end;
    return r;
}

// Candidate j (< the position's candidate count) of the start position at `slot`, whose segments are seg(0),
// seg(1), ...: a walk over the segments before it.
template <class SegAt>
__device__ __forceinline__ uint4 cand_at(const DictView& d, SegAt seg, uint32_t slot, uint32_t j) {
    uint32_t h = 0, end = slot;
    uint2 s = seg(0u);
    for (;;) {
        end += uint32_t(int32_t(s.y) >> 16);
        const uint32_t c = s.y & 0xFFFFu;
        if (j < c) break;
        j -= c;
        s = seg(++h);
    }
    return seg_record(d, s, j, end);
}

// Segment encoder of one start position.  The count pass of k_candidates keeps up to kMaxSegs segments in shared
// memory (column-major, [segment][thread], so the accesses of a warp are conflict-free) and counts the rest; a
// position with more is walked again after the allocation, straight into the pool, with ends_cnt set.
constexpr uint32_t kMaxSegs = 8;
struct SegOut {
    uint2* dst;          // segment h goes to dst[h * stride] while h < cap
    uint32_t stride, cap;
    uint32_t n;          // segments so far, also those past cap
    uint32_t last;       // end slot of the segment before; the position's slot at first
    uint32_t* ends_cnt;  // non-null: every candidate is also counted into its end row
    __device__ __forceinline__ void put(uint32_t x, uint32_t y) {
        if (n < cap) dst[n * stride] = make_uint2(x, y);
        ++n;
    }
    __device__ __forceinline__ void push(uint32_t v, uint32_t end, uint32_t count) {
        if (count == 0) return;
        if (ends_cnt) atomicAdd(&ends_cnt[end], count);
        int32_t delta = int32_t(end - last);
        while (delta > kSegMaxDelta || delta < -kSegMaxDelta) {
            const int32_t step = delta > 0 ? kSegMaxDelta : -kSegMaxDelta;
            put(v, uint32_t(step) << 16);
            delta -= step;
        }
        last = end;
        for (;;) {
            const uint32_t c = min(count, 0xFFFFu);
            put(v, (uint32_t(delta) << 16) | c);
            count -= c;
            if (count == 0) break;
            v += c;  // the next run starts c records further; for postings `index` stays one before the run
            delta = 0;
        }
    }
};

// Lexicon::common_prefix_iterator (lexicon.rs:33-46): crawdad common-prefix search over the double
// array (trie.rs:49-56); every hit is one segment, the postings list of its key (posting.rs:18-21).
// BND (bounded batches): the walk stops at q_end = lim(sw), the first required boundary after sw, so no word that
// crosses it is a candidate or counts as a match.
template <bool COUNT, bool BND = false>
__device__ __forceinline__ uint32_t walk_lexicon(const uint4* __restrict__ nodes, uint32_t num_nodes,
                                                 const uint32_t* __restrict__ codes,
                                                 const uint32_t* __restrict__ groupable, uint32_t sw, WalkStats& st,
                                                 SegOut* so = nullptr, uint32_t lex_flag = 0, uint32_t q_end = 0) {
    if (num_nodes == 0) return 0;
    uint32_t count = 0, node = 0, d = 0, hits = 0;
    uint32_t nbase = __ldg(&nodes[0].x);
    uint32_t q = sw;
    for (;; ++q) {
        if (BND && q >= q_end) break;
        uint32_t code = codes[q];
        if (code == kInvalidCode) break;  // unmapped character or the sentence's sentinel
        if (nbase & kFlag) break;         // a leaf has no children
        uint32_t child = nbase ^ code;
        if (child >= num_nodes) break;
        const uint4 nd = __ldg(&nodes[child]);  // one 16-byte load per step: base, check, and the key ending here
        if ((nd.y & kMask) != node) break;
        node = child;
        nbase = nd.x;
        ++d;
        if (nd.z == kNone) continue;
        const uint32_t v = nd.z;
        const uint32_t plen = nd.w;
        if (so) so->push(v | lex_flag, q + 1, plen);
        count += plen;
        ++hits;
        if (COUNT) {
            st.p += 1 + plen;
            st.w += plen;
        }
    }
    if (COUNT) {
        uint32_t f = groupable[q] != 0 ? 1u : 0u;  // 0 when the walk ran off the end of the sentence
        st.m += d + f;
        st.t += d + f + hits;
        st.walks += 1;
    }
    return count;
}

// UnkHandler::gen_unk_words (unknown.rs:69-116) with scan_entries (:119-137): every span is one segment.
__device__ __forceinline__ uint32_t gen_unknown(const DictView& d, uint32_t sw, uint32_t ci, uint32_t g,
                                                bool has_matched, SegOut* so = nullptr) {
    if (has_matched && !ci_invoke(ci)) return 0;
    const uint32_t e0 = __ldg(&d.unk_off[ci_base(ci)]), e1 = __ldg(&d.unk_off[ci_base(ci) + 1]);
    const uint32_t ne = e1 - e0;
    uint32_t count = 0;
    auto span = [&](uint32_t end) {
        if (so) so->push(kSegUnk | e0, end, ne);
        count += ne;
    };
    bool grouped = false;
    if (ci_group(ci)) {
        grouped = true;
        if ((unsigned long long)(g - 1) <= d.max_grouping) {  // :91-93
            span(sw + g);
            has_matched = true;
        }
    }
    uint32_t lim = min(ci_length(ci), g);
    for (uint32_t i = 1; i <= lim; ++i) {
        if (grouped && i == g) continue;
        span(sw + i);  // sw + i <= sentence length because i <= groupable
        has_matched = true;
    }
    if (!has_matched) span(sw + 1);  // :112-115
    return count;
}

// Where the word of start position `slot` begins (tokenizer.rs:117-130); g0 = groupable[slot], 0 for the sentinel.
// At a space (ignore_space) the groupable run is skipped; a skip that reaches the end of the sentence leaves the
// trailing flag and no candidates.
struct StartWord {
    uint32_t sw, skip, flags, ci, g;
    bool active;
    uint32_t lim;  // BND only: lim(sw) - sw
};
//
// BND: w.lim = lim(sw) - sw (bnd_dist), and g is clipped to it wherever gen_unknown uses it, so that a boundary ends a
// character group.  The space skip is not affected.
template <bool BND = false>
__device__ __forceinline__ StartWord start_word(const DictView& d, const Batch& b, uint32_t slot, uint32_t g0) {
    StartWord w{slot, 0, 0, 0, 0, g0 != 0, 0};
    if (w.active) {
        uint32_t ci0 = b.cinfo[slot];
        if (ci_cate(ci0) & d.space_mask) {  // tokenizer.rs:117-125: skip the groupable run at a space
            w.skip = g0;
            w.sw = slot + w.skip;
        }
        w.g = w.skip ? b.groupable[w.sw] : g0;
        if (w.g == 0) {  // start_word == len: tokenizer.rs:128-130
            w.flags = kInfoTrailing;
            w.active = false;
        } else {
            w.ci = w.skip ? b.cinfo[w.sw] : ci0;
            if (BND) {
                w.lim = b.bnd_dist[w.sw];
                w.g = min(w.g, w.lim);
            }
        }
    }
    return w;
}

// Candidate count of an active start position: user lexicon, system lexicon, then unknown words, the order of
// Tokenizer::add_lattice_edges.  Its segments go to `so` (so.last = the position's slot).
template <bool BND = false>
__device__ __forceinline__ uint32_t count_candidates(const DictView& d, const Batch& b, const StartWord& w, SegOut& so) {
    WalkStats st{0, 0, 0, 0, 0};
    uint32_t cu = 0;
    if (d.usr_table)
        cu = walk_lexicon<false, BND>(d.usr_nodes, d.usr_num_nodes, b.code_usr, b.groupable, w.sw, st, &so, kSegUser,
                                      w.sw + w.lim);
    uint32_t cs = walk_lexicon<false, BND>(d.sys_nodes, d.sys_num_nodes, b.code_sys, b.groupable, w.sw, st, &so, 0,
                                           w.sw + w.lim);
    return cu + cs + gen_unknown(d, w.sw, w.ci, w.g, (cu + cs) != 0, &so);  // (cu + cs) != 0: a lexicon word starts here
}

// Candidate header of a start position with g0 != 0: {segment ptr, candidate count}, plus the skip / flags side entry.
__device__ __forceinline__ void store_info(const Batch& b, uint32_t slot, uint32_t ptr, uint32_t cnt, const StartWord& w) {
    const bool special = (w.skip | w.flags) != 0;
    b.info[slot] = make_uint2(ptr, cnt | (special ? kInfoSpecial : 0u));
    if (special) b.info_ex[slot] = make_uint2(w.skip, w.flags);
}

template <class Out>
__device__ __forceinline__ uint32_t csv_fields(const uint8_t* __restrict__ p, uint32_t n, Out out);

// Required tokens: does the feature of word `id` of lexicon `lex` (0 system, 1 user, 2 unknown entries) match
// pattern p?  Each constrained field (SpanArgs::pf, ascending field index) must equal its bytes; a field past the
// feature's last one does not match (it reads as '*', which no constrained field is).
__device__ __forceinline__ bool span_match(const DictView& d, const SpanArgs& sp, uint32_t lex, uint32_t id, uint32_t p) {
    if (p == kSpanAny) return true;
    const uint32_t k1 = sp.pat_off[p + 1];
    uint32_t k = sp.pat_off[p], pos = 0;
    if (k == k1) return true;
    const uint32_t a = d.feat_off[lex][id];
    uint3 c = sp.pf[k];
    bool ok = true;
    const uint32_t nf = csv_fields(d.feat[lex] + a, d.feat_off[lex][id + 1] - a, [&](uint32_t field, uint8_t ch) {
        while (k < k1 && c.x < field) {  // the constrained field before this one is complete
            ok &= pos == c.z;
            if (++k < k1) c = sp.pf[k];
            pos = 0;
        }
        if (k < k1 && c.x == field) {
            ok &= pos < c.z && sp.pat_bytes[c.y + pos] == ch;
            ++pos;
        }
    });
    for (; k < k1; pos = 0) {
        ok &= c.x < nf && pos == c.z;
        if (++k < k1) c = sp.pf[k];
    }
    return ok;
}

// The postings of the one key of a lexicon that spans [sw, end) exactly, filtered by pattern p: every maximal run of
// matching records is one segment (its index one before the run's first record, as SegOut::push continues a list).
__device__ __forceinline__ uint32_t span_postings(const DictView& d, const SpanArgs& sp, const uint4* __restrict__ nodes,
                                                  uint32_t num_nodes, const uint4* __restrict__ post,
                                                  const uint32_t* __restrict__ codes, uint32_t sw, uint32_t end,
                                                  uint32_t p, uint32_t lex_flag, SegOut& so) {
    if (num_nodes == 0) return 0;
    uint32_t node = 0, nbase = __ldg(&nodes[0].x), hit = kNone, plen = 0;
    for (uint32_t q = sw; q < end; ++q) {  // walk_lexicon, to `end` only
        const uint32_t code = codes[q];
        if (code == kInvalidCode || (nbase & kFlag)) return 0;
        const uint32_t child = nbase ^ code;
        if (child >= num_nodes) return 0;
        const uint4 nd = __ldg(&nodes[child]);
        if ((nd.y & kMask) != node) return 0;
        node = child;
        nbase = nd.x;
        hit = nd.z;
        plen = nd.w;
    }
    if (hit == kNone) return 0;
    uint32_t count = 0;
    for (uint32_t j = 0; j < plen;) {
        uint32_t j1 = j;
        while (j1 < plen) {
            const uint32_t widx = __ldg(&post[hit + 1 + j1]).z;
            if (!span_match(d, sp, widx >> 30, widx & 0x3FFFFFFFu, p)) break;
            ++j1;
        }
        so.push((hit + j) | lex_flag, end, j1 - j);
        count += j1 - j;
        j = j1 + 1;
    }
    return count;
}

// Candidates of a start position whose word starts a span (tag = {length in characters, pattern}): the user, then
// the system lexicon's words of exactly the span's surface that match the pattern; without any, one unknown word
// over the whole span per unk.def entry of the start character's category that matches (all of them when none does).
__device__ __forceinline__ uint32_t count_span(const DictView& d, const Batch& b, const SpanArgs& sp, const StartWord& w,
                                               uint2 tag, SegOut& so) {
    const uint32_t end = w.sw + tag.x;
    uint32_t cnt = 0;
    if (d.usr_table) cnt = span_postings(d, sp, d.usr_nodes, d.usr_num_nodes, d.usr_post, b.code_usr, w.sw, end, tag.y, kSegUser, so);
    cnt += span_postings(d, sp, d.sys_nodes, d.sys_num_nodes, d.sys_post, b.code_sys, w.sw, end, tag.y, 0, so);
    if (cnt) return cnt;
    const uint32_t e0 = __ldg(&d.unk_off[ci_base(w.ci)]), e1 = __ldg(&d.unk_off[ci_base(w.ci) + 1]);
    bool all = true;
    for (uint32_t e = e0; all && e < e1; ++e) all = !span_match(d, sp, 2, e, tag.y);
    for (uint32_t e = e0; e < e1;) {
        uint32_t e2 = e;
        while (e2 < e1 && (all || span_match(d, sp, 2, e2, tag.y))) ++e2;
        so.push(kSegUnk | e, end, e2 - e);
        cnt += e2 - e;
        e = e2 + 1;
    }
    return cnt;
}

// start_word of a span batch: a position strictly inside a span gets no candidates (no node ends there, so the
// reference's loop skips it); *tag receives the span tag of the word's start.  A space skip that lands strictly inside
// a span (the skipped run continues into it through a category the space shares) would start a word there: the batch
// is refused (kFlagBadSpan).
__device__ __forceinline__ StartWord start_word_spans(const DictView& d, const Batch& b, const SpanArgs& sp, uint32_t slot,
                                                      uint32_t g0, uint2* tag) {
    *tag = make_uint2(0, 0);
    const StartWord none{slot, 0, 0, 0, 0, false, 0};
    if (g0 != 0 && sp.tag[slot].x == kSpanInside) return none;
    const StartWord w = start_word<true>(d, b, slot, g0);
    if (w.active) *tag = sp.tag[w.sw];
    if (tag->x == kSpanInside) {
        atomicOr(b.flags, kFlagBadSpan);
        *tag = make_uint2(0, 0);
        return none;
    }
    return w;
}

// BND: the bounded instantiation (required boundaries in b.bnd_dist); the unbounded one is the code as it was.
// SPAN (k_candidates_spans, BND too): the span rules of count_span / start_word_spans on top.
template <bool BND, bool SPAN>
__device__ __forceinline__ void candidates_body(const DictView& d, const Batch& b, const SpanArgs& sp) {
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    // A rejected batch (see stand_down) leaves every thread out of range.  The flag word is read next to the slot
    // total instead of in front of it: with 256-thread blocks that live for one trie walk, a dependent extra round
    // trip at the top costs 8 % of this kernel (profiles/r01e_k3_variants_ab.md).
    const uint32_t batch_flags = *b.flags;
    const uint32_t total_slots = b.slot_off[b.n_sent];
    if (slot == 0 && total_slots > b.launch_slots) atomicOr(b.flags, kFlagSlotsOverflow);
    const bool in_range = slot < total_slots && !(batch_flags & kFlagBadOffsets);
    uint32_t g0 = in_range ? b.groupable[slot] : 0;
    uint2 tag = make_uint2(0, 0);
    const StartWord sw = SPAN ? start_word_spans(d, b, sp, slot, g0, &tag) : start_word<BND>(d, b, slot, g0);
    const bool active = sw.active;
    uint32_t cnt = 0;
    __shared__ uint2 s_segs[kMaxSegs][256];
    SegOut so{&s_segs[0][threadIdx.x], 256, kMaxSegs, 0, slot, nullptr};
    if (active) cnt = (SPAN && tag.x) ? count_span(d, b, sp, sw, tag, so) : count_candidates<BND>(d, b, sw, so);
    const uint32_t nseg = so.n;
    // Block-aggregated allocation from the segment pool: a scan inside each warp, the eight warp totals through
    // shared memory, ONE atomicAdd per block.  (One atomic per warp was 1.3 M same-address atomics per batch, and
    // every warp sat on the round trip of its own; the pool also comes out in slot order block by block.)  The
    // candidates are counted alongside: they are the lattice nodes, and the rows must hold them.
    uint32_t incl = cnt, sincl = nseg;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(kFull, incl, o), sv = __shfl_up_sync(kFull, sincl, o);
        if (lane >= uint32_t(o)) {
            incl += v;
            sincl += sv;
        }
    }
    __shared__ uint32_t s_warp_total[8], s_warp_segs[8];
    __shared__ unsigned long long s_block_base, s_block_cand;
    const uint32_t wid = threadIdx.x >> 5;
    if (lane == 31) {
        s_warp_total[wid] = incl;
        s_warp_segs[wid] = sincl;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t run = 0, srun = 0;
        for (int i = 0; i < 8; ++i) {  // warp totals -> exclusive offsets inside the block
            const uint32_t t = s_warp_total[i], st = s_warp_segs[i];
            s_warp_total[i] = run;
            s_warp_segs[i] = srun;
            run += t;
            srun += st;
        }
        s_block_base = srun ? atomicAdd(b.seg_ctr, (unsigned long long)srun) : 0ull;
        s_block_cand = run ? atomicAdd(b.pool_ctr, (unsigned long long)run) : 0ull;
        if (s_block_base + srun > (unsigned long long)b.seg_cap || s_block_cand + run > (unsigned long long)b.cand_cap)
            atomicOr(b.flags, kFlagPoolOverflow);
    }
    __syncthreads();
    const unsigned long long wbase = s_block_base + s_warp_segs[wid], cbase = s_block_cand + s_warp_total[wid];
    const bool fits = wbase + __shfl_sync(kFull, sincl, 31) <= (unsigned long long)b.seg_cap &&
                      cbase + __shfl_sync(kFull, incl, 31) <= (unsigned long long)b.cand_cap;
    const uint32_t ptr = uint32_t(wbase) + (sincl - nseg);
    if (in_range && g0 != 0) store_info(b, slot, ptr, fits ? cnt : 0, sw);
    // Fill: the position's segments go to the pool as they are, and its candidates into their end rows.
    if (!(active && fits && cnt)) return;
    if (nseg <= kMaxSegs) {
        uint32_t end = slot;
        for (uint32_t h = 0; h < nseg; ++h) {
            const uint2 s = s_segs[h][threadIdx.x];
            end += uint32_t(int32_t(s.y) >> 16);
            if (s.y & 0xFFFFu) atomicAdd(&b.ends_cnt[end], s.y & 0xFFFFu);
            b.seg[ptr + h] = s;
        }
    } else {  // more segments than the buffer holds: walk again, straight into the pool
        SegOut out{b.seg + ptr, 1, nseg, 0, slot, b.ends_cnt};
        if (SPAN && tag.x)
            count_span(d, b, sp, sw, tag, out);
        else
            count_candidates<BND>(d, b, sw, out);
    }
}

template <bool BND>
__global__ void __launch_bounds__(256) k_candidates(DictView d, Batch b) {
    candidates_body<BND, false>(d, b, SpanArgs{});
}

__global__ void __launch_bounds__(256) k_candidates_spans(DictView d, Batch b, SpanArgs sp) {
    candidates_body<true, true>(d, b, sp);
}

// Required boundaries of sentence s -> bnd_dist, in two passes of the warp.  (1) One lane per boundary: a boundary b
// (sentence-relative byte offset) with 0 < b < len marks the character that starts at byte b (binary search of
// byte_pos over the sentence's slots; the slots are cleared first).  (2) Right to left over 32-character chunks, as
// decode_one solves groupable: bnd_dist[c] = the first marked position after c (or n) - c.  Runs after decode_one of
// the same sentence.
// Validates the list on the way: offsets in order and inside bnd, values non-decreasing, <= len and on a UTF-8 lead
// byte; anything else raises kFlagBadBoundary.  A boundary at 0 or len marks nothing: every token already ends there.
// `extra(mark, base, n, bo, len)` runs between the two passes, once the boundaries are marked (mark_spans_one).
struct NoMarks {
    __device__ void operator()(uint32_t*, uint32_t, uint32_t, unsigned long long, unsigned long long) const {}
};
template <class Extra = NoMarks>
__device__ __forceinline__ void mark_bounds_one(const Batch& b, uint32_t s, uint32_t lane, Extra extra = {}) {
    const unsigned long long j0 = b.bnd_off[s], j1 = b.bnd_off[s + 1];
    const bool listed = !(j1 < j0 || j1 > b.n_bnd);
    const unsigned long long bo = b.byte_off[s], len = b.byte_off[s + 1] - bo;
    const uint32_t base = b.slot_off[s], n = b.slot_off[s + 1] - base - 1;
    uint32_t* mark = b.bnd_dist + base;
    for (uint32_t i = lane; i <= n; i += 32) mark[i] = 0;
    __syncwarp();
    bool bad = !listed;
    for (unsigned long long j = j0 + lane; listed && j < j1; j += 32) {
        const uint32_t v = b.bnd[j];
        if (v > len || (j > j0 && b.bnd[j - 1] > v) || (v < len && (b.utf8[bo + v] & 0xC0) == 0x80)) {
            bad = true;
            continue;
        }
        if (v == 0 || v == len) continue;
        uint32_t lo = 0, hi = n;  // byte_pos[base + n] == len > v
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (b.byte_pos[base + mid] < v)
                lo = mid + 1;
            else
                hi = mid;
        }
        mark[lo] = 1;
    }
    if (__any_sync(kFull, bad) && lane == 0) atomicOr(b.flags, kFlagBadBoundary);
    extra(mark, base, n, bo, len);
    __syncwarp();
    uint32_t next = n;  // the first marked position right of the chunks done so far
    for (int k = int((n + 31) / 32) - 1; k >= 0; --k) {
        const uint32_t c = uint32_t(k) * 32 + lane;
        const uint32_t m = __ballot_sync(kFull, c < n && mark[c] != 0);
        const uint32_t above = lane == 31 ? 0u : m >> (lane + 1);
        if (c < n) mark[c] = (above ? c + uint32_t(__ffs(above)) : next) - c;
        if (m) next = uint32_t(k) * 32 + uint32_t(__ffs(m)) - 1;
    }
    if (lane == 0) mark[n] = 0;
}

__global__ void __launch_bounds__(256) k_mark_bounds(Batch b) {
    if (stand_down(*b.flags)) return;
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
#pragma unroll 1
    for (uint32_t r = 0; r < VBT_SENT_PER_WARP; ++r) {
        const uint32_t s = w * VBT_SENT_PER_WARP + r;
        if (s >= b.n_sent) return;
        mark_bounds_one(b, s, lane);
    }
}

// Required tokens of sentence s, between the passes of mark_bounds_one: one lane per span marks its start and end
// as boundaries and tags its start; then the warp tags the interiors in one left-to-right pass over 32-character
// chunks (a prefix max of the span ends started so far), so a long span costs no lane more than its share.  Validates the list (offsets in order and inside sp.rec; start < end <= len,
// both on UTF-8 lead bytes or at len; no overlap with the span before; a known pattern; no explicit boundary strictly
// inside; with ignore_space no start at a SPACE character) and raises kFlagBadSpan otherwise.  An invalid span marks
// nothing.
__device__ __forceinline__ void mark_spans_one(const Batch& b, const SpanArgs& sp, uint32_t s, uint32_t lane) {
    mark_bounds_one(b, s, lane, [&](uint32_t* mark, uint32_t base, uint32_t n, unsigned long long bo, unsigned long long len) {
        uint2* tag = sp.tag + base;
        for (uint32_t i = lane; i <= n; i += 32) tag[i] = make_uint2(0, 0);
        __syncwarp();
        const unsigned long long j0 = sp.off[s], j1 = sp.off[s + 1];
        const bool listed = !(j1 < j0 || j1 > sp.n);
        bool bad = !listed;
        auto slot_of = [&](uint32_t v) {  // the character that starts at byte v (n for v == len)
            uint32_t lo = 0, hi = n;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (b.byte_pos[base + mid] < v)
                    lo = mid + 1;
                else
                    hi = mid;
            }
            return lo;
        };
        for (unsigned long long j = j0 + lane; listed && j < j1; j += 32) {
            const uint3 r = sp.rec[j];
            if (r.x >= r.y || r.y > len || (b.utf8[bo + r.x] & 0xC0) == 0x80 ||
                (r.y < len && (b.utf8[bo + r.y] & 0xC0) == 0x80) || (j > j0 && sp.rec[j - 1].y > r.x) ||
                (r.z != kSpanAny && r.z >= sp.n_pat)) {
                bad = true;
                continue;
            }
            const uint32_t ca = slot_of(r.x), cb = slot_of(r.y);
            if (ci_cate(b.cinfo[base + ca]) & sp.space_mask) {  // the space skip would move the word's start past it
                bad = true;
                continue;
            }
            tag[ca] = make_uint2(cb - ca, r.z);
            if (ca > 0) mark[ca] = 1;
            if (cb < n) mark[cb] = 1;
        }
        __syncwarp();
        // Interiors: c is inside a span when a span started before c ends after it.  The spans of a valid list are
        // disjoint, so a mark found there is an explicit boundary, not another span's end.
        uint32_t open_end = 0;  // the largest span end started in the chunks done so far
        for (uint32_t c0 = 0; c0 < n; c0 += 32) {
            const uint32_t c = c0 + lane;
            const uint32_t len_c = c < n ? tag[c].x : 0u;
            uint32_t e = len_c ? c + len_c : 0u;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(kFull, e, o);
                if (lane >= uint32_t(o)) e = max(e, v);
            }
            const uint32_t before = __shfl_up_sync(kFull, e, 1);
            const uint32_t reach = max(open_end, lane ? before : 0u);
            if (c < n && !len_c && reach > c) {
                if (mark[c]) bad = true;  // an explicit boundary inside the span
                tag[c] = make_uint2(kSpanInside, 0);
            }
            open_end = max(open_end, __shfl_sync(kFull, e, 31));
        }
        if (__any_sync(kFull, bad) && lane == 0) atomicOr(b.flags, kFlagBadSpan);
    });
}

__global__ void __launch_bounds__(256) k_mark_spans(Batch b, SpanArgs sp) {
    if (stand_down(*b.flags)) return;
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
#pragma unroll 1
    for (uint32_t r = 0; r < VBT_SENT_PER_WARP; ++r) {
        const uint32_t s = w * VBT_SENT_PER_WARP + r;
        if (s >= b.n_sent) return;
        mark_spans_one(b, sp, s, lane);
    }
}

// Side array for counted runs: per slot {M, T, P, W} so that k_viterbi can sum them over the
// positions the reference actually visits.  Filled by a second, counting-only kernel.
__global__ void __launch_bounds__(256) k_candidate_stats(DictView d, Batch b, uint4* stats) {
    if (stand_down(*b.flags)) return;
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= b.slot_off[b.n_sent]) return;
    uint32_t g0 = b.groupable[slot];
    uint4 out = make_uint4(0, 0, 0, 0);
    if (g0 != 0) {
        uint32_t sw = slot, ci0 = b.cinfo[slot];
        if (ci_cate(ci0) & d.space_mask) sw = slot + g0;
        uint32_t g = b.groupable[sw];
        if (g != 0) {
            WalkStats st{0, 0, 0, 0, 0};
            uint32_t cu = 0;
            if (d.usr_table)
                cu = walk_lexicon<true>(d.usr_nodes, d.usr_num_nodes, b.code_usr, b.groupable, sw, st);
            uint32_t cs = walk_lexicon<true>(d.sys_nodes, d.sys_num_nodes, b.code_sys, b.groupable, sw, st);
            uint32_t ck = gen_unknown(d, sw, b.cinfo[sw], g, (cu + cs) != 0);
            out = make_uint4(st.m, st.t, st.p, st.w + ck);
            out.x |= st.walks << 24;  // <= 2 walks; M stays far below 2^24 per position
        }
    }
    stats[slot] = out;
}

// ---------------------------------------------------------------------------------------------
// K3: Tokenizer::build_lattice_inner (tokenizer.rs:94-139) + Lattice::insert_node / search_min_node /
//     insert_eos (lattice.rs:85-151).
//
// G lanes per sentence (32 / G sentences per warp, walking their positions in lockstep): lane j of a
// group owns candidate j of the current start position, the group's predecessors {cost, right} are
// staged in registers and broadcast with width-G shuffles.  The typical position has ~7 candidates
// and ~8 predecessors, so G = 8 keeps most lanes busy where one warp per sentence left 3/4 idle.
// ---------------------------------------------------------------------------------------------

// Candidate header of one start position as {seg_ptr, cand_cnt, skip, flags}; the last two live in a side array
// that only the few positions with a skipped space run or the trailing flag ever touch.
__device__ __forceinline__ uint4 load_info(const Batch& b, uint32_t slot) {
    const uint2 i8 = b.info[slot];
    uint4 r = make_uint4(i8.x, i8.y & ~kInfoSpecial, 0, 0);
    if (i8.y & kInfoSpecial) {
        const uint2 ex = b.info_ex[slot];
        r.z = ex.x;
        r.w = ex.y;
    }
    return r;
}

// The lattice bookkeeping shared by k_viterbi and k_viterbi2.  Every lane of the warp calls these helpers; `sidx` is
// the group's sentence in launch order and the group's lane 0 (gl == 0) writes the per-sentence records.

// Start of the sweep of sentence `sidx`: returns its slots {first, sentinel} (both 0 without a sentence).  An empty
// sentence gets its EOS record here; any other gets its BOS node.
__device__ __forceinline__ uint2 begin_sentence(const Batch& b, uint32_t sidx, uint32_t gl) {
    uint32_t slot = 0, slot_end = 0;
    if (sidx < b.n_sent) {
        const uint32_t s = b.order ? b.order[sidx] : sidx;
        slot = b.slot_off[s];
        slot_end = b.slot_off[s + 1] - 1;
        if (gl == 0) {
            if (slot == slot_end) {  // Worker::tokenize returns early on an empty sentence (worker.rs:50-52)
                b.eos[s] = make_uint4(kNone, 0, 0, 0);
            } else {  // Lattice::insert_bos (lattice.rs:72-83): right_id 0, cost 0
                const uint32_t eo = b.ends_meta[slot].x;
                b.ends_hot[eo] = make_int2(0, 0);
                b.ends_cold[eo] = make_uint4(kNone, kNone, kNone, 0);
                b.ends_meta[slot].y = eo + 1;
            }
        }
    }
    __syncwarp();
    return make_uint2(slot, slot_end);
}

// Lattice::insert_node (lattice.rs:103-127): every valid lane pushes its candidate `cd` {left | right << 16, word
// cost in the low half, word idx, end slot} into ends[end_word], whose next free entry is `fill`, in candidate order.
// Its best total is `best`, reached from start slot `slot` through predecessor `bestk` of the row at entry `eo`.
// End slots of different sentences never coincide, so one warp-wide match suffices.  Returns the row's new fill on
// the lane that stored it (rank 0 among the lanes ending there), 0 on every other lane.
// k_marg_forward depends on this numbering: it assigns every candidate the same lattice entry again (BOS first, then
// positions in order, candidates in candidate order) and follows the sweep's position rules (a non-empty row, the
// space skip, the trailing break).  A change to either in k_viterbi / k_viterbi2 must be made there too; the
// marginal tests against tests/marginal_oracle.py catch a mismatch.
__device__ __forceinline__ uint32_t insert_node(const Batch& b, bool valid, const uint4& cd, int32_t best, uint32_t slot,
                                                uint32_t eo, uint32_t bestk, uint32_t fill) {
    const uint32_t vmask = __ballot_sync(kFull, valid);
    uint32_t new_fill = 0;
    if (valid) {
        const uint32_t peers = __match_any_sync(vmask, cd.w);
        const uint32_t rank = __popc(peers & lanemask_lt());
        const uint32_t idx = fill + rank;
        const int32_t cost = int32_t(uint32_t(best) + uint32_t(int32_t(int16_t(cd.y & 0xFFFFu))));
        b.ends_hot[idx] = make_int2(cost, int32_t(cd.x >> 16));
        // lattice.rs:144 keeps the predecessor index as u16
        b.ends_cold[idx] = make_uint4(slot, eo + (bestk & 0xFFFFu), cd.z, uint32_t(cost));
        if (rank == 0) {
            new_fill = fill + __popc(peers);
            b.ends_meta[cd.w].y = new_fill;
        }
    }
    __syncwarp();
    return new_fill;
}

// What k_viterbi's counters need of a finished sentence: the size of its EOS row, its base slot and its length.
struct SentenceEnd {
    uint32_t K, base, n;
};

// Lattice::insert_eos (lattice.rs:85-101): left_id 0, no word cost; the G lanes of the group take the predecessors
// in the row of `slot_end` and lane 0 writes b.eos.  Conn is the kernel's connector (ConnRow or ConnCol).
template <int G, class Conn>
__device__ __forceinline__ SentenceEnd insert_eos(const DictView& d, const Batch& b, uint32_t sidx, uint32_t slot_end,
                                                  uint32_t gl) {
    const bool has_sentence = sidx < b.n_sent;
    const uint32_t s = has_sentence ? (b.order ? b.order[sidx] : sidx) : 0;
    const uint32_t base = has_sentence ? b.slot_off[s] : 0;
    const uint32_t n = has_sentence ? b.slot_off[s + 1] - 1 - base : 0;
    const uint32_t eos_start = slot_end - base;  // n, or the start of the trailing space run
    uint32_t K = 0, eo = 0;
    if (n > 0) {
        const uint2 m = b.ends_meta[slot_end];
        eo = m.x;
        K = m.y - m.x;
    }
    // minimise the signed 64-bit key (cost << 32 | ~index): smallest cost, then the LARGEST index
    // among ties — the `<=` rule of search_min_node
    long long bestkey = LLONG_MAX;
    const Conn conn_eos(d, 0);  // BOS_EOS_CONNECTION_ID (common.rs:18)
    const uint32_t max_k = __reduce_max_sync(kFull, K);
    for (uint32_t k0 = 0; k0 < max_k; k0 += G) {
        long long key = LLONG_MAX;
        if (k0 + gl < K) {
            int2 pr = b.ends_hot[eo + k0 + gl];
            int32_t v = int32_t(uint32_t(pr.x) + uint32_t(conn_eos.cost(d, uint32_t(pr.y))));
            key = (long long)(((unsigned long long)uint32_t(v) << 32) | (unsigned long long)(~(k0 + gl)));
        }
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) key = min(key, __shfl_xor_sync(kFull, key, o, G));
        bestkey = min(bestkey, key);
    }
    if (n > 0 && gl == 0) {
        const bool none = K == 0;
        const uint32_t bestk = (~uint32_t(bestkey)) & 0xFFFFu;  // lattice.rs:144 `i as u16`
        b.eos[s] = make_uint4(none ? kNone : eo + bestk, eos_start, uint32_t(int32_t(bestkey >> 32)), 0);
    }
    return {K, base, n};
}

// ConnectorCost::cost(right_id, left_id) for one fixed left id (one candidate).
template <int CONN>
struct ConnRow;

template <>
struct ConnRow<0> {  // MatrixConnector::cost (matrix_connector.rs:79-85,121-124): one 2-byte gather
    // The image stores the matrix transposed, mt[right][left]: the lanes of a group share the predecessor's
    // right id and differ in their candidates' left ids, so with usage-sorted ids the frequent candidates of
    // one request fall into the same 128-byte line of row `right` instead of one line per candidate row.
    uint32_t off;  // the image builder refuses matrices of 2^32 entries or more, so 32-bit indices suffice
    __device__ __forceinline__ ConnRow(const DictView& d, uint32_t left) : off(left * d.conn_stride_left) {}
    __device__ __forceinline__ int32_t cost(const DictView& d, uint32_t right) const {
        return int32_t(__ldg(d.matrix + (off + right * d.conn_stride_right)));
    }
};

template <>
struct ConnRow<1> {  // RawConnector::cost (raw_connector.rs:155-160) = Scorer::accumulate_cost (scorer.rs:240-267)
    const uint32_t* __restrict__ lf;
    __device__ __forceinline__ ConnRow(const DictView& d, uint32_t left) : lf(d.left_feats + size_t(left) * d.feat_T) {}
    __device__ __forceinline__ int32_t cost(const DictView& d, uint32_t right) const {
        const uint32_t* __restrict__ rf = d.right_feats + size_t(right) * d.feat_T;
        uint32_t score = 0;
        for (uint32_t t = 0; t < d.feat_T; ++t) {
            const uint32_t key1 = __ldg(rf + t), key2 = __ldg(lf + t);
            if (key1 < d.n_bases) {  // INVALID_FEATURE_ID (0x7fffffff) never passes
                const uint32_t pos = __ldg(d.sc_bases + key1) ^ key2;
                if (pos < d.n_checks && __ldg(d.sc_checks + pos) == key1) score += uint32_t(__ldg(d.sc_costs + pos));
            }
        }
        return int32_t(score);
    }
};

template <>
struct ConnRow<2> {  // DualConnector::cost (dual_connector.rs:269-280): reduced-matrix gather + one 8-lane scorer row
    const int16_t* __restrict__ row;
    uint4 l0, l1;  // the candidate's eight raw feature ids stay in registers across its predecessors
    __device__ __forceinline__ ConnRow(const DictView& d, uint32_t left)
        : row(d.matrix + size_t(__ldg(d.left_conn + left)) * d.num_right) {
        const uint4* __restrict__ lf = reinterpret_cast<const uint4*>(d.left_feats + size_t(left) * 8);
        l0 = __ldg(lf);
        l1 = __ldg(lf + 1);
    }
    __device__ __forceinline__ uint32_t lane(const DictView& d, uint32_t key1, uint32_t key2) const {
        if (key1 < d.n_bases) {
            const uint32_t pos = __ldg(d.sc_bases + key1) ^ key2;
            if (pos < d.n_checks && __ldg(d.sc_checks + pos) == key1) return uint32_t(__ldg(d.sc_costs + pos));
        }
        return 0;
    }
    __device__ __forceinline__ int32_t cost(const DictView& d, uint32_t right) const {
        const uint4* __restrict__ rf = reinterpret_cast<const uint4*>(d.right_feats + size_t(right) * 8);
        const uint4 r0 = __ldg(rf), r1 = __ldg(rf + 1);
        uint32_t score = uint32_t(int32_t(__ldg(row + __ldg(d.right_conn + right))));
        score += lane(d, r0.x, l0.x) + lane(d, r0.y, l0.y) + lane(d, r0.z, l0.z) + lane(d, r0.w, l0.w);
        score += lane(d, r1.x, l1.x) + lane(d, r1.y, l1.y) + lane(d, r1.z, l1.z) + lane(d, r1.w, l1.w);
        return int32_t(score);
    }
};

// The sweep of k_viterbi over sentence `sidx` of each G-lane group of the calling warp (every lane calls it).
template <int G, bool COUNT, int CONN>
__device__ __forceinline__ void viterbi_sweep(const DictView& d, const Batch& b, const uint4* __restrict__ stats, uint32_t sidx) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t sub = lane / G, gl = lane % G;
    unsigned long long cntE = 0, cntN = 2, cM = 0, cT = 0, cP = 0, cW = 0, cWalks = 0;

    // Loop state is kept slot-absolute (current slot, the slot whose row EOS connects to, first slot after a
    // skipped space run) so that nothing but these three words lives across the gather loop; the sentence
    // index, its base slot and its length are looked up again where the sweep ends.
    const uint2 range = begin_sentence(b, sidx, gl);
    uint32_t slot = range.x, slot_end = range.y;
    uint32_t skip_slot = slot;
    // Row metadata and candidate header of a position are fetched one position early, so that its candidates and
    // predecessors can be requested as soon as the position starts (one round trip less on the chain).
    uint2 m_cur = make_uint2(0, 0);
    uint4 info_cur = make_uint4(0, 0, 0, 0);
    if (slot < slot_end) {
        m_cur = b.ends_meta[slot];
        info_cur = load_info(b, slot);
    }
    const uint32_t group_mask = G == 32 ? kFull : (((1u << (G & 31)) - 1u) << (sub * G));
    while (__any_sync(kFull, slot < slot_end)) {
        const bool active = slot < slot_end;
        uint32_t K = 0, eo = 0;
        uint4 info = make_uint4(0, 0, 0, 0);
        if (active) {
            eo = m_cur.x;
            K = m_cur.y - m_cur.x;
            info = info_cur;
        }
        // A fill count read this early misses the nodes this very position appends to the next row: k_fix
        // carries the count the group itself wrote there.
        uint2 m_nx = make_uint2(0, 0);
        uint4 info_nx = make_uint4(0, 0, 0, 0);
        uint32_t k_fix = 0;
        if (active && slot + 1 < slot_end) {
            m_nx = b.ends_meta[slot + 1];
            info_nx = load_info(b, slot + 1);
        }
        // positions inside a skipped space run are never start_node; K == 0: has_previous_node fails
        bool visit = active && slot >= skip_slot && K != 0;  // (lattice.rs:155-157, tokenizer.rs:110-114)
        if (visit && (info.w & kInfoTrailing)) {  // tokenizer.rs:128-130: EOS starts here, the sweep ends
            slot_end = slot;
            visit = false;
        }
        if (visit && info.z) skip_slot = slot + info.z + 1;  // next start_node = start_word + 1 (tokenizer.rs:134-135)
        const uint32_t ncand = visit ? info.y : 0;
        if (COUNT && stats && visit && gl == 0) {
            uint4 stv = stats[slot];
            cWalks += stv.x >> 24;
            cM += stv.x & 0xFFFFFFu;
            cT += stv.y;
            cP += stv.z;
            cW += stv.w;
            cntE += (unsigned long long)K * ncand;
            cntN += ncand;
        }
        const uint32_t max_cand = __reduce_max_sync(kFull, ncand);
        // first chunk of predecessors: independent of the candidates, so issue it alongside their load
        int2 pr_first = make_int2(0, 0);
        if (visit && gl < K) pr_first = b.ends_hot[eo + gl];
        for (uint32_t c0 = 0; c0 < max_cand; c0 += G) {
            const bool valid = c0 + gl < ncand;
            uint4 cd = make_uint4(0, 0, 0, 0);
            uint32_t fill = 0;
            if (valid) {
                cd = cand_at(d, [&](uint32_t h) { return __ldg(&b.seg[info.x + h]); }, slot, c0 + gl);
                // row metadata of the node's end position: independent of the minimum search, fetch now
                const uint2 me = b.ends_meta[cd.w];
                fill = me.y;  // next free entry of that row (absolute)
            }
            const uint32_t left = cd.x & 0xFFFFu;
            const ConnRow<CONN> conn(d, left);
            // Lattice::add_connid_counts (lattice.rs:170-176): one (left, pred.right) edge per predecessor
            if (COUNT && b.lid_count && valid) atomicAdd(&b.lid_count[left], (unsigned long long)K);
            // Lattice::search_min_node (lattice.rs:129-151): `<=` keeps the LAST minimum
            int32_t best = INT32_MAX;
            uint32_t bestk = 0;
            const uint32_t Kv = valid ? K : 0;
            const uint32_t max_k = __reduce_max_sync(kFull, Kv);
            for (uint32_t k0 = 0; k0 < max_k; k0 += G) {
                int2 pr = pr_first;
                if (k0 != 0) {
                    pr = make_int2(0, 0);
                    if (k0 + gl < K) pr = b.ends_hot[eo + k0 + gl];
                }
                if (COUNT && b.rid_count && c0 == 0 && k0 + gl < K && ncand)
                    atomicAdd(&b.rid_count[uint32_t(pr.y)], (unsigned long long)ncand);
                const uint32_t kc = min(uint32_t(G), max_k - k0);
#pragma unroll 8
                for (uint32_t kk = 0; kk < kc; ++kk) {
                    int32_t pc = __shfl_sync(kFull, pr.x, kk, G);
                    uint32_t prr = uint32_t(__shfl_sync(kFull, pr.y, kk, G));
                    if (k0 + kk < Kv) {
                        // MatrixConnector::cost (matrix_connector.rs:79-85,121-124); i32 wrapping add
                        int32_t v = int32_t(uint32_t(pc) + uint32_t(conn.cost(d, prr)));
                        if (v <= best) {
                            best = v;
                            bestk = k0 + kk;
                        }
                    }
                }
            }
            const uint32_t row_fill = insert_node(b, valid, cd, best, slot, eo, bestk, fill);
            if (row_fill && cd.w == slot + 1) k_fix = row_fill;
        }
        k_fix = __reduce_max_sync(group_mask, k_fix);  // fills only grow: the last chunk's count is the largest
        m_cur = make_uint2(m_nx.x, max(m_nx.y, k_fix));
        info_cur = info_nx;
        if (slot < slot_end) ++slot;
    }

    const SentenceEnd e = insert_eos<G, ConnRow<CONN>>(d, b, sidx, slot_end, gl);
    if (COUNT) {
        cntE += e.K;
        if (b.lid_count && e.n > 0) {  // lattice.rs:178-181: the EOS edges are counted over ends[len_char]
            const uint2 ml = b.ends_meta[e.base + e.n];
            const uint32_t nl = ml.y - ml.x;
            for (uint32_t k = gl; k < nl; k += G) atomicAdd(&b.rid_count[uint32_t(b.ends_hot[ml.x + k].y)], 1ull);
            if (gl == 0 && nl) atomicAdd(&b.lid_count[0], (unsigned long long)nl);
        }
        if (b.counters && e.n > 0 && gl == 0) {
            atomicAdd(&b.counters[kCntE], cntE);
            atomicAdd(&b.counters[kCntN], cntN);
            atomicAdd(&b.counters[kCntM], cM);
            atomicAdd(&b.counters[kCntT], cT);
            atomicAdd(&b.counters[kCntP], cP);
            atomicAdd(&b.counters[kCntW], cW);
            atomicAdd(&b.counters[kCntWalks], cWalks);
        }
    }
}

template <int G, bool COUNT, int CONN>
__global__ void __launch_bounds__(128, (CONN == 0 && !COUNT) ? VBT_K3_MIN_BLOCKS : 8) k_viterbi(DictView d, Batch b, const uint4* __restrict__ stats) {
    if (stand_down(*b.flags)) return;
    constexpr uint32_t SPW = 32 / G;  // sentences per warp
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    viterbi_sweep<G, COUNT, CONN>(d, b, stats, warp * SPW + (threadIdx.x & 31) / G);
}

// ---------------------------------------------------------------------------------------------
// K3, second design (round 2).  Same mapping as k_viterbi (G lanes per sentence, lane = candidate, sequential over
// start positions), rebuilt around what the r01f profile showed to be the limits — warp-instruction issue and the
// LSU data pipe of the L1 (shuffles, spills and gathers all queue there):
//   * the predecessors {cost, right} of a position are staged once in shared memory and read back two at a time
//     with one LDS.128 (a broadcast inside the group) instead of two SHFL per predecessor;
//   * the gather address is one multiply-add on a per-candidate column pointer (the matrix is stored transposed);
//   * no state is carried across positions except three slot numbers: nothing spills at 32 registers;
//   * exact lower-bound pruning (PRUNE): every candidate record carries lb = min over ALL right ids of
//     M[right][left], so a predecessor with cost + lb > best-so-far cannot reach the minimum, not even tie it,
//     and its gather is skipped.  Predecessors are still visited in row order with `<=`, so the LAST minimal one
//     wins exactly as in Lattice::search_min_node (lattice.rs:129-151).  The bound arithmetic assumes that no i32
//     addition wraps: batches holding a sentence longer than kPruneMaxChars characters take the unpruned path,
//     which keeps the reference's wrapping adds.
// ---------------------------------------------------------------------------------------------

#ifndef VBT_K3V2_WARPS
#define VBT_K3V2_WARPS 4  // warps per block of k_viterbi2
#endif
#ifndef VBT_K3V2_MIN_BLOCKS
// 48 warps per SM = 40 registers per thread.  On H100 the 32-register build (64 warps) spills in the search loop;
// measured on an H100 SXM 80 GB at 700 W with 16 lanes per sentence, the 40-register build (no spills in the pruned
// instantiations) runs the 1 M-sentence synth-unidic batch in 14.1 ms against 18.4 ms (32 warps, 43 registers:
// 14.8 ms).
#define VBT_K3V2_MIN_BLOCKS (48 / VBT_K3V2_WARPS)
#endif

constexpr int kPredCap = 32;                             // predecessors staged per pass
constexpr int32_t kPredSentinel = INT32_MAX - 70000;     // + any i16 stays below INT32_MAX and above every real best

// Connection cost into one fixed left id for k_viterbi2.
template <int CONN>
struct ConnCol;
template <>
struct ConnCol<0> {
    // The engine places the matrix so that it does not cross a 4 GiB boundary (DictView::matrix_window): the
    // high address word is then the same for every entry and a lookup is ONE multiply-add on the low word,
    //     lo = right * (2 * stride_right) + colbase,   colbase = lo(matrix) + 2 * stride_left * left,
    // followed by the 2-byte load.  colbase / stride / hi are opaque (volatile asm) so that the compiler keeps
    // them in registers across the predecessor loop instead of recomputing them from the left id per lookup,
    // which is what it does when squeezed into 32 registers.
    uint32_t colbase, stride2, hi, zero;
    __device__ __forceinline__ ConnCol(const DictView& d, uint32_t left) {
        zero = d.opaque_zero;
        const unsigned long long base = reinterpret_cast<unsigned long long>(d.matrix);
        asm volatile("mad.lo.u32 %0, %1, %2, %3;" : "=r"(colbase) : "r"(left), "r"(d.conn_stride_left * 2u), "r"(uint32_t(base)));
        stride2 = d.conn_stride_right * 2u;  // uniform: the compiler may keep these two in uniform registers
        hi = uint32_t(base >> 32);
    }
    __device__ __forceinline__ int32_t cost(const DictView&, uint32_t right) const {
        int32_t m;
        asm("{\n\t.reg .u32 lo;\n\t.reg .u64 a;\n\tmad.lo.u32 lo, %1, %2, %3;\n\tmov.b64 a, {lo, %4};\n\t"
            "ld.global.nc.s16 %0, [a];\n\t}"
            : "=r"(m)
            : "r"(right), "r"(stride2), "r"(colbase), "r"(hi));
        return m;
    }
    // Two predecessors of Lattice::search_min_node, staged at shared address `pp` as {cost, right} pairs.  Phase 1
    // tests both (PRUNE: cost + lb <= best, lb = cost_word >> 16; otherwise: its address lies below `plim`, the end
    // of this lane's row) and issues the surviving 2-byte gathers together; phase 2 folds them in row order with
    // `<=`, so the LAST minimum wins.  A bound that is one batch old is still a bound: `best` only falls.  The shared
    // address of the winner is its token (`besttok`).
#define VBT_V2_DECL(i) ".reg .pred p" #i ";\n\t.reg .s32 c" #i ", m" #i ";\n\t.reg .u32 r" #i ", l" #i ";\n\t.reg .u64 a" #i ";\n\t"
#define VBT_V2_TEST_PRUNE(i) "add.s32 t, c" #i ", lb;\n\tsetp.le.s32 p" #i ", t, %0;\n\t"
#define VBT_V2_TEST_PLAIN(i) "add.u32 l" #i ", %2, " #i "*8;\n\tsetp.lt.u32 p" #i ", l" #i ", %3;\n\t"
#define VBT_V2_LOAD(i) \
    "mad.lo.u32 l" #i ", r" #i ", %4, %5;\n\tmov.b64 a" #i ", {l" #i ", %6};\n\t@p" #i " ld.global.nc.s16 m" #i ", [a" #i "];\n\t"
#define VBT_V2_FOLD(i) \
    "@p" #i " add.s32 t, c" #i ", m" #i ";\n\tsetp.le.and.s32 q, t, %0, p" #i ";\n\tselp.s32 %0, t, %0, q;\n\t" \
    "add.u32 k, %2, " #i "*8;\n\tselp.u32 %1, k, %1, q;\n\t"
#define VBT_V2_HEAD "{\n\t.reg .pred q;\n\t.reg .s32 t, lb;\n\t.reg .u32 k;\n\t"
#define VBT_V2_OPERANDS \
    : "+r"(best), "+r"(besttok) : "r"(pp), "r"(PRUNE ? cost_word : plim), "r"(stride2), "r"(colbase), "r"(hi)
    // `zero` is a run-time zero the compiler cannot see through: the first fold reads m0 | (m1 & zero) = m0, one
    // LOP3 that needs BOTH gathers, so the two loads are issued back to back (left alone, ptxas at 32 registers
    // sinks the second load below the first fold and the two round trips serialise).
#define VBT_V2_FOLD0_JOIN \
    "lop3.b32 k, m0, m1, %7, 0xF8;\n\t@p0 add.s32 t, c0, k;\n\tsetp.le.and.s32 q, t, %0, p0;\n\t" \
    "selp.s32 %0, t, %0, q;\n\tselp.u32 %1, %2, %1, q;\n\t"
    template <bool PRUNE>
    __device__ __forceinline__ void batch2(uint32_t pp, uint32_t cost_word, uint32_t plim, int32_t& best,
                                           uint32_t& besttok) const {
        if (PRUNE)
            asm volatile(VBT_V2_HEAD VBT_V2_DECL(0) VBT_V2_DECL(1) "ld.shared.v4.b32 {c0, r0, c1, r1}, [%2];\n\tshr.s32 lb, %3, 16;\n\t"
                         VBT_V2_TEST_PRUNE(0) VBT_V2_TEST_PRUNE(1) VBT_V2_LOAD(0) VBT_V2_LOAD(1)  //
                         VBT_V2_FOLD0_JOIN VBT_V2_FOLD(1) "}" VBT_V2_OPERANDS, "r"(zero));
        else
            asm volatile(VBT_V2_HEAD VBT_V2_DECL(0) VBT_V2_DECL(1) "ld.shared.v4.b32 {c0, r0, c1, r1}, [%2];\n\t"
                         VBT_V2_TEST_PLAIN(0) VBT_V2_TEST_PLAIN(1) VBT_V2_LOAD(0) VBT_V2_LOAD(1)  //
                         VBT_V2_FOLD0_JOIN VBT_V2_FOLD(1) "}" VBT_V2_OPERANDS, "r"(zero));
    }
};

// Raw / Dual connectors: plain C++ over ConnRow::cost, same interface.
template <int CONN>
struct ConnCol : ConnRow<CONN> {
    const DictView& dv;
    __device__ __forceinline__ ConnCol(const DictView& d, uint32_t left) : ConnRow<CONN>(d, left), dv(d) {}
    template <bool PRUNE>
    __device__ __forceinline__ void batch2(uint32_t pp, uint32_t, uint32_t plim, int32_t& best, uint32_t& besttok) const {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const uint32_t p = pp + 8 * i;
            if (p < plim) {
                int2 pr;
                asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(pr.x), "=r"(pr.y) : "r"(p));
                const int32_t v = int32_t(uint32_t(pr.x) + uint32_t(this->cost(dv, uint32_t(pr.y))));  // i32 wrapping add
                if (v <= best) {
                    best = v;
                    besttok = p;
                }
            }
        }
    }
};

// Shared-memory window of one warp of k_viterbi2: a staging row per sentence ({cost, right} of the predecessors, up
// to kPredCap per pass plus padding to whole batches; the odd multiple of 32 bytes skews the rows across the banks),
// and per sentence the descriptor of its current position {seg_ptr, slot, row offset, K}, its candidate count and
// its first G segments.
template <int G>
struct V2Shared {
    static constexpr uint32_t SPW = 32 / G;
    static constexpr uint32_t kRowBytes = (kPredCap + 4) * 8;
    int2 rows[SPW][kPredCap + 4];
    uint4 desc[SPW];
    uint32_t cnt[8];
    uint2 segs[SPW][G];
};

template <int G, int CONN, bool PRUNE, bool SPACE>
__device__ __forceinline__ void viterbi2_sweep(const DictView& d, const Batch& b, const uint32_t sw /* shared-window address of this warp's V2Shared */) {
    constexpr uint32_t SPW = 32 / G;  // sentences per warp
    constexpr uint32_t kRowBytes = V2Shared<G>::kRowBytes;
    constexpr uint32_t kDescOff = SPW * kRowBytes, kCntOff = kDescOff + SPW * 16, kSegOff = kCntOff + 8 * 4;
    static_assert(kSegOff == offsetof(V2Shared<G>, segs), "V2Shared layout");
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t gl = lane % G, sub = lane / G;
    const uint32_t sidx = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * SPW + sub;

    const uint2 range = begin_sentence(b, sidx, gl);
    uint32_t slot = range.x, slot_end = range.y;
    uint32_t skip_slot = slot;
    while (__any_sync(kFull, slot < slot_end)) {
        uint32_t K = 0, eo = 0, cptr = 0, ncand = 0;
        if (slot < slot_end) {  // two independent loads, one round trip
            const uint2 m = b.ends_meta[slot];
            const uint2 inf = b.info[slot];
            eo = m.x;
            K = m.y - m.x;
            // positions inside a skipped space run are never start_node; K == 0: has_previous_node fails
            if ((!SPACE || slot >= skip_slot) && K != 0) {  // (lattice.rs:155-157, tokenizer.rs:110-114)
                cptr = inf.x;
                ncand = inf.y;
            }
        }
        if (SPACE && (ncand & kInfoSpecial)) {
            ncand &= ~kInfoSpecial;
            const uint2 ex = b.info_ex[slot];
            if (ex.y & kInfoTrailing) {  // tokenizer.rs:128-130: EOS starts here, the sweep ends
                slot_end = slot;
                ncand = 0;
            } else if (ex.x) {
                skip_slot = slot + ex.x + 1;  // next start_node = start_word + 1 (tokenizer.rs:134-135)
            }
        }
        if (ncand == 0) K = 0;
        // The position's first G segments, one per lane of the group, for the lanes that take its candidates below
        // (a position rarely has more; those are read from the pool).  Loaded now, stored to shared memory after the
        // predecessor copies are under way.  Past the position's own segments a lane loads a neighbour's: unused.
        const bool stage = ncand != 0 && cptr + gl < b.seg_cap;
        uint2 sg = make_uint2(0, 0);
        if (stage) sg = __ldg(&b.seg[cptr + gl]);
        const uint32_t max_k = __reduce_max_sync(kFull, K);
        // The candidates of the warp's sentences are dealt to the 32 lanes as ONE pool (sentence after sentence):
        // a position with 3 candidates next to one with 13 fills half a warp, not two rounds of 8-lane groups.
        // Every group publishes its position; a lane then finds which sentence its pool index falls into.
        if (gl == 0) {
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sw + kDescOff + sub * 16u), "r"(cptr), "r"(slot),
                         "r"(eo), "r"(K)
                         : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(sw + kCntOff + sub * 4u), "r"(ncand) : "memory");
        }
        const uint32_t total = __reduce_add_sync(kFull, gl == 0 ? ncand : 0u);
        // Staging of the predecessors {cost, right} of every sentence's row, padded with sentinels to whole batches.
        // In the usual case (no row longer than kPredCap) it is started here with asynchronous copies (cp.async:
        // global -> shared without a register or a scoreboard entry in between) so that it overlaps the loads of
        // the candidates below; the copies are awaited right before the first batch.  Rows are 8-byte aligned only,
        // which rules out the 16-byte granular bulk copies (cp.async.bulk).
        const bool one_pass = max_k <= uint32_t(kPredCap);
        if (one_pass && total) {
            const uint32_t n_stage = (max_k + 1u) & ~1u;
            const uint32_t own = sw + sub * kRowBytes;
#pragma unroll 1
            for (uint32_t k = gl; k < n_stage; k += G) {
                if (k < K)
                    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(own + k * 8u), "l"(b.ends_hot + eo + k) : "memory");
                else
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(own + k * 8u), "r"(kPredSentinel), "r"(0) : "memory");
            }
        }
        if (stage)
            asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(sw + kSegOff + lane * 8u), "r"(sg.x), "r"(sg.y) : "memory");
        __syncwarp();
        for (uint32_t q0 = 0; q0 < total; q0 += 32) {
            const uint32_t q = q0 + lane;
            const bool valid = q < total;
            uint32_t s2 = 0, before = 0;
            {
                bool adv = true;
#pragma unroll
                for (uint32_t i = 0; i + 1 < SPW; ++i) {
                    uint32_t c;
                    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(c) : "r"(sw + kCntOff + i * 4u));
                    adv = adv && q >= before + c;
                    if (adv) {
                        before += c;
                        s2 = i + 1;
                    }
                }
            }
            uint4 ds;  // {seg_ptr, slot, row offset, K} of the sentence this lane's candidate belongs to
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(ds.x), "=r"(ds.y), "=r"(ds.z), "=r"(ds.w)
                         : "r"(sw + kDescOff + s2 * 16u));
            uint4 cd = make_uint4(0, 0, 0, 0);
            uint32_t nxt = 0;
            if (valid) {
                const uint32_t segs = sw + kSegOff + s2 * (G * 8u);  // lane (s2, h) staged segment h
                cd = cand_at(
                    d,
                    [&](uint32_t h) {
                        uint2 s;
                        if (h < uint32_t(G))
                            asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(s.x), "=r"(s.y) : "r"(segs + h * 8u));
                        else
                            s = __ldg(&b.seg[ds.x + h]);
                        return s;
                    },
                    ds.y, q - before);
                // next free entry of the row the node ends in: independent of the search, and of the record's load
                nxt = b.ends_meta[cd.w].y;
            }
            const ConnCol<CONN> conn(d, cd.x & 0xFFFFu);
            // Lattice::search_min_node (lattice.rs:129-151): `<=` keeps the LAST minimum
            int32_t best = (PRUNE && !valid) ? INT32_MIN : INT32_MAX;  // INT32_MIN: nothing passes the bound
            uint32_t bestk = 0;
#pragma unroll 1
            for (uint32_t k0 = 0; k0 < max_k; k0 += kPredCap) {
                // This pass covers predecessors [k0, k0 + kc) of every row, staged by the row's own group and padded
                // with sentinels to whole batches of two.
                const uint32_t kc = min(uint32_t(kPredCap), max_k - k0);
                const uint32_t n_stage = (kc + 1u) & ~1u;
                if (one_pass) {
                    if (q0 == 0) {  // the copies started above have had the candidates' round trip to arrive
                        asm volatile("cp.async.wait_all;" ::: "memory");
                        __syncwarp();
                    }
                } else {  // rows longer than kPredCap: pass after pass, staged synchronously
                    __syncwarp();
                    const uint32_t own = sw + sub * kRowBytes;
#pragma unroll 1
                    for (uint32_t k = gl; k < n_stage; k += G) {
                        int2 pr = make_int2(kPredSentinel, 0);
                        if (k0 + k < K) pr = b.ends_hot[eo + k0 + k];
                        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(own + k * 8u), "r"(pr.x), "r"(pr.y) : "memory");
                    }
                    __syncwarp();
                }
                // the shared address of a predecessor doubles as its token: index = k0 + (token - row) / 8
                const uint32_t row = sw + s2 * kRowBytes;
                const uint32_t plim = row + (valid ? min(ds.w - min(ds.w, k0), kc) : 0u) * 8u;  // end of this lane's row
                uint32_t besttok = kNone;
                const uint32_t pend = row + n_stage * 8u;
#pragma unroll 1
                for (uint32_t pp = row; pp < pend; pp += 16u) conn.template batch2<PRUNE>(pp, cd.y, plim, best, besttok);
                if (besttok != kNone) bestk = k0 + ((besttok - row) >> 3);
            }
            insert_node(b, valid, cd, best, ds.y, ds.z, bestk, nxt);
        }
        if (slot < slot_end) ++slot;
    }
    insert_eos<G, ConnCol<CONN>>(d, b, sidx, slot_end, gl);
}

// PRUNE and its unpruned twin are separate kernels launched back to back (each keeps its own register allocation);
// the one the batch does not call for — kFlagLongSentence decides, and only the device knows it — returns at once.
// SPACE = the tokenizer ignores spaces: only then can a position carry a skip or the trailing flag.
template <int G, int CONN, bool PRUNE, bool SPACE, bool TWIN>
__global__ void __launch_bounds__(32 * VBT_K3V2_WARPS, CONN == 0 ? VBT_K3V2_MIN_BLOCKS : (32 / VBT_K3V2_WARPS)) k_viterbi2(DictView d, Batch b) {
    const uint32_t batch_flags = *b.flags;
    if (stand_down(batch_flags)) return;
    if (TWIN && PRUNE == ((batch_flags & kFlagLongSentence) != 0)) return;
    __shared__ __align__(16) V2Shared<G> s_warp[VBT_K3V2_WARPS];
    const uint32_t sp = uint32_t(__cvta_generic_to_shared(&s_warp[threadIdx.x >> 5]));
    viterbi2_sweep<G, CONN, PRUNE, SPACE>(d, b, sp);
}

// ---------------------------------------------------------------------------------------------
// K4: Lattice::append_top_nodes (lattice.rs:159-168) + Token accessors (token.rs:21-92)
// ---------------------------------------------------------------------------------------------

// f(entry, end position) for each node of sentence s's best path, from EOS back (base = the sentence's first slot).
template <class F>
__device__ __forceinline__ void walk_best(const Batch& b, uint32_t s, uint32_t base, F f) {
    const uint4 eo = b.eos[s];
    if (eo.x == kNone) return;
    uint32_t cur = eo.x, end_node = eo.y;
    while (end_node != 0) {
        const uint4 c = b.ends_cold[cur];
        f(cur, end_node);
        end_node = c.x - base;
        cur = c.y;
    }
}

// The 24-byte vbt_token record at t of the lattice entry whose ends_cold word is c, ending at slot end_slot of the
// sentence whose first slot is base, with `total` as its total cost.  start_char is the entry's start_word
// (token.rs:21-24), the bytes are those of start_word and the end (token.rs:28-32).
__device__ __forceinline__ void write_node_record(const Batch& b, uint2* t, uint32_t base, uint32_t end_slot, const uint4& c,
                                                  uint32_t total) {
    const uint32_t start_node = c.x - base;
    const uint32_t start_word = start_node + ((b.info[c.x].y & kInfoSpecial) ? b.info_ex[c.x].x : 0u);
    t[0] = make_uint2(start_word, end_slot - base);
    t[1] = make_uint2(b.byte_pos[base + start_word], b.byte_pos[end_slot]);
    t[2] = make_uint2(c.z, total);  // word_idx, total_cost
}

// The path walk (backtrack_count_one, a thread per sentence) counts the tokens and leaves, for the k-th node from the
// end, {lattice entry, end position} in the sentence's own stretch of `ends_meta` (dead after K3, one entry per
// character, and a path has at most one node per character).  Once the token offsets are known the records are built
// from those entries — the pointer chase is not repeated and neighbouring lanes write neighbouring records.
// It chases the path itself rather than through walk_best: that would load the slot offset before the EOS entry, and
// k_backtrack, which inlines this, is on the hot path.
__device__ __forceinline__ void backtrack_count_one(const Batch& b, uint32_t s) {
    uint4 e = b.eos[s];
    uint32_t k = 0;
    if (e.x != kNone) {
        const uint32_t base = b.slot_off[s];
        uint32_t cur = e.x, end_node = e.y;
        while (end_node != 0) {
            uint4 c = b.ends_cold[cur];
            b.ends_meta[base + k] = make_uint2(cur, end_node);
            ++k;
            end_node = c.x - base;
            cur = c.y;
        }
    }
    b.n_tok[s] = k;
    if (b.counters && k) atomicAdd(&b.counters[kCntK], (unsigned long long)k);
}

// Token records of sentence s at tok_off[s], from the path entries backtrack_count_one left (a warp per sentence).
__device__ __forceinline__ void backtrack_write_one(const Batch& b, uint32_t s, uint32_t lane) {
    const uint32_t base = b.slot_off[s];
    const unsigned long long t0 = b.tok_off[s];
    const uint32_t n = uint32_t(b.tok_off[s + 1] - t0);
    uint2* out = reinterpret_cast<uint2*>(b.tokens);
    // the record of write_node_record, spelled out: k_small_batch, which inlines this, keeps its code that way
    for (uint32_t k = lane; k < n; k += 32) {
        const uint2 pe = b.ends_meta[base + k];  // k-th node from the end of the path
        const uint4 c = b.ends_cold[pe.x];
        const uint32_t end_node = pe.y;
        const uint32_t start_node = c.x - base;
        const uint2 i8 = b.info[c.x];
        const uint32_t start_word = start_node + ((i8.y & kInfoSpecial) ? b.info_ex[c.x].x : 0u);  // token.rs:21-24 uses start_word
        const uint2 bytes = make_uint2(b.byte_pos[base + start_word], b.byte_pos[base + end_node]);  // token.rs:28-32
        if (b.compact) {  // opt-in 16-byte record: the character range is a function of the caller's own UTF-8
            reinterpret_cast<uint4*>(b.tokens)[t0 + (n - 1 - k)] = make_uint4(bytes.x, bytes.y, c.z, c.w);
            continue;
        }
        uint2* t = out + (t0 + (n - 1 - k)) * 3;
        t[0] = make_uint2(start_word, end_node);
        t[1] = bytes;
        t[2] = make_uint2(c.z, c.w);  // word_idx, total_cost
    }
}

// K4: backtrack_count + token-offset scan + records, one pass over tiles of TILE consecutive sentences: a thread
// chases each sentence's path, the tile looks back for its token offset (tile_prefix), then the block (256 threads)
// writes the tile's records, which are contiguous, a thread per record.  MARG: with the marginal of every token,
// prob = exp(â + b̂ - â(EOS)) of its lattice entry.  A rejected batch (stand_down) gets no records and zero token
// offsets.  TILE = kBackTile, or kBackTileSmall for batches too small to give every SM a kBackTile tile.
static_assert(kBackTile == 256, "a thread per sentence, eight warps");

template <bool MARG, uint32_t TILE>
__global__ void __launch_bounds__(256) k_backtrack(Batch b, MargArgs m, unsigned long long* tile_state,
                                                   uint32_t* ticket) {
    __shared__ uint32_t s_off[TILE + 1], s_base[TILE], s_warp[8];
    __shared__ uint32_t s_tile;
    __shared__ unsigned long long s_excl;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t tile = take_tile(ticket, &s_tile);
    const uint32_t s0 = tile * TILE, nt = min(TILE, b.n_sent - s0);
    const bool stand = stand_down(*b.flags);
    const uint32_t s = s0 + threadIdx.x;
    uint32_t k = 0;
    if (!stand && threadIdx.x < nt) {
        backtrack_count_one(b, s);
        k = b.n_tok[s];
        s_base[threadIdx.x] = b.slot_off[s];
    }
    uint32_t x = k;  // block-wide exclusive scan of the token counts
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(kFull, x, o);
        if (lane >= uint32_t(o)) x += y;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    uint32_t before = 0, agg = 0;
    for (uint32_t i = 0; i < 8; ++i) {
        before += i < wid ? s_warp[i] : 0u;
        agg += s_warp[i];
    }
    const uint32_t local = before + x - k;
    if (threadIdx.x < TILE) s_off[threadIdx.x] = local;  // == agg from thread nt on
    if (threadIdx.x == 255) s_off[TILE] = agg;
    if (wid == 0) {
        const unsigned long long excl = tile_prefix(tile_state, tile, agg, lane);
        if (lane == 0) {
            s_excl = excl;
            if (s0 + nt == b.n_sent) b.tok_off[b.n_sent] = excl + agg;
        }
    }
    __syncthreads();
    const unsigned long long excl = s_excl;
    if (threadIdx.x < nt) b.tok_off[s] = excl + local;
    if (stand) return;
    // kRecBatch records per thread at a time, each gather step issued for all of them before the next: the chain
    // path entry -> ends_cold -> info -> byte_pos is three dependent round trips per record
    constexpr uint32_t kRecBatch = 4;
#pragma unroll 1
    for (uint32_t i0 = threadIdx.x; i0 < agg; i0 += 256 * kRecBatch) {
        uint32_t j[kRecBatch];
        uint2 pe[kRecBatch];
        uint4 c[kRecBatch];
        uint2 i8[kRecBatch];
#pragma unroll
        for (uint32_t q = 0; q < kRecBatch; ++q) {
            const uint32_t i = i0 + q * 256;
            j[q] = 0;  // the tile's sentence of token i: the last j with s_off[j] <= i
            for (uint32_t step = TILE / 2; step > 0; step >>= 1)
                if (j[q] + step < nt && s_off[j[q] + step] <= i) j[q] += step;
            const uint32_t n = s_off[j[q] + 1] - s_off[j[q]];
            if (i < agg) pe[q] = b.ends_meta[s_base[j[q]] + (n - 1 - (i - s_off[j[q]]))];  // the kk-th node from the end
        }
#pragma unroll
        for (uint32_t q = 0; q < kRecBatch; ++q)
            if (i0 + q * 256 < agg) c[q] = b.ends_cold[pe[q].x];
#pragma unroll
        for (uint32_t q = 0; q < kRecBatch; ++q)
            if (i0 + q * 256 < agg) i8[q] = b.info[c[q].x];
#pragma unroll
        for (uint32_t q = 0; q < kRecBatch; ++q) {
            const uint32_t i = i0 + q * 256;
            if (i >= agg) break;
            const uint32_t base = s_base[j[q]], start_node = c[q].x - base;
            const uint32_t start_word = start_node + ((i8[q].y & kInfoSpecial) ? b.info_ex[c[q].x].x : 0u);  // token.rs:21-24
            const uint2 bytes = make_uint2(b.byte_pos[base + start_word], b.byte_pos[base + pe[q].y]);  // token.rs:28-32
            if (b.compact) {
                reinterpret_cast<uint4*>(b.tokens)[excl + i] = make_uint4(bytes.x, bytes.y, c[q].z, c[q].w);
            } else {
                uint2* t = reinterpret_cast<uint2*>(b.tokens) + (excl + i) * 3;
                t[0] = make_uint2(start_word, pe[q].y);
                t[1] = bytes;
                t[2] = make_uint2(c[q].z, c[q].w);  // word_idx, total_cost
            }
            if (MARG) {
                const double2 ab = m.ab[pe[q].x];
                m.token_prob[excl + i] = float(exp(ab.x + ab.y - m.a_eos[s0 + j[q]]));
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Marginals (MargArgs in kernels.cuh): one warp per sentence, positions left to right (forward) and right to left
// (backward).  A lane owns one node at a time and folds that node's terms sequentially.
// ---------------------------------------------------------------------------------------------

// log(exp(a) + exp(b)) with -inf as the empty sum
__device__ __forceinline__ double lse2(double a, double b) {
    const double hi = fmax(a, b), lo = fmin(a, b);
    return lo == -INFINITY ? hi : hi + log1p(exp(lo - hi));
}

// Folds the path of cost x that reaches a node with log weight `a` (relative to its own prefix minimum) into the
// running {rmin, L}: rmin = the least cost so far, L = log-sum-exp relative to rmin.
__device__ __forceinline__ void marg_push(long long x, double a, double theta, long long& rmin, double& L) {
    if (x < rmin) {
        if (rmin != LLONG_MAX) L -= theta * double(rmin - x);
        rmin = x;
    }
    L = lse2(L, a - theta * double(x - rmin));
}

// The sentence of warp `sidx` as {first slot, sentinel slot}, or false without one.
__device__ __forceinline__ bool marg_sentence(const Batch& b, uint32_t sidx, uint32_t& s, uint32_t& base, uint32_t& last) {
    if (sidx >= b.n_sent) return false;
    s = b.order ? b.order[sidx] : sidx;
    base = b.slot_off[s];
    last = b.slot_off[s + 1] - 1;
    return true;
}

// LW: the sampling instantiation, which also keeps each entry's {left id, word cost} in m.lw.  LSE = false: the
// near-best lattice's instantiation, which writes only R, r_eos, ncand and cand_entry (no log-sum-exp, m.ab unread).
template <int CONN, bool LW = false, bool LSE = true>
__global__ void __launch_bounds__(256) k_marg_forward(DictView d, Batch b, MargArgs m) {
    if (stand_down(*b.flags)) return;
    const uint32_t lane = threadIdx.x & 31;
    uint32_t s, base, last;
    if (!marg_sentence(b, (blockIdx.x * blockDim.x + threadIdx.x) >> 5, s, base, last)) return;
    if (base == last) {  // an empty sentence: one (empty) path
        if (lane == 0) {
            m.r_eos[s] = 0;
            if (LSE) {
                m.a_eos[s] = 0.0;
                m.path_prob[s] = 1.f;
            }
        }
        return;
    }
    for (uint32_t i = lane; i <= last - base; i += 32) m.fill[base + i] = b.ends_meta[base + i].x + (i == 0 ? 1u : 0u);
    if (lane == 0) {  // BOS
        const uint32_t bos = b.ends_meta[base].x;
        m.R[bos] = 0;
        if (LSE) m.ab[bos] = make_double2(0.0, -INFINITY);
    }
    __syncwarp();
    const double th = m.theta;
    // the lattice entries of the candidates of the visited positions, numbered in position order from the sentence's
    // first row offset: there are fewer of them than the sentence's rows hold (BOS is one more)
    uint32_t centry = b.ends_meta[base].x;
    uint32_t slot_end = last, skip_slot = base;
    // the positions K3 visits, by the rules of its sweep (tokenizer.rs:110-135): a non-empty row, outside a skipped
    // space run, and the trailing flag ends the sweep
    for (uint32_t slot = base; slot < slot_end; ++slot) {
        const uint2 me = b.ends_meta[slot];  // final after K3: every node ending here came from an earlier position
        const uint32_t eo = me.x, K = me.y - me.x;
        const uint4 info = load_info(b, slot);
        const bool visit = slot >= skip_slot && K != 0;
        if (visit && (info.w & kInfoTrailing)) {
            slot_end = slot;
            break;
        }
        if (visit && info.z) skip_slot = slot + info.z + 1;
        const uint32_t ncand = visit ? info.y : 0;
        if (lane == 0) m.ncand[slot] = ncand;
        for (uint32_t c0 = 0; c0 < ncand; c0 += 32) {
            const uint32_t c = c0 + lane;
            const bool valid = c < ncand;
            uint4 cd = make_uint4(0, 0, 0, 0);
            uint32_t peers = 0, f = 0;
            const uint32_t vmask = __ballot_sync(kFull, valid);
            if (valid) {
                cd = cand_at(d, [&](uint32_t h) { return __ldg(&b.seg[info.x + h]); }, slot, c);
                peers = __match_any_sync(vmask, cd.w);
                f = m.fill[cd.w];
            }
            __syncwarp();
            if (valid) {  // the entry insert_node gave this candidate
                const uint32_t rank = __popc(peers & lanemask_lt());
                const uint32_t idx = f + rank;
                m.cand_entry[centry + c] = idx;
                if (rank == 0) m.fill[cd.w] = f + __popc(peers);
                const ConnRow<CONN> conn(d, cd.x & 0xFFFFu);
                const long long wc = int16_t(cd.y & 0xFFFFu);
                long long rmin = LLONG_MAX;
                double L = -INFINITY;
                for (uint32_t k = 0; k < K; ++k) {
                    const long long x = m.R[eo + k] + conn.cost(d, uint32_t(b.ends_hot[eo + k].y)) + wc;
                    if (LSE)
                        marg_push(x, m.ab[eo + k].x, th, rmin, L);
                    else
                        rmin = min(rmin, x);
                }
                m.R[idx] = rmin;
                if (LSE) m.ab[idx].x = L;
                if (LW) m.lw[idx] = (cd.x & 0xFFFFu) | (cd.y << 16);
            }
            __syncwarp();
        }
        centry += ncand;
    }
    if (lane == 0) {  // EOS: left id 0, no word cost
        const uint2 me = b.ends_meta[slot_end];
        const uint32_t K = me.y - me.x;
        const ConnRow<CONN> conn(d, 0);
        long long rmin = LLONG_MAX;
        double L = -INFINITY;
        for (uint32_t k = 0; k < K; ++k) {
            const long long x = m.R[me.x + k] + conn.cost(d, uint32_t(b.ends_hot[me.x + k].y));
            if (LSE)
                marg_push(x, m.ab[me.x + k].x, th, rmin, L);
            else
                rmin = min(rmin, x);
        }
        m.r_eos[s] = rmin;
        if (LSE) {
            m.a_eos[s] = L;
            m.path_prob[s] = K ? float(exp(-L)) : 0.f;
        }
    }
}

// The rows of a non-empty sentence right to left, as the backward passes walk them (a warp per sentence, a lane per
// entry; slot_end = the row EOS connects to), with the successors of each entry in the numbering k_marg_forward gave
// the candidates' entries:
//   eos(n, c)         each entry n of the row EOS connects to, c = conn(right(n), 0) (EOS: left id 0, no word cost);
//   row(n, nc, succ)  each entry n of every other row, nc = the candidates of its position (0 beyond EOS's row and at
//                     a position the sweep skips: n has no successor), and with nc > 0, succ(f) calls f(e, cost) for
//                     each successor entry e in candidate order, segment by segment; cost() = conn(right(n), left(e)) +
//                     wcost(e), looked up only when called.
template <int CONN, class Eos, class Row>
__device__ __forceinline__ void backward_rows(const DictView& d, const Batch& b, const MargArgs& m, uint32_t base, uint32_t last,
                                              uint32_t slot_end, uint32_t lane, Eos eos, Row row) {
    // one past the last candidate entry k_marg_forward numbered (it counts from the sentence's first row offset)
    uint32_t centry = 0;
    for (uint32_t slot = base + lane; slot < slot_end; slot += 32) centry += m.ncand[slot];
    centry = b.ends_meta[base].x + __reduce_add_sync(kFull, centry);
    for (uint32_t slot = last + 1; slot-- > base;) {
        const uint2 me = b.ends_meta[slot];
        const uint32_t eo = me.x, K = me.y - me.x;
        if (slot == slot_end) {
            const ConnRow<CONN> conn(d, 0);
            for (uint32_t k = lane; k < K; k += 32) eos(eo + k, conn.cost(d, uint32_t(b.ends_hot[eo + k].y)));
        } else {
            const uint32_t nc = slot < slot_end ? m.ncand[slot] : 0u;
            const uint32_t sptr = nc ? b.info[slot].x : 0u;
            centry -= nc;
            for (uint32_t k = lane; k < K; k += 32) {
                row(eo + k, nc, [&](auto f) {
                    const uint32_t right = uint32_t(b.ends_hot[eo + k].y);
                    uint32_t c = 0, end = slot;
                    for (uint32_t h = 0; c < nc; ++h) {
                        const uint2 sg = __ldg(&b.seg[sptr + h]);
                        end += uint32_t(int32_t(sg.y) >> 16);
                        for (uint32_t j = 0; j < (sg.y & 0xFFFFu); ++j, ++c) {
                            const uint4 cd = seg_record(d, sg, j, end);
                            const uint32_t e = m.cand_entry[centry + c];
                            f(e, [&] {
                                const ConnRow<CONN> conn(d, cd.x & 0xFFFFu);
                                return (long long)conn.cost(d, right) + int16_t(cd.y & 0xFFFFu);
                            });
                        }
                    }
                });
            }
        }
        __syncwarp();
    }
}

// UNC: the uncertainty instantiation (UncertaintyArgs in kernels.cuh), which also folds P(edge) * delta(edge) of every
// edge it visits into a float64 per lane and writes u.entropy and u.log_path_prob; the other reads no u.
template <int CONN, bool UNC = false>
__global__ void __launch_bounds__(256) k_marg_backward(DictView d, Batch b, MargArgs m, UncertaintyArgs u) {
    if (stand_down(*b.flags)) return;
    const uint32_t lane = threadIdx.x & 31;
    uint32_t s, base, last;
    if (!marg_sentence(b, (blockIdx.x * blockDim.x + threadIdx.x) >> 5, s, base, last)) return;
    if (base == last) {  // an empty sentence: one empty path
        if (UNC && lane == 0) {
            u.entropy[s] = 0.0;
            u.log_path_prob[s] = 0.0;
        }
        return;
    }
    const uint32_t slot_end = base + b.eos[s].y;  // the row EOS connects to
    const long long r_eos = m.r_eos[s];
    const double th = m.theta;
    // UNC: P(edge) = exp(â(k) + [b̂(c) - theta delta] - â(EOS)); no path at all (â(EOS) = -inf) folds nothing
    const double a_eos = UNC ? m.a_eos[s] : 0.0;
    const bool fold = UNC && a_eos != -INFINITY;
    double ed = 0.0;  // this lane's sum of P delta
    backward_rows<CONN>(
        d, b, m, base, last, slot_end, lane,
        [&](uint32_t n, long long c) {
            const long long x = m.R[n] + c;
            m.ab[n].y = -th * double(x - r_eos);
            if (fold) ed += exp(m.ab[n].x - th * double(x - r_eos) - a_eos) * double(x - r_eos);
        },
        [&](uint32_t n, uint32_t nc, auto succ) {
            double L = -INFINITY;  // no successor at all: -inf
            if (nc) {
                const long long rk = m.R[n];
                const double ak = fold ? m.ab[n].x - a_eos : 0.0;  // UNC: â(n) - â(EOS)
                succ([&](uint32_t e, auto cost) {
                    const long long x = rk + cost();
                    const double t = m.ab[e].y - th * double(x - m.R[e]);
                    L = lse2(L, t);
                    if (fold) ed += exp(ak + t) * double(x - m.R[e]);
                });
            }
            m.ab[n].y = L;
        });
    if (UNC) {  // the lanes' sums in a fixed order: a butterfly over lane indices
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ed += __shfl_xor_sync(kFull, ed, o);
        if (lane == 0) {
            u.entropy[s] = fold ? a_eos + th * ed : 0.0;
            u.log_path_prob[s] = fold ? -a_eos : -INFINITY;  // ln P(best) of no path at all: ln 0
        }
    }
}

// Boundary probabilities (UncertaintyArgs): a warp per sentence, a lane per row (position).  After k_marg_backward.
__global__ void __launch_bounds__(256) k_boundary_probs(Batch b, MargArgs m, UncertaintyArgs u) {
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (s >= b.n_sent) return;
    const uint32_t base = b.slot_off[s], last = b.slot_off[s + 1] - 1;
    if (lane == 0) {
        u.pos_off[s] = base;
        if (s + 1 == b.n_sent) u.pos_off[s + 1] = last + 1;
    }
    if (rows_unreadable(*b.flags)) return;
    if (base == last) {  // an empty sentence: its one (empty) path ends where it starts
        if (lane == 0) u.boundary_prob[base] = 1.f;
        return;
    }
    const double a_eos = m.a_eos[s];
    const bool path = a_eos != -INFINITY;
    for (uint32_t slot = base + lane; slot <= last; slot += 32) {
        float p = 0.f;
        if (path && slot == base) {
            p = 1.f;  // BOS
        } else if (path) {
            const uint2 me = b.ends_meta[slot];
            double sum = 0.0;
            for (uint32_t e = me.x; e < me.y; ++e) {
                const double2 ab = m.ab[e];
                sum += exp(ab.x + ab.y - a_eos);
            }
            p = float(sum);
        }
        u.boundary_prob[slot] = p;
    }
}

// Near-best lattice (MarginArgs in kernels.cuh): G(n), the least exact cost from entry n to EOS, over k_marg_backward's
// row walk (backward_rows) with min-plus in place of log-sum-exp.
template <int CONN>
__global__ void __launch_bounds__(256) k_margin_backward(DictView d, Batch b, MargArgs m, MarginArgs g) {
    if (stand_down(*b.flags)) return;
    const uint32_t lane = threadIdx.x & 31;
    uint32_t s, base, last;
    if (!marg_sentence(b, (blockIdx.x * blockDim.x + threadIdx.x) >> 5, s, base, last) || base == last) return;
    backward_rows<CONN>(
        d, b, m, base, last, base + b.eos[s].y, lane, [&](uint32_t n, long long c) { g.G[n] = c; },
        [&](uint32_t n, uint32_t nc, auto succ) {
            long long best = LLONG_MAX;  // no successor with a path to EOS: LLONG_MAX
            if (nc)
                succ([&](uint32_t e, auto cost) {
                    const long long ge = g.G[e];
                    if (ge != LLONG_MAX) best = min(best, ge + cost());
                });
            g.G[n] = best;
        });
}

// ---------------------------------------------------------------------------------------------
// Lattice output (LatticeArgs in kernels.cuh): one warp per sentence over the rows K3 filled, ends_meta[slot] =
// {row offset, fill}.  The first slot's row holds only BOS, which is not a node.
// ---------------------------------------------------------------------------------------------

// Nodes of the row of `slot` (i = slot - base); 0 for every row of an empty sentence
__device__ __forceinline__ uint32_t lattice_row_nodes(const Batch& b, uint32_t slot, uint32_t i, bool empty) {
    const uint2 me = b.ends_meta[slot];
    return me.y - me.x - ((i == 0 && !empty) ? 1u : 0u);
}

// The full lattice's numbering: row_base and n_nodes.
__global__ void __launch_bounds__(256) k_lattice_count(Batch b, LatticeArgs l) {
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (s >= b.n_sent) return;
    if (rows_unreadable(*b.flags)) {
        if (lane == 0) l.n_nodes[s] = 0;
        return;
    }
    const uint32_t base = b.slot_off[s], rows = b.slot_off[s + 1] - base;  // the sentinel's row included
    const bool empty = rows == 1;
    uint32_t run = 0;
    for (uint32_t i0 = 0; i0 < rows; i0 += 32) {
        const uint32_t i = i0 + lane;
        const uint32_t c = i < rows ? lattice_row_nodes(b, base + i, i, empty) : 0u;
        uint32_t x = c;  // inclusive warp scan
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(kFull, x, d);
            if (lane >= uint32_t(d)) x += y;
        }
        if (i < rows) l.row_base[base + i] = run + x - c;
        run += __shfl_sync(kFull, x, 31);
    }
    if (lane == 0) l.n_nodes[s] = run;
}

// The near-best lattice's numbering (MarginArgs): the kept nodes in node order, numbered through g.keep.
__global__ void __launch_bounds__(256) k_lattice_count_margin(Batch b, LatticeArgs l, MargArgs m, MarginArgs g) {
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (s >= b.n_sent) return;
    const uint32_t base = b.slot_off[s], last = b.slot_off[s + 1] - 1;
    // an empty sentence keeps nothing, and neither does one without a path
    if (rows_unreadable(*b.flags) || base == last || b.eos[s].x == kNone) {
        if (lane == 0) l.n_nodes[s] = 0;
        return;
    }
    const long long best = m.r_eos[s];
    for (uint32_t slot = base; slot <= last; ++slot) {  // the margin rule
        const uint2 me = b.ends_meta[slot];
        for (uint32_t e = me.x + (slot == base ? 1u : 0u) + lane; e < me.y; e += 32) {
            const long long ge = g.G[e];
            g.keep[e] = (ge != LLONG_MAX && m.R[e] + ge - best <= g.D) ? 0u : kNone;
        }
    }
    __syncwarp();
    if (lane == 0) walk_best(b, s, base, [&](uint32_t e, uint32_t) { g.keep[e] = 0; });  // the best path is always kept
    __syncwarp();
    uint32_t run = 0;
    for (uint32_t slot = base; slot <= last; ++slot) {  // kept indices in node order
        const uint2 me = b.ends_meta[slot];
        for (uint32_t e0 = me.x + (slot == base ? 1u : 0u); e0 < me.y; e0 += 32) {
            const uint32_t e = e0 + lane;
            const bool kept = e < me.y && g.keep[e] == 0;
            const uint32_t bal = __ballot_sync(kFull, kept);
            if (kept) g.keep[e] = run + __popc(bal & lanemask_lt());
            run += __popc(bal);
        }
    }
    if (lane == 0) l.n_nodes[s] = run;
}

// The records, links and (with l.node_prob) node marginals, after the scan of n_nodes gave node_off.  MARGIN = false:
// every node, numbered row_base[slot] + its place in the row.  MARGIN = true: the kept nodes only, numbered by g.keep,
// with `prev` remapped to the kept list (-2 for a predecessor that was not kept) and g.node_margin.
template <bool MARGIN>
__global__ void __launch_bounds__(256) k_lattice_write(Batch b, LatticeArgs l, MargArgs m, MarginArgs g) {
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (s >= b.n_sent || rows_unreadable(*b.flags)) return;
    const uint32_t base = b.slot_off[s], last = b.slot_off[s + 1] - 1;
    // an empty sentence has no nodes; one without a path keeps none
    if (base == last || (MARGIN && b.eos[s].x == kNone)) return;
    const unsigned long long n0 = l.node_off[s];
    const double a_eos = l.node_prob ? m.a_eos[s] : 0.0;
    const long long best = MARGIN ? m.r_eos[s] : 0;
    // the sentence-relative index of entry e of the row of `slot`, any row but the first (or kNone: not kept)
    auto node = [&](uint32_t e, uint32_t slot) { return MARGIN ? g.keep[e] : l.row_base[slot] + (e - b.ends_meta[slot].x); };
    for (uint32_t slot = base; slot <= last; ++slot) {
        const uint2 me = b.ends_meta[slot];
        const uint32_t skip_bos = slot == base ? 1u : 0u;
        const uint32_t rb = MARGIN ? 0u : l.row_base[slot];
        for (uint32_t e = me.x + skip_bos + lane; e < me.y; e += 32) {
            const uint32_t i = MARGIN ? g.keep[e] : rb + (e - me.x - skip_bos);
            if (MARGIN && i == kNone) continue;
            const uint4 c = b.ends_cold[e];  // {start_node slot, best prev entry, word_idx, min_cost}
            const unsigned long long k = n0 + i;
            write_node_record(b, l.nodes + k * 3, base, slot, c, c.w);
            const uint32_t p = c.x == base ? 0u : node(c.y, c.x);  // the first slot's row holds only BOS
            l.links[k] = make_int2(c.x == base ? -1 : (MARGIN && p == kNone) ? -2 : int32_t(p), 0);
            if (MARGIN) g.node_margin[k] = m.R[e] + g.G[e] - best;
            if (l.node_prob) {
                const double2 ab = m.ab[e];
                l.node_prob[k] = float(exp(ab.x + ab.y - a_eos));  // the expression of k_backtrack<true>
            }
        }
    }
    __syncwarp();
    if (lane == 0)  // never the BOS row
        walk_best(b, s, base, [&](uint32_t e, uint32_t end_node) { l.links[n0 + node(e, base + end_node)].y = int32_t(kNodeBest); });
}

// ---------------------------------------------------------------------------------------------
// Segmentation sampling (SampleArgs in kernels.cuh): one lane per (sentence, sample) walk from EOS back to BOS.
// ---------------------------------------------------------------------------------------------

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11) with its standard multipliers
// and Weyl key increments.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k.x += 0x9E3779B9u;
            k.y += 0xBB67AE85u;
        }
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    }
    return c;
}

// The uniform of draw step t of sample j of sentence i: 53 bits of the first two output words, in [0, 1).
__device__ __forceinline__ double sample_uniform(unsigned long long seed, uint32_t t, uint32_t j, uint32_t i) {
    const uint4 x = philox4x32_10(make_uint4(t, j, i, 0u), make_uint2(uint32_t(seed), uint32_t(seed >> 32)));
    return (double(x.x >> 5) * 67108864.0 + double(x.y >> 6)) * (1.0 / 9007199254740992.0);
}

// One walk: count (WRITE = false: its tokens and i32 total into cnt / total) or write (its records, from the end).
template <int CONN, bool WRITE>
__device__ __forceinline__ void sample_walk(const DictView& d, const Batch& b, const MargArgs& m, const SampleArgs& sa) {
    const unsigned long long w = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= (unsigned long long)b.n_sent * sa.n) return;
    const uint32_t sidx = uint32_t(w / sa.n), j = uint32_t(w % sa.n);
    const uint32_t s = b.order ? b.order[sidx] : sidx;
    const unsigned long long walk = (unsigned long long)s * sa.n + j;
    const bool sound = !rows_unreadable(*b.flags);
    const uint32_t base = sound ? b.slot_off[s] : 0u, last = sound ? b.slot_off[s + 1] - 1 : 0u;
    const uint4 eos = sound && base != last ? b.eos[s] : make_uint4(kNone, 0, 0, 0);
    if (eos.x == kNone) {  // an empty sentence, one without a path, or a batch that is re-run or refused
        if (!WRITE) {
            sa.cnt[walk] = 0;
            sa.total[walk] = 0;
        }
        return;
    }
    const uint32_t i = uint32_t(sa.sent_base + s);
    const double th = m.theta;
    uint32_t row = base + eos.y;  // the slot of the row the current node starts at
    uint32_t left = 0;            // EOS: BOS_EOS_CONNECTION_ID, no word cost
    int32_t wc = 0;
    long long r = m.r_eos[s];
    uint32_t tokens = 0, sum = 0;  // sum: the path's cost so far, wrapping like the tokenizer's i32
    unsigned long long at = 0;
    if (WRITE) {
        sum = uint32_t(sa.total[walk]);
        at = sa.off[walk] + sa.cnt[walk];
    }
    for (uint32_t t = 0; row != base; ++t) {
        const uint2 me = b.ends_meta[row];
        const uint32_t eo = me.x, K = me.y - me.x;
        const ConnRow<CONN> conn(d, left);
        double mx = -INFINITY;
        for (uint32_t k = 0; k < K; ++k) {
            const long long x = m.R[eo + k] + conn.cost(d, uint32_t(b.ends_hot[eo + k].y)) + wc;
            mx = fmax(mx, m.ab[eo + k].x - th * double(x - r));
        }
        double S = 0.0;
        for (uint32_t k = 0; k < K; ++k) {
            const long long x = m.R[eo + k] + conn.cost(d, uint32_t(b.ends_hot[eo + k].y)) + wc;
            S += exp(m.ab[eo + k].x - th * double(x - r) - mx);
        }
        const double target = sample_uniform(sa.seed, t, j, i) * S;
        double cum = 0.0;
        uint32_t pick = kNone, last_pos = 0;
        int32_t step = 0, step_last = 0;
        for (uint32_t k = 0; k < K; ++k) {
            const int32_t c = conn.cost(d, uint32_t(b.ends_hot[eo + k].y));
            const long long x = m.R[eo + k] + c + wc;
            const double wk = exp(m.ab[eo + k].x - th * double(x - r) - mx);
            cum += wk;
            const int32_t stp = int32_t(uint32_t(c) + uint32_t(wc));
            if (wk > 0.0) {
                last_pos = k;
                step_last = stp;
            }
            if (cum > target) {
                pick = k;
                step = stp;
                break;
            }
        }
        if (pick == kNone) {
            pick = last_pos;
            step = step_last;
        }
        const uint32_t e = eo + pick;
        if (WRITE) {  // the token's prefix cost = the path's cost through c minus the edge into c
            sum -= uint32_t(step);
            const uint4 c = b.ends_cold[e];
            write_node_record(b, sa.out + (--at) * 3, base, row, c, sum);
            row = c.x;
        } else {
            sum += uint32_t(step);
            row = b.ends_cold[e].x;
        }
        ++tokens;
        const uint32_t lw = m.lw[e];
        left = lw & 0xFFFFu;
        wc = int16_t(lw >> 16);
        r = m.R[e];
    }
    if (!WRITE) {  // the first token's edge from BOS (right id 0, cost 0)
        sum += uint32_t(ConnRow<CONN>(d, left).cost(d, 0u)) + uint32_t(wc);
        sa.cnt[walk] = tokens;
        sa.total[walk] = int32_t(sum);
    }
}

template <int CONN>
__global__ void __launch_bounds__(256) k_sample_count(DictView d, Batch b, MargArgs m, SampleArgs sa) {
    sample_walk<CONN, false>(d, b, m, sa);
}

template <int CONN>
__global__ void __launch_bounds__(256) k_sample_write(DictView d, Batch b, MargArgs m, SampleArgs sa) {
    sample_walk<CONN, true>(d, b, m, sa);
}

// ---------------------------------------------------------------------------------------------
// Posterior decoding (PosteriorArgs in kernels.cuh)
// ---------------------------------------------------------------------------------------------

// p of lattice entry e, as k_lattice_write publishes it
__device__ __forceinline__ float posterior_p(const MargArgs& m, uint32_t e, double a_eos) {
    const double2 ab = m.ab[e];
    return float(exp(ab.x + ab.y - a_eos));
}

// The edge into the node {left, wc} from entry e: conn(right(e), left) + wc, wrapping like the tokenizer's i32.
template <int CONN>
__device__ __forceinline__ uint32_t posterior_step(const DictView& d, const Batch& b, uint32_t e, uint32_t left, int32_t wc) {
    return uint32_t(ConnRow<CONN>(d, left).cost(d, uint32_t(b.ends_hot[e].y))) + uint32_t(wc);
}

template <int CONN>
__global__ void __launch_bounds__(256) k_posterior_sweep(DictView d, Batch b, MargArgs m, PosteriorArgs p) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t sidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (sidx >= b.n_sent) return;
    const uint32_t s = b.order ? b.order[sidx] : sidx;
    const bool sound = !rows_unreadable(*b.flags);
    const uint32_t base = sound ? b.slot_off[s] : 0u, last = sound ? b.slot_off[s + 1] - 1 : 0u;
    const uint4 eos = sound && base != last ? b.eos[s] : make_uint4(kNone, 0, 0, 0);
    if (eos.x == kNone) {  // an empty sentence, one without a path, or a batch that is re-run or refused
        if (lane == 0) {
            p.cnt[s] = 0;
            p.total[s] = 0;
            p.gain[s] = base == last ? 0.0 : -INFINITY;
        }
        return;
    }
    const double a_eos = m.a_eos[s], g1 = p.g1;
    const uint32_t slot_end = base + eos.y;
    if (lane == 0) p.V[base] = 0.0;  // BOS
    __syncwarp();
    for (uint32_t slot = base + 1; slot <= slot_end; ++slot) {
        const uint2 me = b.ends_meta[slot];
        double bx = -INFINITY;
        uint32_t be = kNone;
        for (uint32_t e = me.x + lane; e < me.y; e += 32) {  // a lane's entries in row order: keep the first maximum
            const double vs = p.V[b.ends_cold[e].x];
            if (vs == -INFINITY) continue;
            const double g = __dsub_rn(__dmul_rn(g1, double(posterior_p(m, e, a_eos))), 1.0);
            const double x = __dadd_rn(vs, g);
            if (x > bx) {
                bx = x;
                be = e;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {  // the largest x, then the lowest entry
            const double ox = __shfl_xor_sync(kFull, bx, o);
            const uint32_t oe = __shfl_xor_sync(kFull, be, o);
            if (ox > bx || (ox == bx && oe < be)) {
                bx = ox;
                be = oe;
            }
        }
        if (lane == 0) {
            p.V[slot] = bx;
            p.A[slot] = be;
        }
        __syncwarp();
    }
    if (lane != 0) return;
    p.gain[s] = p.V[slot_end];
    uint32_t row = slot_end, left = 0, tokens = 0, sum = 0;  // EOS: left id 0, no word cost
    int32_t wc = 0;
    while (row != base) {
        const uint32_t e = p.A[row];
        sum += posterior_step<CONN>(d, b, e, left, wc);
        ++tokens;
        const uint32_t lw = m.lw[e];
        left = lw & 0xFFFFu;
        wc = int16_t(lw >> 16);
        row = b.ends_cold[e].x;
    }
    sum += uint32_t(ConnRow<CONN>(d, left).cost(d, 0u)) + uint32_t(wc);  // the first token's edge from BOS
    p.cnt[s] = tokens;
    p.total[s] = int32_t(sum);
}

template <int CONN>
__global__ void __launch_bounds__(256) k_posterior_write(DictView d, Batch b, MargArgs m, PosteriorArgs p) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= b.n_sent || p.cnt[s] == 0) return;
    const uint32_t base = b.slot_off[s];
    const double a_eos = m.a_eos[s];
    uint32_t row = base + b.eos[s].y, left = 0, sum = uint32_t(p.total[s]);
    int32_t wc = 0;
    unsigned long long at = p.off[s] + p.cnt[s];
    while (row != base) {  // a token's prefix cost = the path's cost through its successor minus the edge between them
        const uint32_t e = p.A[row];
        sum -= posterior_step<CONN>(d, b, e, left, wc);
        const uint4 c = b.ends_cold[e];
        write_node_record(b, p.out + (--at) * 3, base, row, c, sum);
        p.prob[at] = posterior_p(m, e, a_eos);
        const uint32_t lw = m.lw[e];
        left = lw & 0xFFFFu;
        wc = int16_t(lw >> 16);
        row = c.x;
    }
}


// ---------------------------------------------------------------------------------------------
// Output stage: the text `tokenize` writes per sentence (tokenize/src/main.rs:83-127):
//   mecab : {surface}\t{feature}\n per token, then EOS\n
//   wakati: surfaces joined by one space, then \n
//   detail: {surface}\t{feature}\tlex_type={:?}\tleft_id={}\tright_id={}\tword_cost={}\ttotal_cost={}\n, then EOS\n
// One warp per sentence.  Pass 1 sizes every sentence, a scan over sentences places it, pass 2 places the tokens
// inside their sentence with a warp scan and copies bytes.  Both passes need only the tokens of their own sentence,
// so a chunk of a batch formats with chunk-local token offsets.
// ---------------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t dec_len(uint32_t v) {
    uint32_t n = 1;
    while (v >= 10) {
        v /= 10;
        ++n;
    }
    return n;
}
__device__ __forceinline__ uint32_t dec_len_signed(int32_t v) {
    return v < 0 ? 1 + dec_len(0u - uint32_t(v)) : dec_len(uint32_t(v));
}
__device__ __forceinline__ uint8_t* put_dec(uint8_t* p, uint32_t v) {
    const uint32_t n = dec_len(v);
    for (uint32_t i = n; i-- > 0;) {
        p[i] = uint8_t('0' + v % 10);
        v /= 10;
    }
    return p + n;
}
__device__ __forceinline__ uint8_t* put_dec_signed(uint8_t* p, int32_t v) {
    if (v < 0) {
        *p++ = '-';
        return put_dec(p, 0u - uint32_t(v));
    }
    return put_dec(p, uint32_t(v));
}
__device__ __forceinline__ uint8_t* put_str(uint8_t* p, const char* s) {
    while (*s) *p++ = uint8_t(*s++);
    return p;
}
__device__ __forceinline__ const char* lex_name(uint32_t lex) {  // LexType's Debug names (dictionary.rs:30-40)
    return lex == 0 ? "System" : lex == 1 ? "User" : "Unknown";
}
__device__ __forceinline__ uint32_t lex_name_len(uint32_t lex) { return lex == 0 ? 6 : lex == 1 ? 4 : 7; }

struct TokenText {
    uint32_t start_byte, surf_len, lex, feat_at, feat_len, word_id;
    int32_t total_cost;
};

__device__ __forceinline__ TokenText token_text(const DictView& d, const uint2* __restrict__ tokens, unsigned long long t) {
    const uint2 bytes = tokens[t * 3 + 1], wc = tokens[t * 3 + 2];
    TokenText x;
    x.start_byte = bytes.x;
    x.surf_len = bytes.y - bytes.x;
    x.lex = wc.x >> 30;
    x.word_id = wc.x & 0x3FFFFFFFu;
    x.total_cost = int32_t(wc.y);
    if (x.lex > 2) {  // not a LexType: treated as a word without feature
        x.lex = 2;
        x.word_id = 0x3FFFFFFFu;
    }
    x.feat_at = 0;
    x.feat_len = 0;
    if (x.word_id < d.n_words[x.lex]) {
        const uint32_t a = __ldg(d.feat_off[x.lex] + x.word_id), b = __ldg(d.feat_off[x.lex] + x.word_id + 1);
        x.feat_at = a;
        x.feat_len = b - a;
    }
    return x;
}

__device__ __forceinline__ uint32_t detail_tail_len(const DictView& d, const TokenText& x) {
    const uint2 pr = x.word_id < d.n_words[x.lex] ? __ldg(d.params[x.lex] + x.word_id) : make_uint2(0, 0);
    return 10 + lex_name_len(x.lex) + 9 + dec_len(pr.x & 0xFFFFu) + 10 + dec_len(pr.x >> 16) + 11 +
           dec_len_signed(int32_t(int16_t(pr.y & 0xFFFFu))) + 12 + dec_len_signed(x.total_cost);
}

// Bytes token t contributes to its sentence's text (separators included, the sentence terminator not).
__device__ __forceinline__ uint32_t token_text_len(const DictView& d, const TokenText& x, uint32_t mode, bool first) {
    if (mode == kOutWakati) return x.surf_len + (first ? 0u : 1u);
    if (mode == kOutMecab) return x.surf_len + 1 + x.feat_len + 1;
    return x.surf_len + 1 + x.feat_len + detail_tail_len(d, x) + 1;
}

// ---- kOutFormat: a format program (format.hpp) interpreted per token --------------------------------------------

// Words of the three lexicons numbered in one range (system, user, unknown): the index of the field table.
__device__ __forceinline__ uint32_t word_global(const DictView& d, uint32_t lex, uint32_t id) {
    return (lex >= 1 ? d.n_words[0] : 0u) + (lex >= 2 ? d.n_words[1] : 0u) + id;
}

// What a format program may print of token t (prev = token t - 1 of the sentence, or BOS: end byte 0, cost 0).
struct FmtTok {
    TokenText x;
    uint32_t end, prev_end;
    int32_t prev_total, word_cost;
    uint32_t ids;          // left | right << 16
    uint32_t keep, entry;  // field table: the fields printed, and the word's first entry
    uint32_t prob_micro;   // %pP: round(marginal * 1e6), in [0, 1e6]
    uint32_t best;         // %pb (lattice text): the node is on the best path
};

template <bool PROB = false, bool BEST = false>
__device__ __forceinline__ FmtTok fmt_tok(const DictView& d, const FormatArgs& f, const FormatProgram& P,
                                          unsigned long long t, unsigned long long t0, const int2* links = nullptr) {
    const uint32_t uses = P.uses;
    FmtTok v;
    v.x = token_text(d, f.tokens, t);
    v.end = v.x.start_byte + v.x.surf_len;
    v.prev_end = 0;
    v.prev_total = 0;
    if ((uses & kUsesPrev) && t > t0) {
        const uint2 pb = f.tokens[(t - 1) * 3 + 1], pc = f.tokens[(t - 1) * 3 + 2];
        v.prev_end = pb.y;
        v.prev_total = int32_t(pc.y);
    }
    const bool known = v.x.word_id < d.n_words[v.x.lex];
    v.ids = 0;
    v.word_cost = 0;
    if ((uses & kUsesParams) && known) {
        const uint2 pr = __ldg(d.params[v.x.lex] + v.x.word_id);
        v.ids = pr.x;
        v.word_cost = int32_t(int16_t(pr.y & 0xFFFFu));
    }
    v.keep = 0;
    v.entry = 0;
    if ((uses & kUsesFields) && known) {
        const uint32_t wg = word_global(d, v.x.lex, v.x.word_id);
        v.keep = __ldg(f.ft_keep + wg);
        v.entry = wg * P.n_fields;
    }
    v.prob_micro = 0;
    if constexpr (PROB) {
        if (uses & kUsesProb) {
            const double pm = rint(double(f.token_prob[t]) * 1e6);
            v.prob_micro = uint32_t(fmin(fmax(pm, 0.0), 1e6));
        }
    }
    if constexpr (BEST) v.best = (uses & kUsesBest) ? (uint32_t(links[t].y) & kNodeBest) : 0u;
    return v;
}

// The value of a numeric op (every op but literals, copies and fields).
__device__ __forceinline__ long long fmt_number(uint32_t kind, const FmtTok& v, uint32_t sent_len) {
    switch (kind) {
        case kOpWordCost: return v.word_cost;
        case kOpTotalCost: return v.x.total_cost;
        case kOpCostDiff: return int32_t(uint32_t(v.x.total_cost) - uint32_t(v.prev_total));
        case kOpConnCost: return int32_t(uint32_t(v.x.total_cost) - uint32_t(v.prev_total) - uint32_t(v.word_cost));
        case kOpStart: return v.x.start_byte;
        case kOpEnd: return v.end;
        case kOpSurfLen: return v.x.surf_len;
        case kOpSurfLenWs: return v.end - v.prev_end;
        case kOpLeftId: return v.ids & 0xFFFFu;
        case kOpRightId: return v.ids >> 16;
        case kOpStat: return v.x.lex == 2 ? 1 : 0;
        default: return sent_len;  // kOpSentLen
    }
}
__device__ __forceinline__ uint32_t num_len(long long x) { return x < 0 ? 1 + dec_len(uint32_t(-x)) : dec_len(uint32_t(x)); }

// Bytes the ops [a, b) of the program write for one token (or for BOS / EOS, with v unused).  PROB: the program may
// print %pP (a separate instantiation, so that the other formats keep their code).
template <bool PROB = false, bool BEST = false>
__device__ __forceinline__ unsigned long long fmt_len(const FormatProgram& P, uint32_t a, uint32_t b, const FormatArgs& f,
                                                      const FmtTok& v, uint32_t sent_len) {
    unsigned long long n = 0;
    for (uint32_t i = a; i < b; ++i) {
        const FormatOp o = P.ops[i];
        switch (o.kind) {
            case kOpLit: n += o.n; break;
            case kOpSurface: n += v.x.surf_len; break;
            case kOpSurfaceWs: n += v.end - v.prev_end; break;
            case kOpWs: n += v.x.start_byte - v.prev_end; break;
            case kOpFeature: n += v.x.feat_len; break;
            case kOpSentence: n += sent_len; break;
            case kOpFields: {
                bool first = true;
                for (uint32_t j = 0; j < o.n; ++j) {
                    const uint32_t k = P.slot[o.at + j];
                    if (!((v.keep >> k) & 1u)) continue;
                    n += (first ? 0u : 1u) + __ldg(f.ft_off + v.entry + k + 1) - __ldg(f.ft_off + v.entry + k);
                    first = false;
                }
                break;
            }
            default:
                if constexpr (PROB) {
                    if (o.kind == kOpProb) {
                        n += 8;  // d.dddddd
                        break;
                    }
                }
                if constexpr (BEST) {
                    if (o.kind == kOpBest) {
                        n += 1;  // '*' or ' '
                        break;
                    }
                }
                n += num_len(fmt_number(o.kind, v, sent_len));
        }
    }
    return n;
}

// The stage runs only on a batch whose tokens are sound: after an input error or an overflow the engine drops or
// re-runs the batch anyway, and its token records may then point anywhere.
__device__ __forceinline__ bool format_stands_down(const FormatArgs& f) {
    return *f.flags & (kFlagsStandDown | kFlagUtf8Error | kFlagPoolOverflow);
}

// kOutFormat: every block stages the program in (dynamic) shared memory; all its threads call this.
__device__ __forceinline__ const FormatProgram* stage_program(const FormatArgs& f, FormatProgram* s_prog) {
    if (f.mode != kOutFormat) return nullptr;
    const FormatProgram* g = f.prog;
    const uint32_t n_ops = g->n_ops, n_slots = g->n_slots, n_lit = g->n_lit;
    auto copy = [&](void* dst, const void* src, uint32_t bytes) {
        for (uint32_t i = threadIdx.x; i < (bytes + 3) / 4; i += blockDim.x)
            static_cast<uint32_t*>(dst)[i] = static_cast<const uint32_t*>(src)[i];
    };
    copy(s_prog, g, kFmtHeaderBytes);
    copy(s_prog->ops, g->ops, n_ops * uint32_t(sizeof(FormatOp)));
    copy(s_prog->slot, g->slot, n_slots);
    copy(s_prog->lit, g->lit, n_lit);
    __syncthreads();
    return s_prog;
}

// Pass 1 for sentence s (a warp per sentence): lane 0 stores its text length in sent_len[s].  PROG: f.mode is
// kOutFormat (a separate instantiation, so that the fixed modes keep their registers).  Sample text (n_samp > 1):
// s is the walk s' * n_samp + j, whose records are tok_off[s] .. tok_off[s + 1], rendered with sentence s' = s / n_samp.
template <bool PROG, bool PROB = false, bool BEST = false>
__device__ __forceinline__ void format_len_one(const DictView& d, const FormatArgs& f, const FormatProgram* P, uint32_t s,
                                               uint32_t lane, const int2* links = nullptr, uint32_t n_samp = 1) {
    const unsigned long long t0 = f.tok_off[s], t1 = f.tok_off[s + 1];
    unsigned long long len = 0;
    if constexpr (PROG) {
        const uint32_t si = s / n_samp;
        const uint32_t sl = uint32_t(f.byte_off[si + 1] - f.byte_off[si]);
        for (unsigned long long t = t0 + lane; t < t1; t += 32) {
            const FmtTok v = fmt_tok<PROB, BEST>(d, f, *P, t, t0, links);
            const uint32_t sec = v.x.lex == 2 ? kSecUnk : kSecNode;
            len += fmt_len<PROB, BEST>(*P, P->sec[sec][0], P->sec[sec][1], f, v, sl);
        }
        for (int k = 16; k > 0; k >>= 1) len += __shfl_xor_sync(kFull, len, k);
        if (lane == 0) {
            FmtTok none{};
            len += fmt_len<PROB, BEST>(*P, P->sec[kSecBos][0], P->sec[kSecBos][1], f, none, sl);
            f.sent_len[s] = len + fmt_len<PROB, BEST>(*P, P->sec[kSecEos][0], P->sec[kSecEos][1], f, none, sl);
        }
    } else {
        for (unsigned long long t = t0 + lane; t < t1; t += 32) len += token_text_len(d, token_text(d, f.tokens, t), f.mode, t == t0);
        for (int k = 16; k > 0; k >>= 1) len += __shfl_xor_sync(kFull, len, k);
        if (lane == 0) f.sent_len[s] = len + (f.mode == kOutWakati ? 1 : 4);  // "\n" or "EOS\n"
    }
}

template <bool PROG, bool PROB = false>
__global__ void __launch_bounds__(256) k_format_len(DictView d, FormatArgs f) {
    extern __shared__ uint4 s_dyn[];
    const FormatProgram* P = PROG ? stage_program(f, reinterpret_cast<FormatProgram*>(s_dyn)) : nullptr;
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (s >= f.n_sent || format_stands_down(f)) return;
    format_len_one<PROG, PROB>(d, f, P, s, lane);
}

__device__ __forceinline__ void warp_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t n, uint32_t lane) {
    for (uint32_t i = lane; i < n; i += 32) dst[i] = src[i];
}

// Writes the ops [a, b) at dst with the whole warp (every lane passes the same arguments); returns the end.
template <bool PROB = false, bool BEST = false>
__device__ __forceinline__ uint8_t* fmt_write(const DictView& d, const FormatProgram& P, uint32_t a, uint32_t b,
                                              const FormatArgs& f, const FmtTok& v, const uint8_t* __restrict__ sent,
                                              uint32_t sent_len, uint8_t* dst, uint32_t lane) {
    for (uint32_t i = a; i < b; ++i) {
        const FormatOp o = P.ops[i];
        switch (o.kind) {
            case kOpLit:
                warp_copy(dst, P.lit + o.at, o.n, lane);
                dst += o.n;
                break;
            case kOpSurface:
                warp_copy(dst, sent + v.x.start_byte, v.x.surf_len, lane);
                dst += v.x.surf_len;
                break;
            case kOpSurfaceWs:
                warp_copy(dst, sent + v.prev_end, v.end - v.prev_end, lane);
                dst += v.end - v.prev_end;
                break;
            case kOpWs:
                warp_copy(dst, sent + v.prev_end, v.x.start_byte - v.prev_end, lane);
                dst += v.x.start_byte - v.prev_end;
                break;
            case kOpFeature:
                if (v.x.feat_len) warp_copy(dst, d.feat[v.x.lex] + v.x.feat_at, v.x.feat_len, lane);
                dst += v.x.feat_len;
                break;
            case kOpSentence:
                warp_copy(dst, sent, sent_len, lane);
                dst += sent_len;
                break;
            case kOpFields: {
                bool first = true;
                for (uint32_t j = 0; j < o.n; ++j) {
                    const uint32_t k = P.slot[o.at + j];
                    if (!((v.keep >> k) & 1u)) continue;
                    if (!first) {
                        if (lane == 0) *dst = o.sep;
                        ++dst;
                    }
                    const uint32_t at = __ldg(f.ft_off + v.entry + k), n = __ldg(f.ft_off + v.entry + k + 1) - at;
                    warp_copy(dst, f.ft_bytes + at, n, lane);
                    dst += n;
                    first = false;
                }
                break;
            }
            default: {
                if constexpr (PROB) {
                    if (o.kind == kOpProb) {  // round(p * 1e6) as d.dddddd
                        if (lane == 0) {
                            dst[0] = uint8_t('0' + v.prob_micro / 1000000u);
                            dst[1] = '.';
                            uint32_t frac = v.prob_micro % 1000000u;
                            for (int k = 7; k >= 2; --k, frac /= 10) dst[k] = uint8_t('0' + frac % 10);
                        }
                        dst += 8;
                        break;
                    }
                }
                if constexpr (BEST) {
                    if (o.kind == kOpBest) {  // MeCab's %pb: '*' on the best path, ' ' elsewhere
                        if (lane == 0) *dst = v.best ? '*' : ' ';
                        dst += 1;
                        break;
                    }
                }
                const long long x = fmt_number(o.kind, v, sent_len);
                if (lane == 0) {
                    if (x < 0) {
                        *dst = '-';
                        put_dec(dst + 1, uint32_t(-x));
                    } else {
                        put_dec(dst, uint32_t(x));
                    }
                }
                dst += num_len(x);
            }
        }
    }
    return dst;
}

// The unquoted text of the fields of a feature string, split as the evaluate tool's parse_csv_row splits it
// (csv-core: a field that begins with '"' is quoted, "" inside it stands for '"', a ',' outside quotes ends the
// field): out(field, byte) for every byte of field text.  Returns the number of fields.
template <class Out>
__device__ __forceinline__ uint32_t csv_fields(const uint8_t* __restrict__ p, uint32_t n, Out out) {
    uint32_t field = 0;
    bool quoted = false, at_start = true;
    for (uint32_t i = 0; i < n; ++i) {
        const uint8_t c = p[i];
        if (quoted) {
            if (c != '"') {
                out(field, c);
            } else if (i + 1 < n && p[i + 1] == '"') {
                out(field, c);
                ++i;
            } else {
                quoted = false;
            }
        } else if (c == '"' && at_start) {
            quoted = true;
        } else if (c == ',') {
            ++field;
            at_start = true;
            continue;
        } else {
            out(field, c);
        }
        at_start = false;
    }
    return field + 1;
}

__device__ __forceinline__ void word_feature(const DictView& d, uint32_t wg, const uint8_t*& p, uint32_t& n) {
    uint32_t lex = 0;
    while (lex < 2 && wg >= d.n_words[lex]) wg -= d.n_words[lex++];
    const uint32_t a = d.feat_off[lex][wg];
    p = d.feat[lex] + a;
    n = d.feat_off[lex][wg + 1] - a;
}

// Field table, pass 1: a thread per word stores which referenced fields it prints and their lengths.
__global__ void __launch_bounds__(256) k_field_table_len(DictView d, FieldTableArgs a) {
    const uint32_t wg = blockIdx.x * blockDim.x + threadIdx.x;
    if (wg >= a.n_words) return;
    const uint8_t* p;
    uint32_t n;
    word_feature(d, wg, p, n);
    uint32_t len[kFmtMaxFields];
    for (uint32_t k = 0; k < kFmtMaxFields; ++k) len[k] = 0;
    uint32_t seen = 0, star = 0;
    const uint32_t nf = csv_fields(p, n, [&](uint32_t field, uint8_t c) {
        const uint32_t k = field <= kFmtMaxFieldIndex ? a.slot_of[field] : 0xFFu;
        if (k == 0xFFu) return;
        if (!((seen >> k) & 1u)) {
            seen |= 1u << k;
            if (c == '*') star |= 1u << k;
        }
        ++len[k];
    });
    uint32_t keep = 0;
    for (uint32_t k = 0; k < a.n_fields; ++k) {
        const bool kept = a.fields[k] < nf && !((star >> k) & 1u);  // a field past the last one counts as '*'
        keep |= uint32_t(kept) << k;
        a.lens[size_t(wg) * a.n_fields + k] = kept ? len[k] : 0u;
    }
    a.keep[wg] = keep;
}

// Field table, pass 2: the same split writes the printed fields at their offsets.
__global__ void __launch_bounds__(256) k_field_table_write(DictView d, FieldTableArgs a) {
    const uint32_t wg = blockIdx.x * blockDim.x + threadIdx.x;
    if (wg >= a.n_words) return;
    const uint32_t keep = a.keep[wg];
    if (!keep) return;
    const uint8_t* p;
    uint32_t n;
    word_feature(d, wg, p, n);
    uint32_t at[kFmtMaxFields];
    for (uint32_t k = 0; k < a.n_fields; ++k) at[k] = a.off[size_t(wg) * a.n_fields + k];
    csv_fields(p, n, [&](uint32_t field, uint8_t c) {
        const uint32_t k = field <= kFmtMaxFieldIndex ? a.slot_of[field] : 0xFFu;
        if (k != 0xFFu && ((keep >> k) & 1u)) a.bytes[at[k]++] = c;
    });
}

// Pass 2 for sentence s (a warp per sentence): its text at text_off[s], which must fit in text_cap.  n_samp > 1: s
// is a walk, as in format_len_one.
template <bool PROG, bool PROB = false, bool BEST = false>
__device__ __forceinline__ void format_write_one(const DictView& d, const FormatArgs& f, const FormatProgram* P, uint32_t s,
                                                 uint32_t lane, const int2* links = nullptr, uint32_t n_samp = 1) {
    const unsigned long long t0 = f.tok_off[s], t1 = f.tok_off[s + 1];
    const uint32_t si = s / n_samp;
    const uint8_t* __restrict__ sent = f.utf8 + f.byte_off[si];
    unsigned long long base = f.text_off[s];  // where the next group of 32 tokens starts
    const bool prog = PROG;
    const uint32_t sl = prog ? uint32_t(f.byte_off[si + 1] - f.byte_off[si]) : 0u;
    if (prog) {
        const FmtTok none{};
        base = fmt_write<PROB, BEST>(d, *P, P->sec[kSecBos][0], P->sec[kSecBos][1], f, none, sent, sl, f.text + base, lane) - f.text;
    }
    for (unsigned long long c = t0; c < t1; c += 32) {
        // lane i stages token c + i; the copies below take one token at a time with all 32 lanes
        const uint32_t cnt = uint32_t(min(32ull, t1 - c));
        TokenText mine = {0, 0, 0, 0, 0, 0, 0};
        unsigned long long len = 0;
        if (lane < cnt && prog) {
            const FmtTok v = fmt_tok<PROB, BEST>(d, f, *P, c + lane, t0, links);
            const uint32_t sec = v.x.lex == 2 ? kSecUnk : kSecNode;
            len = fmt_len<PROB, BEST>(*P, P->sec[sec][0], P->sec[sec][1], f, v, sl);
        } else if (lane < cnt) {
            mine = token_text(d, f.tokens, c + lane);
            len = token_text_len(d, mine, f.mode, c + lane == t0);
        }
        unsigned long long incl = len;  // inclusive warp scan of the group's lengths
        for (int k = 1; k < 32; k <<= 1) {
            const unsigned long long v = __shfl_up_sync(kFull, incl, k);
            if (lane >= uint32_t(k)) incl += v;
        }
        const unsigned long long at = base + incl - len;
        base += __shfl_sync(kFull, incl, 31);
        for (uint32_t j = 0; j < cnt; ++j) {
            if (prog) {  // every lane loads token c + j again: one broadcast load per record
                const FmtTok v = fmt_tok<PROB, BEST>(d, f, *P, c + j, t0, links);
                const uint32_t sec = v.x.lex == 2 ? kSecUnk : kSecNode;
                fmt_write<PROB, BEST>(d, *P, P->sec[sec][0], P->sec[sec][1], f, v, sent, sl, f.text + __shfl_sync(kFull, at, j), lane);
                continue;
            }
            TokenText x;
            x.start_byte = __shfl_sync(kFull, mine.start_byte, j);
            x.surf_len = __shfl_sync(kFull, mine.surf_len, j);
            x.lex = __shfl_sync(kFull, mine.lex, j);
            x.feat_at = __shfl_sync(kFull, mine.feat_at, j);
            x.feat_len = __shfl_sync(kFull, mine.feat_len, j);
            x.word_id = __shfl_sync(kFull, mine.word_id, j);
            x.total_cost = __shfl_sync(kFull, mine.total_cost, j);
            uint8_t* dst = f.text + __shfl_sync(kFull, at, j);
            if (f.mode == kOutWakati) {
                if (c + j != t0) {
                    if (lane == 0) *dst = ' ';
                    ++dst;
                }
                warp_copy(dst, sent + x.start_byte, x.surf_len, lane);
                continue;
            }
            warp_copy(dst, sent + x.start_byte, x.surf_len, lane);
            dst += x.surf_len;
            if (lane == 0) *dst = '\t';
            ++dst;
            if (x.feat_len) warp_copy(dst, d.feat[x.lex] + x.feat_at, x.feat_len, lane);
            dst += x.feat_len;
            if (lane == 0) {
                if (f.mode == kOutDetail) {
                    const uint2 pr = x.word_id < d.n_words[x.lex] ? __ldg(d.params[x.lex] + x.word_id) : make_uint2(0, 0);
                    dst = put_str(dst, "\tlex_type=");
                    dst = put_str(dst, lex_name(x.lex));
                    dst = put_str(dst, "\tleft_id=");
                    dst = put_dec(dst, pr.x & 0xFFFFu);
                    dst = put_str(dst, "\tright_id=");
                    dst = put_dec(dst, pr.x >> 16);
                    dst = put_str(dst, "\tword_cost=");
                    dst = put_dec_signed(dst, int32_t(int16_t(pr.y & 0xFFFFu)));
                    dst = put_str(dst, "\ttotal_cost=");
                    dst = put_dec_signed(dst, x.total_cost);
                }
                *dst = '\n';
            }
        }
    }
    if (prog) {
        const FmtTok none{};
        fmt_write<PROB, BEST>(d, *P, P->sec[kSecEos][0], P->sec[kSecEos][1], f, none, sent, sl, f.text + base, lane);
    } else if (lane == 0) {
        uint8_t* dst = f.text + base;
        if (f.mode != kOutWakati) dst = put_str(dst, "EOS");
        *dst = '\n';
    }
}

template <bool PROG, bool PROB = false>
__global__ void __launch_bounds__(256) k_format_write(DictView d, FormatArgs f) {
    extern __shared__ uint4 s_dyn[];
    const FormatProgram* P = PROG ? stage_program(f, reinterpret_cast<FormatProgram*>(s_dyn)) : nullptr;
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (s >= f.n_sent || format_stands_down(f)) return;
    const unsigned long long total = f.text_off[f.n_sent];
    if (s == 0 && lane == 0) {
        *f.text_total = total;
        if (total > f.text_cap) atomicOr(f.flags, kFlagTextOverflow);
    }
    if (total > f.text_cap) return;  // every warp sees the same total: nothing is written
    format_write_one<PROG, PROB>(d, f, P, s, lane);
}

// Lattice text with %pb: the nodes' links give the best-path flag (separate kernels, so that the instantiations
// above keep their code).
template <bool PROB>
__global__ void __launch_bounds__(256) k_format_len_best(DictView d, FormatArgs f, const int2* links) {
    extern __shared__ uint4 s_dyn[];
    const FormatProgram* P = stage_program(f, reinterpret_cast<FormatProgram*>(s_dyn));
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (s >= f.n_sent || format_stands_down(f)) return;
    format_len_one<true, PROB, true>(d, f, P, s, lane, links);
}

template <bool PROB>
__global__ void __launch_bounds__(256) k_format_write_best(DictView d, FormatArgs f, const int2* links) {
    extern __shared__ uint4 s_dyn[];
    const FormatProgram* P = stage_program(f, reinterpret_cast<FormatProgram*>(s_dyn));
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (s >= f.n_sent || format_stands_down(f)) return;
    const unsigned long long total = f.text_off[f.n_sent];
    if (s == 0 && lane == 0) {
        *f.text_total = total;
        if (total > f.text_cap) atomicOr(f.flags, kFlagTextOverflow);
    }
    if (total > f.text_cap) return;
    format_write_one<true, PROB, true>(d, f, P, s, lane, links);
}

// Sample text: a warp per walk w = s * n + j of the samples (f.tok_off / f.tokens are the sample offsets and records;
// f.sent_len and f.text_off have an entry per walk), rendered with the text of sentence s (separate kernels, so that
// the instantiations above keep their code).  The write pass also stores each sentence's text offset, that of its
// first walk, in sent_text_off[0 .. n_sent].
__device__ __forceinline__ unsigned long long walk_of_warp() {
    return ((unsigned long long)(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
}

template <bool PROG>
__global__ void __launch_bounds__(256) k_format_len_samples(DictView d, FormatArgs f, uint32_t n) {
    extern __shared__ uint4 s_dyn[];
    const FormatProgram* P = PROG ? stage_program(f, reinterpret_cast<FormatProgram*>(s_dyn)) : nullptr;
    const unsigned long long w = walk_of_warp();
    const uint32_t lane = threadIdx.x & 31;
    if (w >= (unsigned long long)(f.n_sent) * n || format_stands_down(f)) return;
    format_len_one<PROG>(d, f, P, uint32_t(w), lane, nullptr, n);
}

template <bool PROG>
__global__ void __launch_bounds__(256) k_format_write_samples(DictView d, FormatArgs f, uint32_t n,
                                                              unsigned long long* sent_text_off) {
    extern __shared__ uint4 s_dyn[];
    const FormatProgram* P = PROG ? stage_program(f, reinterpret_cast<FormatProgram*>(s_dyn)) : nullptr;
    const unsigned long long w = walk_of_warp(), walks = (unsigned long long)(f.n_sent) * n;
    const uint32_t lane = threadIdx.x & 31;
    if (w >= walks || format_stands_down(f)) return;
    const unsigned long long total = f.text_off[walks];
    if (lane == 0 && w % n == 0) sent_text_off[w / n] = f.text_off[w];
    if (w == 0 && lane == 0) {
        sent_text_off[f.n_sent] = total;
        *f.text_total = total;
        if (total > f.text_cap) atomicOr(f.flags, kFlagTextOverflow);
    }
    if (total > f.text_cap) return;
    format_write_one<PROG>(d, f, P, uint32_t(w), lane, nullptr, n);
}

// ---------------------------------------------------------------------------------------------
// k_small_batch: the whole pipeline above for a small host batch in ONE thread block, so that a call costs one
// launch.  The device-wide scans between the kernels become block scans between __syncthreads(); each stage calls
// the per-sentence / per-position bodies of its kernel:
//   count_chars_one -> scan -> decode_one -> start_word / count_candidates (count, then fill) -> scan -> viterbi_sweep
//   (k_viterbi's sweep, 32 lanes per sentence, no pruning) -> backtrack_count_one -> scan -> backtrack_write_one
//   [-> format_len_one -> scan -> format_write_one].
// A warp takes one sentence at a time, a thread one start position.  The batch flags live in shared memory and
// go out with the totals in SmallBatchOut.  A candidate pool or text larger than the buffers the engine gave sets
// kFlagPoolOverflow / kFlagTextOverflow and ends the kernel: the engine then runs the batch on the usual route.
// ---------------------------------------------------------------------------------------------

constexpr uint32_t kSmallThreads = 1024;

// Exclusive prefix of v over the block's threads in thread order; *total = the block's sum.  Every thread calls it.
__device__ __forceinline__ unsigned long long block_exclusive(unsigned long long v, unsigned long long& total,
                                                              unsigned long long* s_warp /* [32] */) {
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    unsigned long long incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(kFull, incl, o);
        if (lane >= uint32_t(o)) incl += t;
    }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    unsigned long long before = 0, sum = 0;
    for (uint32_t i = 0; i < nw; ++i) {
        const unsigned long long t = s_warp[i];
        if (i < wid) before += t;
        sum += t;
    }
    __syncthreads();  // s_warp is free again
    total = sum;
    return before + incl - v;
}

// out(i, exclusive prefix of get(0..i)) for i in [0, n]; out(n) = the total, which is returned.  Every thread calls
// it; everything written is visible to the whole block on return.
template <class Get, class Put>
__device__ __forceinline__ unsigned long long block_scan(uint32_t n, Get get, Put put, unsigned long long* s_warp) {
    unsigned long long carry = 0;
    for (uint32_t base = 0; base < n; base += blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        unsigned long long tile;
        const unsigned long long ex = block_exclusive(i < n ? (unsigned long long)get(i) : 0ull, tile, s_warp);
        if (i < n) put(i, carry + ex);
        carry += tile;
    }
    if (threadIdx.x == 0) put(n, carry);
    __syncthreads();
    return carry;
}

template <int CONN, bool BND>
__global__ void __launch_bounds__(kSmallThreads, 1) k_small_batch(DictView d, Batch b, FormatArgs f, SmallBatchOut* out) {
    __shared__ uint32_t s_flags;
    __shared__ unsigned long long s_warp[32];
    extern __shared__ uint4 s_dyn[];
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
    const uint32_t n = b.n_sent;
    if (tid == 0) s_flags = 0;
    __syncthreads();
    b.flags = &s_flags;
    f.flags = &s_flags;
    uint32_t total_slots = 0;
    unsigned long long n_tokens = 0, text_bytes = 0;
    // K1a, then the slot scan.  `s_flags` is read right after a barrier and written again only after the next one,
    // so every decision taken on it below is the same in all threads.
    for (uint32_t s = wid; s < n; s += nw) count_chars_one(b, s, lane);
    __syncthreads();
    bool ok = !(s_flags & (kFlagsStandDown | kFlagUtf8Error));  // the engine reports the error; nothing else to do
    if (ok) {
        total_slots = uint32_t(block_scan(
            n, [&](uint32_t i) { return b.n_slots[i]; }, [&](uint32_t i, unsigned long long v) { b.slot_off[i] = uint32_t(v); },
            s_warp));
        for (uint32_t s = wid; s < n; s += nw) {  // K1b
            decode_one(d, b, s, lane);
            __syncwarp();
            if (BND) {  // required boundaries: a bad list only raises its flag, the engine reports it
                mark_bounds_one(b, s, lane);
                __syncwarp();
            }
        }
        __syncthreads();
        // K2: a thread per start position; the segment pool is handed out in position order by a scan per block-wide
        // tile, and the candidates are counted the same way (the lattice rows must hold them)
        unsigned long long carry = 0, seg_carry = 0;
        for (uint32_t base = 0; base < total_slots; base += blockDim.x) {
            const uint32_t slot = base + tid;
            const uint32_t g0 = slot < total_slots ? b.groupable[slot] : 0;
            const StartWord w = start_word<BND>(d, b, slot, g0);
            SegOut so{nullptr, 0, 0, 0, slot, nullptr};
            const uint32_t cnt = w.active ? count_candidates<BND>(d, b, w, so) : 0;
            const uint32_t nseg = so.n;
            unsigned long long tile;
            const unsigned long long cptr = carry + block_exclusive(cnt, tile, s_warp);
            carry += tile;
            const unsigned long long ptr = seg_carry + block_exclusive(nseg, tile, s_warp);
            seg_carry += tile;
            if (cptr + cnt > b.cand_cap || ptr + nseg > b.seg_cap) {
                atomicOr(&s_flags, kFlagPoolOverflow);
            } else if (g0 != 0) {
                store_info(b, slot, uint32_t(ptr), cnt, w);
                if (cnt) {
                    SegOut out{b.seg + ptr, 1, nseg, 0, slot, b.ends_cnt};
                    count_candidates<BND>(d, b, w, out);
                }
            }
        }
        __syncthreads();
        ok = !(s_flags & kFlagPoolOverflow);
    }
    if (ok) {
        // lattice rows: ends_meta = {row offset, next free entry} from the node counts per end position
        block_scan(
            total_slots, [&](uint32_t i) { return b.ends_cnt[i]; },
            [&](uint32_t i, unsigned long long v) { b.ends_meta[i] = make_uint2(uint32_t(v), uint32_t(v)); }, s_warp);
        for (uint32_t s = wid; s < n; s += nw) viterbi_sweep<32, false, CONN>(d, b, nullptr, s);  // K3
        __syncthreads();
        for (uint32_t s = tid; s < n; s += blockDim.x) backtrack_count_one(b, s);  // K4a
        __syncthreads();
        n_tokens = block_scan(
            n, [&](uint32_t i) { return b.n_tok[i]; }, [&](uint32_t i, unsigned long long v) { b.tok_off[i] = v; }, s_warp);
        for (uint32_t s = wid; s < n; s += nw) backtrack_write_one(b, s, lane);  // K4b
        if (f.mode != kOutNone) {  // output stage
            __syncthreads();
            const FormatProgram* P = stage_program(f, reinterpret_cast<FormatProgram*>(s_dyn));
            for (uint32_t s = wid; s < n; s += nw) {
                if (P)
                    format_len_one<true>(d, f, P, s, lane);
                else
                    format_len_one<false>(d, f, P, s, lane);
            }
            __syncthreads();
            text_bytes = block_scan(
                n, [&](uint32_t i) { return f.sent_len[i]; }, [&](uint32_t i, unsigned long long v) { f.text_off[i] = v; },
                s_warp);
            if (text_bytes > f.text_cap) {
                if (tid == 0) atomicOr(&s_flags, kFlagTextOverflow);
            } else {
                for (uint32_t s = wid; s < n; s += nw) {
                    if (P)
                        format_write_one<true>(d, f, P, s, lane);
                    else
                        format_write_one<false>(d, f, P, s, lane);
                }
            }
        }
    }
    __syncthreads();
    if (tid == 0) {
        out->flags = s_flags;
        out->total_slots = total_slots;
        out->n_tokens = n_tokens;
        out->text_bytes = text_bytes;
    }
}

}  // namespace

// f(conn) with conn = std::integral_constant<int, CONN> of the dictionary's connector kind, for the kernels that are
// instantiated per connector (0 Matrix, 1 Raw, 2 Dual).
template <class F>
static void with_connector(const DictView& d, F f) {
    if (d.connector_kind == 1)
        f(std::integral_constant<int, 1>{});
    else if (d.connector_kind == 2)
        f(std::integral_constant<int, 2>{});
    else
        f(std::integral_constant<int, 0>{});
}

void launch_small_batch(const DictView& d, const Batch& b, const FormatArgs& f, SmallBatchOut* out, cudaStream_t st) {
    const size_t smem = f.mode == kOutFormat ? sizeof(FormatProgram) : 0;
    with_connector(d, [&](auto conn) {
        if (b.bnd_dist)
            k_small_batch<conn, true><<<1, kSmallThreads, smem, st>>>(d, b, f, out);
        else
            k_small_batch<conn, false><<<1, kSmallThreads, smem, st>>>(d, b, f, out);
    });
}

void launch_format_len(const DictView& d, const FormatArgs& f, cudaStream_t st, const int2* links) {
    if (!f.n_sent) return;
    if (links && f.mode == kOutFormat)
        f.token_prob ? k_format_len_best<true><<<(f.n_sent + 7) / 8, 256, sizeof(FormatProgram), st>>>(d, f, links)
                     : k_format_len_best<false><<<(f.n_sent + 7) / 8, 256, sizeof(FormatProgram), st>>>(d, f, links);
    else if (f.mode == kOutFormat)
        f.token_prob ? k_format_len<true, true><<<(f.n_sent + 7) / 8, 256, sizeof(FormatProgram), st>>>(d, f)
                     : k_format_len<true><<<(f.n_sent + 7) / 8, 256, sizeof(FormatProgram), st>>>(d, f);
    else
        k_format_len<false><<<(f.n_sent + 7) / 8, 256, 0, st>>>(d, f);
}

void launch_format_write(const DictView& d, const FormatArgs& f, cudaStream_t st, const int2* links) {
    if (!f.n_sent) return;
    if (links && f.mode == kOutFormat)
        f.token_prob ? k_format_write_best<true><<<(f.n_sent + 7) / 8, 256, sizeof(FormatProgram), st>>>(d, f, links)
                     : k_format_write_best<false><<<(f.n_sent + 7) / 8, 256, sizeof(FormatProgram), st>>>(d, f, links);
    else if (f.mode == kOutFormat)
        f.token_prob ? k_format_write<true, true><<<(f.n_sent + 7) / 8, 256, sizeof(FormatProgram), st>>>(d, f)
                     : k_format_write<true><<<(f.n_sent + 7) / 8, 256, sizeof(FormatProgram), st>>>(d, f);
    else
        k_format_write<false><<<(f.n_sent + 7) / 8, 256, 0, st>>>(d, f);
}

void launch_format_len_samples(const DictView& d, const FormatArgs& f, uint32_t n, cudaStream_t st) {
    const unsigned long long blocks = ((unsigned long long)(f.n_sent) * n + 7) / 8;
    if (!blocks) return;
    if (f.mode == kOutFormat)
        k_format_len_samples<true><<<unsigned(blocks), 256, sizeof(FormatProgram), st>>>(d, f, n);
    else
        k_format_len_samples<false><<<unsigned(blocks), 256, 0, st>>>(d, f, n);
}

void launch_format_write_samples(const DictView& d, const FormatArgs& f, uint32_t n, unsigned long long* sent_text_off,
                                 cudaStream_t st) {
    const unsigned long long blocks = ((unsigned long long)(f.n_sent) * n + 7) / 8;
    if (!blocks) return;
    if (f.mode == kOutFormat)
        k_format_write_samples<true><<<unsigned(blocks), 256, sizeof(FormatProgram), st>>>(d, f, n, sent_text_off);
    else
        k_format_write_samples<false><<<unsigned(blocks), 256, 0, st>>>(d, f, n, sent_text_off);
}

void launch_field_table_len(const DictView& d, const FieldTableArgs& a, cudaStream_t st) {
    if (a.n_words) k_field_table_len<<<(a.n_words + 255) / 256, 256, 0, st>>>(d, a);
}

void launch_field_table_write(const DictView& d, const FieldTableArgs& a, cudaStream_t st) {
    if (a.n_words) k_field_table_write<<<(a.n_words + 255) / 256, 256, 0, st>>>(d, a);
}

void launch_front(const DictView& d, const Batch& b, const TileScan& ts, cudaStream_t st) {
    if (!b.n_sent) return;
    k_front<<<scan_tiles(b.n_sent, kFrontTile), 256, 0, st>>>(d, b, ts.state, ts.ticket);
}

void launch_mark_bounds(const Batch& b, cudaStream_t st) {
    if (!b.n_sent) return;
    uint32_t blocks = (b.n_sent + 8 * VBT_SENT_PER_WARP - 1) / (8 * VBT_SENT_PER_WARP);
    k_mark_bounds<<<blocks, 256, 0, st>>>(b);
}

void launch_mark_spans(const Batch& b, const SpanArgs& sp, cudaStream_t st) {
    if (!b.n_sent) return;
    uint32_t blocks = (b.n_sent + 8 * VBT_SENT_PER_WARP - 1) / (8 * VBT_SENT_PER_WARP);
    k_mark_spans<<<blocks, 256, 0, st>>>(b, sp);
}

void launch_candidates(const DictView& d, const Batch& b, uint32_t max_slots, cudaStream_t st, const SpanArgs* sp) {
    if (!max_slots) return;
    uint32_t blocks = (max_slots + 255) / 256;
    if (sp)
        k_candidates_spans<<<blocks, 256, 0, st>>>(d, b, *sp);
    else if (b.bnd_dist)
        k_candidates<true><<<blocks, 256, 0, st>>>(d, b);
    else
        k_candidates<false><<<blocks, 256, 0, st>>>(d, b);
}

void launch_candidate_stats(const DictView& d, const Batch& b, uint32_t max_slots, uint4* stats, cudaStream_t st) {
    if (!max_slots) return;
    uint32_t blocks = (max_slots + 255) / 256;
    k_candidate_stats<<<blocks, 256, 0, st>>>(d, b, stats);
}

template <int G>
static int launch_viterbi_g(const DictView& d, const Batch& b, const uint4* stats, int kernel, cudaStream_t st,
                            uint32_t* route) {
    const uint32_t per_block = 4 * (32 / G);  // 4 warps per block
    const uint32_t blocks = (b.n_sent + per_block - 1) / per_block;
    const bool counted = stats || b.lid_count;
    // k_viterbi2's matrix lookups assume a matrix inside one 4 GiB window (the engine arranges that when it can)
    if (!counted && kernel != 0 && (d.connector_kind != 0 || d.matrix_window)) {
        const bool space = d.space_mask != 0;
        const uint32_t per_block2 = VBT_K3V2_WARPS * (32 / G);
        const uint32_t blocks2 = (b.n_sent + per_block2 - 1) / per_block2;
#define VBT_LAUNCH_V2(CONN, PRUNE, TWIN)                                        \
    do {                                                                        \
        if (space)                                                              \
            k_viterbi2<G, CONN, PRUNE, true, TWIN><<<blocks2, 32 * VBT_K3V2_WARPS, 0, st>>>(d, b);  \
        else                                                                    \
            k_viterbi2<G, CONN, PRUNE, false, TWIN><<<blocks2, 32 * VBT_K3V2_WARPS, 0, st>>>(d, b); \
    } while (0)
        if (d.connector_kind == 1) {
            VBT_LAUNCH_V2(1, false, false);
        } else if (d.connector_kind == 2) {
            VBT_LAUNCH_V2(2, false, false);
        } else if (kernel == 1) {  // the pruned kernel and its twin for batches with very long sentences
            VBT_LAUNCH_V2(0, true, true);
            VBT_LAUNCH_V2(0, false, true);
        } else {
            VBT_LAUNCH_V2(0, false, false);
        }
#undef VBT_LAUNCH_V2
        const bool pruned = d.connector_kind == 0 && kernel == 1;
        *route = pruned ? kRouteV2PrunedOrTwin : kRouteV2Unpruned;
        return pruned ? 2 : 1;
    }
    *route = kRouteV1;
    if (d.connector_kind == 1) {
        if (counted)
            k_viterbi<G, true, 1><<<blocks, 128, 0, st>>>(d, b, stats);
        else
            k_viterbi<G, false, 1><<<blocks, 128, 0, st>>>(d, b, stats);
    } else if (d.connector_kind == 2) {
        if (counted)
            k_viterbi<G, true, 2><<<blocks, 128, 0, st>>>(d, b, stats);
        else
            k_viterbi<G, false, 2><<<blocks, 128, 0, st>>>(d, b, stats);
    } else if (counted) {
        k_viterbi<G, true, 0><<<blocks, 128, 0, st>>>(d, b, stats);
    } else {
        k_viterbi<G, false, 0><<<blocks, 128, 0, st>>>(d, b, stats);
    }
    return 1;
}

int launch_viterbi(const DictView& d, const Batch& b, const uint4* stats, int lanes_per_sentence, int kernel,
                   cudaStream_t st, uint32_t* route) {
    *route = kRouteNone;
    if (!b.n_sent) return 0;
    switch (lanes_per_sentence) {
        case 4: return launch_viterbi_g<4>(d, b, stats, kernel, st, route);
        case 8: return launch_viterbi_g<8>(d, b, stats, kernel, st, route);
        case 32: return launch_viterbi_g<32>(d, b, stats, kernel, st, route);
        default: return launch_viterbi_g<16>(d, b, stats, kernel, st, route);
    }
}


template <bool MARG>
static void launch_backtrack_marg(const Batch& b, const MargArgs& m, const TileScan& ts, cudaStream_t st) {
    int dev = 0, sms = 0;  // on failure sms stays 0 and the large tile is taken
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    unsigned long long* state = ts.state + scan_tiles(b.n_sent, kFrontTile);
    if (b.n_sent >= uint64_t(kBackTile) * uint32_t(sms))
        k_backtrack<MARG, kBackTile><<<scan_tiles(b.n_sent, kBackTile), 256, 0, st>>>(b, m, state, ts.ticket + 1);
    else
        k_backtrack<MARG, kBackTileSmall><<<scan_tiles(b.n_sent, kBackTileSmall), 256, 0, st>>>(b, m, state, ts.ticket + 1);
}

void launch_backtrack(const Batch& b, const MargArgs* m, const TileScan& ts, cudaStream_t st) {
    if (!b.n_sent) return;
    if (m)
        launch_backtrack_marg<true>(b, *m, ts, st);
    else
        launch_backtrack_marg<false>(b, MargArgs{}, ts, st);
}

void launch_marginals(const DictView& d, const Batch& b, const MargArgs& m, FwdKind fwd, BwdKind bwd,
                      const UncertaintyArgs& u, const MarginArgs* g, cudaStream_t st) {
    if (!b.n_sent) return;
    const uint32_t blocks = (b.n_sent + 7) / 8;  // a warp per sentence
    with_connector(d, [&](auto conn) {
        if (fwd == kFwdLseLw)
            k_marg_forward<conn, true><<<blocks, 256, 0, st>>>(d, b, m);
        else if (fwd == kFwdLse)
            k_marg_forward<conn><<<blocks, 256, 0, st>>>(d, b, m);
        else if (fwd == kFwdR)
            k_marg_forward<conn, false, false><<<blocks, 256, 0, st>>>(d, b, m);
        if (bwd == kBwdUnc)
            k_marg_backward<conn, true><<<blocks, 256, 0, st>>>(d, b, m, u);
        else if (bwd == kBwdPlain)
            k_marg_backward<conn><<<blocks, 256, 0, st>>>(d, b, m, UncertaintyArgs{});
    });
    if (u.boundary_prob) k_boundary_probs<<<blocks, 256, 0, st>>>(b, m, u);
    if (g) with_connector(d, [&](auto conn) { k_margin_backward<conn><<<blocks, 256, 0, st>>>(d, b, m, *g); });
}

void launch_lattice_count(const Batch& b, const LatticeArgs& l, const MargArgs& m, const MarginArgs* g, cudaStream_t st) {
    if (!b.n_sent) return;
    const uint32_t blocks = (b.n_sent + 7) / 8;  // a warp per sentence
    if (g)
        k_lattice_count_margin<<<blocks, 256, 0, st>>>(b, l, m, *g);
    else
        k_lattice_count<<<blocks, 256, 0, st>>>(b, l);
}

void launch_lattice_write(const Batch& b, const LatticeArgs& l, const MargArgs& m, const MarginArgs* g, cudaStream_t st) {
    if (!b.n_sent) return;
    const uint32_t blocks = (b.n_sent + 7) / 8;
    if (g)
        k_lattice_write<true><<<blocks, 256, 0, st>>>(b, l, m, *g);
    else
        k_lattice_write<false><<<blocks, 256, 0, st>>>(b, l, m, MarginArgs{});
}

void launch_sample_count(const DictView& d, const Batch& b, const MargArgs& m, const SampleArgs& s, cudaStream_t st) {
    const unsigned long long walks = (unsigned long long)b.n_sent * s.n;
    if (!walks) return;
    const uint32_t blocks = uint32_t((walks + 255) / 256);  // a lane per walk
    with_connector(d, [&](auto conn) { k_sample_count<conn><<<blocks, 256, 0, st>>>(d, b, m, s); });
}

void launch_sample_write(const DictView& d, const Batch& b, const MargArgs& m, const SampleArgs& s, cudaStream_t st) {
    const unsigned long long walks = (unsigned long long)b.n_sent * s.n;
    if (!walks) return;
    const uint32_t blocks = uint32_t((walks + 255) / 256);
    with_connector(d, [&](auto conn) { k_sample_write<conn><<<blocks, 256, 0, st>>>(d, b, m, s); });
}

void launch_posterior_sweep(const DictView& d, const Batch& b, const MargArgs& m, const PosteriorArgs& p, cudaStream_t st) {
    if (!b.n_sent) return;
    const uint32_t blocks = (b.n_sent + 7) / 8;  // a warp per sentence
    with_connector(d, [&](auto conn) { k_posterior_sweep<conn><<<blocks, 256, 0, st>>>(d, b, m, p); });
}

void launch_posterior_write(const DictView& d, const Batch& b, const MargArgs& m, const PosteriorArgs& p, cudaStream_t st) {
    if (!b.n_sent) return;
    const uint32_t blocks = (b.n_sent + 255) / 256;  // a thread per sentence
    with_connector(d, [&](auto conn) { k_posterior_write<conn><<<blocks, 256, 0, st>>>(d, b, m, p); });
}

}  // namespace vbt
