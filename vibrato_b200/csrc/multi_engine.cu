// One tokenizer over several GPUs of one node (SURVEY.md §8(e); the reference has no counterpart — a vibrato
// Worker is a single CPU thread, worker.rs:13-31 — so the contract is BASELINE.json's north_star: "split the
// batch with one NCCL broadcast of the dictionary and a gather of token spans over NVLink").
//
//   * The dictionary image is uploaded ONCE (to the first device) and broadcast to the others with
//     ncclBroadcast; NCCL is bound at run time (dlopen of libnccl.so.2) so that the single-GPU library keeps no
//     link-time dependency on it.  Where NCCL cannot be loaded the same bytes travel by cudaMemcpyPeerAsync
//     (still NVLink / NVSwitch, still one PCIe upload).
//   * A batch is cut into contiguous shards of about equal BYTES (sentences are independent units; work is
//     proportional to characters), one per device; every device runs the ordinary single-device engine on its
//     shard from its own host thread (pinned to the CPUs of the GPU's NUMA node), so H2D copies, kernels and
//     D2H copies of different devices overlap and use their own PCIe links.
//   * Host results: once every shard's token count is known the shards' token records are copied straight into
//     ONE pinned result at their final positions (no host-side merge pass); token offsets are made global on
//     the device before they leave it.  The output stage ("output_mode") formats each shard's text on its device
//     and places it the same way.  The result is indistinguishable from a single-device one.
//   * Device-resident batches (vbt_tokenize_batch_device): the input sits on the first device, shards reach the
//     other devices by peer copies, and the token records come back to the first device with grouped
//     ncclSend / ncclRecv (the "gather of token spans over NVLink"; peer copies without NCCL).
#include "engine.hpp"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>  // types and enums only: every entry point is resolved with dlsym
#include <pthread.h>
#include <sched.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <thread>

namespace vbt {

namespace {

void cuda_check(cudaError_t e, const char* what) {
    if (e != cudaSuccess) throw Error(kCuda, std::string(what) + ": " + cudaGetErrorString(e));
}
#define CK(x) cuda_check((x), #x)

// ---- NCCL, bound at run time ---------------------------------------------------------------------
struct Nccl {
    void* so = nullptr;
    ncclResult_t (*GetVersion)(int*) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    int version = 0;

    static Nccl* get() {  // nullptr when the library (or one of its symbols) is missing
        static Nccl inst;
        static bool tried = false;
        if (!tried) {
            tried = true;
            const char* off = std::getenv("VBT_NO_NCCL");
            if (off && off[0] == '1') return nullptr;
            inst.so = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
            if (inst.so) {
                bool ok = true;
                auto sym = [&](const char* n) {
                    void* p = dlsym(inst.so, n);
                    ok = ok && p;
                    return p;
                };
                inst.GetVersion = reinterpret_cast<decltype(inst.GetVersion)>(sym("ncclGetVersion"));
                inst.GetErrorString = reinterpret_cast<decltype(inst.GetErrorString)>(sym("ncclGetErrorString"));
                inst.CommInitAll = reinterpret_cast<decltype(inst.CommInitAll)>(sym("ncclCommInitAll"));
                inst.CommDestroy = reinterpret_cast<decltype(inst.CommDestroy)>(sym("ncclCommDestroy"));
                inst.Broadcast = reinterpret_cast<decltype(inst.Broadcast)>(sym("ncclBroadcast"));
                inst.Send = reinterpret_cast<decltype(inst.Send)>(sym("ncclSend"));
                inst.Recv = reinterpret_cast<decltype(inst.Recv)>(sym("ncclRecv"));
                inst.GroupStart = reinterpret_cast<decltype(inst.GroupStart)>(sym("ncclGroupStart"));
                inst.GroupEnd = reinterpret_cast<decltype(inst.GroupEnd)>(sym("ncclGroupEnd"));
                if (!ok) {
                    dlclose(inst.so);
                    inst.so = nullptr;
                } else {
                    inst.GetVersion(&inst.version);
                }
            }
        }
        return inst.so ? &inst : nullptr;
    }
    void check(ncclResult_t r, const char* what) const {
        if (r != ncclSuccess) throw Error(kCuda, std::string(what) + ": " + GetErrorString(r));
    }
};
#define NK(x) nccl_->check((x), #x)

// ---- CPU affinity: the cores of the NUMA node a GPU hangs off ---------------------------------------
std::vector<int> parse_cpulist(const std::string& s) {
    std::vector<int> out;
    std::stringstream ss(s);
    std::string part;
    while (std::getline(ss, part, ',')) {
        int a = 0, b = 0;
        if (std::sscanf(part.c_str(), "%d-%d", &a, &b) == 2) {
            for (int c = a; c <= b; ++c) out.push_back(c);
        } else if (std::sscanf(part.c_str(), "%d", &a) == 1) {
            out.push_back(a);
        }
    }
    return out;
}

std::vector<int> numa_cpus_of_device(int device) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) return {};
    for (char* p = bus; *p; ++p) *p = char(std::tolower(*p));
    std::ifstream f(std::string("/sys/bus/pci/devices/") + bus + "/numa_node");
    int node = -1;
    if (!(f >> node) || node < 0) return {};
    std::ifstream g("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist");
    std::string list;
    if (!std::getline(g, list)) return {};
    return parse_cpulist(list);
}

void pin_this_thread(const std::vector<int>& cpus) {
    if (cpus.empty()) return;
    cpu_set_t allowed, want;
    CPU_ZERO(&want);
    if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return;
    int n = 0;
    for (int c : cpus)
        if (c < CPU_SETSIZE && CPU_ISSET(c, &allowed)) {
            CPU_SET(c, &want);
            ++n;
        }
    if (n) pthread_setaffinity_np(pthread_self(), sizeof want, &want);  // never widens the process's own mask
}

class MultiEngine final : public Engine {
   public:
    MultiEngine(const std::vector<int>& devices, const uint8_t* host_blob, uint64_t n_bytes, bool ignore_space,
                uint64_t max_grouping_len)
        : dev_(devices) {
        const int n = int(dev_.size());
        int count = 0;
        if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0)
            throw Error(kNoDevice, "no CUDA device available: the tokenizer has no CPU fallback");
        // A device listed more than once runs one shard per entry (an engine with its own streams and image copy):
        // the sharded path on one GPU, not a faster one.  NCCL refuses a repeated device, so peer copies serve then.
        bool distinct = true;
        for (int i = 0; i < n; ++i) {
            if (dev_[i] < 0 || dev_[i] >= count) throw Error(kInvalidArgument, "device ordinal out of range");
            for (int j = 0; j < i; ++j) distinct = distinct && dev_[j] != dev_[i];
        }
        nccl_ = distinct ? Nccl::get() : nullptr;
        stream_.resize(n);
        image_.resize(n, nullptr);
        cpus_.resize(n);
        for (int i = 0; i < n; ++i) {
            CK(cudaSetDevice(dev_[i]));
            CK(cudaStreamCreateWithFlags(&stream_[i], cudaStreamNonBlocking));
            CK(cudaMalloc(&image_[i], n_bytes));
            cpus_[i] = numa_cpus_of_device(dev_[i]);
            for (int j = 0; j < n; ++j) {  // peer access for the device-resident route (NVLink / NVSwitch)
                if (dev_[i] == dev_[j]) continue;
                int can = 0;
                cudaDeviceCanAccessPeer(&can, dev_[i], dev_[j]);
                if (can) {
                    cudaError_t e = cudaDeviceEnablePeerAccess(dev_[j], 0);
                    if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
                }
            }
        }
        // one PCIe upload, then the image goes from device to device
        CK(cudaSetDevice(dev_[0]));
        CK(cudaMemcpyAsync(image_[0], host_blob, n_bytes, cudaMemcpyHostToDevice, stream_[0]));
        CK(cudaStreamSynchronize(stream_[0]));
        if (n > 1) {
            if (nccl_) {
                comm_.resize(n);
                NK(nccl_->CommInitAll(comm_.data(), n, dev_.data()));
                NK(nccl_->GroupStart());
                for (int i = 0; i < n; ++i) {
                    CK(cudaSetDevice(dev_[i]));
                    NK(nccl_->Broadcast(image_[i], image_[i], n_bytes, ncclUint8, 0, comm_[i], stream_[i]));
                }
                NK(nccl_->GroupEnd());
                transport_ = "nccl " + std::to_string(nccl_->version);
            } else {
                for (int i = 1; i < n; ++i)
                    CK(cudaMemcpyPeerAsync(image_[i], dev_[i], image_[0], dev_[0], n_bytes, stream_[i]));
                transport_ = "cudaMemcpyPeer";
            }
            for (int i = 0; i < n; ++i) {
                CK(cudaSetDevice(dev_[i]));
                CK(cudaStreamSynchronize(stream_[i]));
            }
        } else {
            transport_ = "single device";
        }
        for (int i = 0; i < n; ++i) {
            eng_.push_back(Engine::create(dev_[i], nullptr, reinterpret_cast<uint64_t>(image_[i]), n_bytes, ignore_space,
                                          max_grouping_len));
            if (n > 1) eng_.back()->set_option("chunk_sentences", 0);  // a shard runs as one piece: overlap comes from the devices
        }
        std::memset(stage_ms_, 0, sizeof stage_ms_);
        std::memset(counters_, 0, sizeof counters_);
    }

    ~MultiEngine() override {
        eng_.clear();
        for (size_t i = 0; i < dev_.size(); ++i) {
            cudaSetDevice(dev_[i]);
            if (nccl_ && i < comm_.size() && comm_[i]) nccl_->CommDestroy(comm_[i]);
            cudaFree(image_[i]);
            cudaStreamDestroy(stream_[i]);
        }
        pinned_free(h_off_);
        pinned_free(h_bnd_off_);
        pinned_free(h_bnd_);
        pinned_free(h_span_off_);
        pinned_free(h_span_);
        cudaSetDevice(dev_[0]);
        for (DevBuf& b : gather_) b.release();
    }

    // ---- host batches --------------------------------------------------------------------------------
    HostResult* run_host(const char* utf8, const uint64_t* byte_off, uint64_t n_sent, const Bounds* bnd) override {
        const int n = int(dev_.size());
        reruns_ = Reruns{};
        if (n == 1) {  // nothing to split: the device's own chunked, overlapped host pipeline
            HostResult* r = eng_[0]->run_host(utf8, byte_off, n_sent, bnd);
            collect_stats();
            return r;
        }
        check_samples(n_sent);
        // offsets whose last lies below their first are a batch too large on one device (check_size), and so in the
        // shard whose window then wraps; the others are checked here, before the split
        if (n_sent && byte_off[n_sent] >= byte_off[0]) check_offsets(byte_off, n_sent, ~0ull);
        const std::vector<uint64_t> cut = split_by_bytes(byte_off, n_sent, n);
        const Outputs out = outputs();
        std::vector<Totals> count(n);
        run_on_all([&](int i) {
            const Bounds sb = shard_bounds(bnd, cut[i]);  // the draws of sentence k are those of the whole batch
            count[i] = eng_[i]->run_shard(utf8, byte_off + cut[i], cut[i + 1] - cut[i], -1, cut[i], out.text, bnd ? &sb : nullptr);
        });
        // every shard's outputs are copied straight to their final positions; the last shard, even when it is empty,
        // also delivers the closing offsets
        const std::vector<Totals> base = prefix_sums(count);
        HostResult* r = pool_.acquire(out, n_sent, base[n]);
        run_on_all([&](int i) { eng_[i]->fetch_shard(r, cut[i], base[i], i == n - 1); });
        collect_stats();
        return r;
    }
    void release(HostResult* r) override {
        if (!r) return;
        if (dev_.size() == 1)
            eng_[0]->release(r);
        else
            pool_.release(r);
    }

    // ---- device-resident batches: input on the first device, results gathered back to it ------------------
    void run_device(uint64_t d_utf8, uint64_t d_byte_off, uint64_t n_sent, uint64_t n_bytes, const Bounds* bnd) override {
        const int n = int(dev_.size());
        reruns_ = Reruns{};
        if (n == 1) {
            eng_[0]->run_device(d_utf8, d_byte_off, n_sent, n_bytes, bnd);
            collect_stats();
            return;
        }
        last_ = DeviceOutputs{};
        check_samples(n_sent);
        CK(cudaSetDevice(dev_[0]));
        // the split needs the offsets on the host (pinned staging buffer, one copy); they are checked there, before
        // the shards size their copies of the input from them
        if ((n_sent + 1) * 8 > h_off_cap_) {
            pinned_free(h_off_);
            h_off_cap_ = size_t(double((n_sent + 1) * 8) * 1.25) + 64;
            h_off_ = static_cast<uint64_t*>(pinned_alloc(h_off_cap_));
        }
        CK(cudaMemcpyAsync(h_off_, reinterpret_cast<const void*>(d_byte_off), (n_sent + 1) * 8, cudaMemcpyDeviceToHost, stream_[0]));
        CK(cudaStreamSynchronize(stream_[0]));
        check_offsets(h_off_, n_sent, n_bytes);
        // boundary lists: to the host as well, and from there to every shard like those of a host batch (they are
        // validated on the devices)
        Bounds hb;
        if (bnd) {
            hb.spans = bnd->spans;  // the patterns are host memory already
            if (bnd->off) {
                grow_pinned(h_bnd_off_, h_bnd_off_cap_, (n_sent + 1) * 8);
                grow_pinned(h_bnd_, h_bnd_cap_, bnd->n * 4 + 4);
                CK(cudaMemcpyAsync(h_bnd_off_, bnd->off, (n_sent + 1) * 8, cudaMemcpyDeviceToHost, stream_[0]));
                if (bnd->n) CK(cudaMemcpyAsync(h_bnd_, bnd->bnd, bnd->n * 4, cudaMemcpyDeviceToHost, stream_[0]));
                hb.off = static_cast<const uint64_t*>(h_bnd_off_);
                hb.bnd = static_cast<const uint32_t*>(h_bnd_);
                hb.n = bnd->n;
            }
            if (bnd->spans.off) {
                grow_pinned(h_span_off_, h_span_off_cap_, (n_sent + 1) * 8);
                grow_pinned(h_span_, h_span_cap_, bnd->spans.n * 12 + 12);
                CK(cudaMemcpyAsync(h_span_off_, bnd->spans.off, (n_sent + 1) * 8, cudaMemcpyDeviceToHost, stream_[0]));
                if (bnd->spans.n)
                    CK(cudaMemcpyAsync(h_span_, bnd->spans.rec, bnd->spans.n * 12, cudaMemcpyDeviceToHost, stream_[0]));
                hb.spans.off = static_cast<const uint64_t*>(h_span_off_);
                hb.spans.rec = static_cast<const uint32_t*>(h_span_);
            }
            CK(cudaStreamSynchronize(stream_[0]));
        }
        const std::vector<uint64_t> cut = split_by_bytes(h_off_, n_sent, n);
        std::vector<Totals> count(n);
        run_on_all([&](int i) {
            const Bounds sb = shard_bounds(bnd ? &hb : nullptr, cut[i]);
            count[i] = eng_[i]->run_shard(reinterpret_cast<const char*>(d_utf8), h_off_ + cut[i], cut[i + 1] - cut[i], dev_[0],
                                          cut[i], false, bnd ? &sb : nullptr);  // no text, like the single-device entry point
        });
        const std::vector<Totals> base = prefix_sums(count);
        run_on_all([&](int i) { eng_[i]->rebase_shard(base[i]); });
        // gather on the first device: every array of every shard at its final position
        Outputs out = outputs();
        out.text = false;
        CK(cudaSetDevice(dev_[0]));
        for (int a = 0; a < kNumArrays; ++a)
            if (out.has(a)) gather_[a].ensure(out.bytes(a, n_sent, base[n], true) + out.elem_bytes(a), 1.25);
        // the pieces of shard i: {destination on the first device, source on device i, bytes}
        struct Piece {
            void* dst;
            const void* src;
            uint64_t bytes;
        };
        auto pieces = [&](int i) {
            const uint64_t* src = eng_[i]->last_device().addr;
            std::vector<Piece> v;
            for (int a = 0; a < kNumArrays; ++a) {
                const uint64_t bytes = out.has(a) ? out.bytes(a, cut[i + 1] - cut[i], count[i], i == n - 1) : 0;
                if (bytes)
                    v.push_back({gather_[a].as<uint8_t>() + out.at(a, cut[i], base[i]), reinterpret_cast<const void*>(src[a]), bytes});
            }
            return v;
        };
        for (const Piece& p : pieces(0))  // shard 0 is already on the first device
            CK(cudaMemcpyAsync(p.dst, p.src, p.bytes, cudaMemcpyDeviceToDevice, stream_[0]));
        if (n > 1 && nccl_) {
            NK(nccl_->GroupStart());
            for (int i = 1; i < n; ++i) {
                const std::vector<Piece> v = pieces(i);
                CK(cudaSetDevice(dev_[i]));
                for (const Piece& p : v) NK(nccl_->Send(p.src, p.bytes, ncclUint8, 0, comm_[i], stream_[i]));
                CK(cudaSetDevice(dev_[0]));
                for (const Piece& p : v) NK(nccl_->Recv(p.dst, p.bytes, ncclUint8, i, comm_[0], stream_[0]));
            }
            NK(nccl_->GroupEnd());
        } else {
            for (int i = 1; i < n; ++i)
                for (const Piece& p : pieces(i)) CK(cudaMemcpyPeerAsync(p.dst, dev_[0], p.src, dev_[i], p.bytes, stream_[0]));
        }
        for (int i = 0; i < n; ++i) {
            CK(cudaSetDevice(dev_[i]));
            CK(cudaStreamSynchronize(stream_[i]));
        }
        collect_stats();
        last_.made = out;
        last_.total = base[n];
        for (int a = 0; a < kNumArrays; ++a) last_.addr[a] = out.has(a) ? reinterpret_cast<uint64_t>(gather_[a].p) : 0;
    }
    const DeviceOutputs& last_device() const override { return dev_.size() == 1 ? eng_[0]->last_device() : last_; }

    // ---- everything else is forwarded ------------------------------------------------------------------
    void set_counting(bool on) override {
        for (auto& e : eng_) e->set_counting(on);
    }
    void set_option(const std::string& name, long long value) override {
        if (name == "chunk_sentences") return;  // shards are not chunked (see the constructor)
        for (auto& e : eng_) e->set_option(name, value);
        if (name == "sample_base") sample_base_ = uint64_t(value);
    }
    void set_format(const FormatProgram* p) override {
        try {
            for (auto& e : eng_) e->set_format(p);  // each device builds its own field table
        } catch (...) {
            for (auto& e : eng_) e->set_format(nullptr);
            throw;
        }
    }
    Outputs outputs() const override { return eng_[0]->outputs(); }
    void set_marginals(double theta) override {
        for (auto& e : eng_) e->set_marginals(theta);
    }
    double marginals() const override { return eng_[0]->marginals(); }
    void set_sampling(uint32_t n, double theta, uint64_t seed) override {
        for (auto& e : eng_) e->set_sampling(n, theta, seed);  // the first refuses what all would
    }
    uint32_t sampling() const override { return eng_[0]->sampling(); }
    void set_posterior(bool on, double gamma) override {
        for (auto& e : eng_) e->set_posterior(on, gamma);  // the first refuses what all would
    }
    bool posterior() const override { return eng_[0]->posterior(); }
    int lattice() const override { return eng_[0]->lattice(); }
    void set_stream(uint64_t stream) override {
        if (stream) throw Error(kUnsupported, "a multi-device tokenizer runs on its own streams");
    }
    const float* stage_ms() const override { return stage_ms_; }
    uint64_t launch_count() const override { return launches_; }
    const uint64_t* counters() const override { return counters_; }
    void connid_counts(uint64_t* lid, uint64_t* rid, uint32_t* num_left, uint32_t* num_right) override {
        uint32_t nl = 0, nr = 0;
        eng_[0]->connid_counts(nullptr, nullptr, &nl, &nr);
        if (num_left) *num_left = nl;
        if (num_right) *num_right = nr;
        if (!lid || !rid) return;
        std::vector<uint64_t> l(nl), r(nr);
        std::fill(lid, lid + nl, 0);
        std::fill(rid, rid + nr, 0);
        for (auto& e : eng_) {
            e->connid_counts(l.data(), r.data(), nullptr, nullptr);
            for (uint32_t i = 0; i < nl; ++i) lid[i] += l[i];
            for (uint32_t i = 0; i < nr; ++i) rid[i] += r[i];
        }
    }
    Totals run_shard(const char*, const uint64_t*, uint64_t, int, uint64_t, bool, const Bounds*) override {
        throw Error(kInternal, "not a shard engine");
    }
    void rebase_shard(const Totals&) override { throw Error(kInternal, "not a shard engine"); }
    void fetch_shard(HostResult*, uint64_t, const Totals&, bool) override { throw Error(kInternal, "not a shard engine"); }
    int device() const override { return dev_[0]; }
    uint32_t token_bytes() const override { return eng_[0]->token_bytes(); }
    std::string describe() const override {
        std::string s = "{\"devices\": [";
        for (size_t i = 0; i < dev_.size(); ++i) s += (i ? ", " : "") + std::to_string(dev_[i]);
        s += "], \"dictionary_transport\": \"" + transport_ + "\", \"token_gather\": \"" +
             std::string(dev_.size() > 1 ? (nccl_ ? "ncclSend/ncclRecv" : "cudaMemcpyPeer") : "none") + "\", \"numa_pinned\": [";
        for (size_t i = 0; i < dev_.size(); ++i) s += (i ? ", " : "") + std::string(cpus_[i].empty() ? "false" : "true");
        return s + "], " + reruns_json(reruns_) + "}";
    }
    Reruns last_reruns() const override { return reruns_; }

   private:
    // Contiguous shards of about equal bytes: cut[i] = first sentence of shard i, cut[n] = n_sent.
    static std::vector<uint64_t> split_by_bytes(const uint64_t* off, uint64_t n_sent, int n) {
        std::vector<uint64_t> cut(size_t(n) + 1, n_sent);
        cut[0] = 0;
        const uint64_t first = n_sent ? off[0] : 0, total = n_sent ? off[n_sent] - first : 0;
        for (int i = 1; i < n; ++i) {
            const uint64_t target = first + total / uint64_t(n) * uint64_t(i);
            const uint64_t* p = std::lower_bound(off, off + n_sent + 1, target);
            cut[i] = std::max<uint64_t>(cut[i - 1], std::min<uint64_t>(uint64_t(p - off), n_sent));
        }
        return cut;
    }

    // What k_count_chars refuses on one device: a sentence that ends before it starts or beyond `end` bytes.  A shard
    // cut from such offsets would copy a wrapped window or bytes past the caller's buffer.
    static void check_offsets(const uint64_t* off, uint64_t n_sent, uint64_t end) {
        for (uint64_t i = 0; i < n_sent; ++i)
            if (off[i + 1] < off[i] || off[i + 1] > end) throw Error(kInvalidArgument, kBadOffsetsMsg);
    }

    // The sample offsets of a whole batch are indexed in 32 bits (every shard checks its own part too).
    void check_samples(uint64_t n_sent) const {
        if (n_sent * sampling() >= 0xFFFFFFFFull)
            throw Error(kInvalidArgument, "sampling: n_sent * n must stay below 2^32: split the batch or draw fewer samples");
        if (sample_base_ + n_sent > 0x100000000ull)
            throw Error(kInvalidArgument, "sampling: sample_base + n_sent exceeds 2^32, the range of the draws' sentence index");
    }

    static void grow_pinned(void*& p, size_t& cap, size_t bytes) {
        if (bytes <= cap) return;
        pinned_free(p);
        cap = size_t(double(bytes) * 1.25) + 64;
        p = pinned_alloc(cap);
    }

    // The boundary lists of the shard that starts at sentence `first` (host memory): its slice of the offsets.
    static Bounds shard_bounds(const Bounds* bnd, uint64_t first) {
        if (!bnd) return Bounds{};
        Bounds sb = *bnd;
        if (sb.off) sb.off += first;
        if (sb.spans.off) sb.spans.off += first;
        return sb;
    }

    // One host thread per device (the calling thread takes the first): each call blocks on its own device.  Of the
    // shards that failed, the error one device would report for the whole batch wins: any other error before the
    // input errors, those in their order (kInputErrors), then the first shard.
    template <typename F>
    void run_on_all(F&& f) {
        const int n = int(dev_.size());
        std::vector<std::string> err(n);
        std::vector<Status> st(n, kOk);
        auto body = [&](int i) {
            try {
                f(i);
            } catch (const Error& e) {
                st[i] = e.code;
                err[i] = e.what();
            } catch (const std::exception& e) {
                st[i] = kInternal;
                err[i] = e.what();
            }
        };
        std::vector<std::thread> th;
        for (int i = 1; i < n; ++i)
            th.emplace_back([&, i] {
                pin_this_thread(cpus_[i]);
                body(i);
            });
        body(0);
        for (auto& t : th) t.join();
        auto rank = [&](int i) {
            for (int k = 0; k < kNumInputErrors; ++k)
                if (err[i] == kInputErrors[k].msg) return k + 1;
            return 0;
        };
        int worst = -1;
        for (int i = 0; i < n; ++i)
            if (st[i] != kOk && (worst < 0 || rank(i) < rank(worst))) worst = i;
        if (worst >= 0) throw Error(st[worst], err[worst]);
    }

    void collect_stats() {
        std::memset(stage_ms_, 0, sizeof stage_ms_);
        std::memset(counters_, 0, sizeof counters_);
        launches_ = 0;
        for (auto& e : eng_) {
            const Reruns r = e->last_reruns();  // the shards' attempts add up
            for (int k = 0; k < kNumReruns; ++k) reruns_[k] += r[k];
            const float* s = e->stage_ms();
            for (int i = 0; i < kNumStages; ++i) stage_ms_[i] = std::max(stage_ms_[i], s[i]);  // devices run side by side
            const uint64_t* c = e->counters();
            for (int i = 0; i < 10; ++i) counters_[i] += c[i];
            launches_ += e->launch_count();
        }
    }

    // base[i][g] = the records of group g in the shards before shard i (base[n] = all of them).
    static std::vector<Totals> prefix_sums(const std::vector<Totals>& count) {
        std::vector<Totals> base(count.size() + 1, Totals{});
        for (size_t i = 0; i < count.size(); ++i)
            for (int g = 0; g < kNumGroups; ++g) base[i + 1][g] = base[i][g] + count[i][g];
        return base;
    }

    std::vector<int> dev_;
    Nccl* nccl_ = nullptr;
    std::vector<ncclComm_t> comm_;
    std::vector<cudaStream_t> stream_;
    std::vector<void*> image_;
    std::vector<std::vector<int>> cpus_;
    std::vector<std::unique_ptr<Engine>> eng_;
    std::string transport_;
    ResultPool pool_;
    uint64_t* h_off_ = nullptr;  // pinned
    size_t h_off_cap_ = 0;
    void* h_bnd_off_ = nullptr;  // pinned: the boundary lists of a device-resident batch, cut into shards on the host
    void* h_bnd_ = nullptr;
    size_t h_bnd_off_cap_ = 0, h_bnd_cap_ = 0;
    void* h_span_off_ = nullptr;  // pinned: the span lists of a device-resident batch, likewise
    void* h_span_ = nullptr;
    size_t h_span_off_cap_ = 0, h_span_cap_ = 0;
    DevBuf gather_[kNumArrays];  // the outputs of a gathered device-resident batch, on the first device
    DeviceOutputs last_;         // what the last device-resident call gathered there (last_device)
    uint64_t sample_base_ = 0;  // option "sample_base" (every engine adds it to its shard's first sentence)
    float stage_ms_[kNumStages];
    uint64_t counters_[10];
    uint64_t launches_ = 0;
    Reruns reruns_{};  // the attempts the last call re-ran over all its shards (describe())
};

}  // namespace

std::unique_ptr<Engine> Engine::create_multi(const std::vector<int>& devices, const uint8_t* host_blob, uint64_t n_bytes,
                                             bool ignore_space, uint64_t max_grouping_len) {
    if (devices.empty()) throw Error(kInvalidArgument, "no device given");
    return std::unique_ptr<Engine>(new MultiEngine(devices, host_blob, n_bytes, ignore_space, max_grouping_len));
}

void pin_thread_to_device_numa_node(int device) { pin_this_thread(numa_cpus_of_device(device)); }

}  // namespace vbt
