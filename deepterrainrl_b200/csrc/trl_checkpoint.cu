// deepterrainrl_b200 -- checkpoints of a handle and its trainers (include/terrainrl_b200.h: trl_checkpoint_save,
// trl_create_from_checkpoint).  A handle restored from a checkpoint in another process answers every later call, bit for bit, as the
// handle that saved it would have; DESIGN.md §11 lists what a checkpoint holds and what it leaves out.
//
// File (little-endian, fixed layout): "TRLCKPT1", u32 version, u32 section count, one FileSection record per section, then the
// sections' bytes in table order.  Sections of kind 0 are read before the handle is built (the scene pack, the sizes, the slots'
// contents, the trainers' parameters, the caller's blob); sections of kind 1 are the state poured into the built handle and trainers.
// Every section carries a 64-bit digest computed on the device over the array itself (trl_digest_kernel): a restore recomputes it
// over the arrays it uploaded, which checks the whole path from the file to HBM.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/terrainrl_b200.h"
#include "trl_handle.h"
#include "trl_mix64.h"

namespace trl {

constexpr unsigned long long kDigestK = 0xD1342543DE82EF95ull;

struct DigestRange {
    const unsigned char* p;     // 8-byte aligned
    unsigned long long bytes;
};

// out[s] += sum over the 64-bit little-endian words w_i of section s (the tail zero-padded) of mix64(w_i + (i + 1) K), mod 2^64.
// Wrapping addition is associative and commutative, so the grid-stride partial sums of any grid add up to the same value.
// grid (any, number of sections), 256 threads; out zeroed by the caller
__global__ void __launch_bounds__(256) trl_digest_kernel(const DigestRange* __restrict__ tab, unsigned long long* __restrict__ out) {
    const DigestRange r = tab[blockIdx.y];
    const unsigned long long full = r.bytes >> 3, words = (r.bytes + 7) >> 3;
    const unsigned long long* w = reinterpret_cast<const unsigned long long*>(r.p);
    unsigned long long s = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < words;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        unsigned long long v = 0;
        if (i < full) v = w[i];
        else
            for (unsigned k = 0; k < (unsigned)(r.bytes & 7); ++k) v |= (unsigned long long)r.p[8 * i + k] << (8 * k);
        s += mix64(v + (i + 1) * kDigestK);
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __shared__ unsigned long long part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += part[k];
        if (t) atomicAdd(out + blockIdx.y, t);
    }
}

}  // namespace trl

using namespace trl;

namespace {

constexpr char kMagic[8] = {'T', 'R', 'L', 'C', 'K', 'P', 'T', '1'};
constexpr uint32_t kVersion = 1;
constexpr int kNameLen = 48;
constexpr size_t kStageBytes = (size_t)64 << 20;     // pinned staging between the file and device memory

struct FileSection {
    char name[kNameLen];
    uint32_t dtype;
    uint32_t kind;          // 0: read before the handle is built, 1: state restored into the built handle
    uint64_t bytes;
    uint64_t digest;
};
static_assert(sizeof(FileSection) == 72, "fixed layout");

// what a restore needs before it can build the handle (section "meta")
struct Meta {
    int32_t n, mode;
    uint64_t rng_seed;
    int32_t trainers;         // bit p: policy slot p has a trainer
    int32_t policies;         // bit p >= 1: policy slot p holds its own net
    int32_t terrains;         // bit s >= 1: terrain slot s is loaded
    int32_t slots_active, train_slots;
    int32_t terrain_type[kMaxTerrainSlots];
};

// device memory freed when the scope ends
struct DevBuf {
    void* p = nullptr;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
};
struct PinnedBuf {
    unsigned char* p = nullptr;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    ~PinnedBuf() { if (p) cudaFreeHost(p); }
};

#define CKF(call, what)                                                                                         \
    do {                                                                                                        \
        cudaError_t e__ = (call);                                                                               \
        if (e__ != cudaSuccess) return trl_fail(std::string(what) + ": " + cudaGetErrorString(e__));            \
    } while (0)

// the restatement the file's kind-0 sections are checked with before anything is built from them
uint64_t host_digest(const unsigned char* p, size_t bytes) {
    uint64_t s = 0;
    for (size_t i = 0; 8 * i < bytes; ++i) {
        uint64_t v = 0;
        std::memcpy(&v, p + 8 * i, std::min<size_t>(8, bytes - 8 * i));
        s += mix64(v + (i + 1) * kDigestK);
    }
    return s;
}

// the digests of `secs` (device arrays, or host bytes staged through one device buffer) in one launch
int device_digests(const std::vector<CkptSection>& secs, cudaStream_t st, std::vector<uint64_t>* out) {
    out->assign(secs.size(), 0);
    if (secs.empty()) return 0;
    size_t host_total = 8;
    unsigned long long max_words = 1;
    for (const CkptSection& s : secs) {
        if (!s.dev) host_total += (s.bytes + 7) / 8 * 8;
        max_words = std::max<unsigned long long>(max_words, (s.bytes + 7) / 8);
    }
    DevBuf stage, tab, sums;
    CKF(cudaMalloc(&stage.p, host_total), "checkpoint digest");
    CKF(cudaMalloc(&tab.p, secs.size() * sizeof(DigestRange)), "checkpoint digest");
    CKF(cudaMalloc(&sums.p, secs.size() * 8), "checkpoint digest");
    std::vector<unsigned char> host(host_total, 0);
    std::vector<DigestRange> ranges(secs.size());
    size_t off = 0;
    for (size_t k = 0; k < secs.size(); ++k) {
        const CkptSection& s = secs[k];
        if (s.dev) {
            if (((uintptr_t)s.dev & 7u) != 0) return trl_fail("checkpoint: section '" + s.name + "' is not 8-byte aligned");
            ranges[k] = DigestRange{(const unsigned char*)s.dev, s.bytes};
        } else {
            if (s.bytes) std::memcpy(host.data() + off, s.host, s.bytes);
            ranges[k] = DigestRange{(const unsigned char*)stage.p + off, s.bytes};
            off += (s.bytes + 7) / 8 * 8;
        }
    }
    CKF(cudaMemcpyAsync(stage.p, host.data(), host_total, cudaMemcpyHostToDevice, st), "checkpoint digest");
    CKF(cudaMemcpyAsync(tab.p, ranges.data(), ranges.size() * sizeof(DigestRange), cudaMemcpyHostToDevice, st), "checkpoint digest");
    CKF(cudaMemsetAsync(sums.p, 0, secs.size() * 8, st), "checkpoint digest");
    const unsigned gx = (unsigned)std::min<unsigned long long>(1024, (max_words + 2047) / 2048);
    const DigestRange* d_tab = (const DigestRange*)tab.p;
    unsigned long long* d_sums = (unsigned long long*)sums.p;
    TRL_LAUNCH(trl_digest_kernel, dim3(gx, (unsigned)secs.size()), 256, 0, st, d_tab, d_sums);
    CKF(cudaGetLastError(), "trl_digest_kernel");
    CKF(cudaMemcpyAsync(out->data(), sums.p, secs.size() * 8, cudaMemcpyDeviceToHost, st), "checkpoint digest");
    CKF(cudaStreamSynchronize(st), "checkpoint digest");
    return 0;
}

// The handle's state that later calls read, with every stream drained.  Not listed: the pending decision lists (empty between two
// calls, checked at save), the decision scratch (act2, the slot sort / chunk tables), the cell statistics (recomputed by every
// trl_eval_stats_cell), the host staging of the readers, captured graphs and counters of launches and timers.
int handle_state(trl_handle* h, std::vector<CkptSection>* out) {
    const Buffers& B = h->B;
    const size_t n = (size_t)h->n, S = (size_t)B.S, W = 1 + 2 * S + (size_t)B.A;
    int cnt[2] = {0, 0};
    CKF(cudaMemcpy(&cnt[0], B.tuple_count, 4, cudaMemcpyDeviceToHost), "checkpoint");
    CKF(cudaMemcpy(&cnt[1], B.dist_count, 4, cudaMemcpyDeviceToHost), "checkpoint");
    const size_t rows = (size_t)std::min(std::max(cnt[0], 0), B.tuple_cap), dists = (size_t)std::min(std::max(cnt[1], 0), B.dist_cap);
    auto host = [&](const std::string& name, int dtype, void* p, size_t bytes) { out->push_back(CkptSection{name, dtype, nullptr, p, bytes, bytes}); };
    auto dev = [&](const std::string& name, int dtype, const void* p, size_t bytes, size_t cap) {
        out->push_back(CkptSection{name, dtype, const_cast<void*>(p), nullptr, bytes, cap});
    };
    auto fixed = [&](const std::string& name, int dtype, const void* p, size_t bytes) { dev(name, dtype, p, bytes, bytes); };
    host("mc", 0, &h->mc, sizeof(ModelConst));      // physics parameters, the exploration noise scale, the scene's terrain blend
    host("ex", 0, h->ex, sizeof(h->ex));
    host("terrain_table", 0, h->terrain, sizeof(h->terrain));
    host("terrain_lerp", 3, &h->terrain_lerp, 8);
    host("tuples_dropped", 0, &h->tuples_dropped, 8);
    if (h->slots_active) {
        host("env_slot_host", 1, h->env_slot_host.data(), n * 4);
        fixed("env_slot", 1, h->P.env_slot, n * 4);
    }
    if (!h->env_terrain_host.empty()) host("env_terrain_host", 1, h->env_terrain_host.data(), n * 4);
    if (h->env_phys) {       // physics slots: written only once one is loaded, so a handle without keeps the same file
        host("env_phys_host", 1, h->env_phys_host.data(), n * 4);
        fixed("env_phys", 1, h->env_phys, 2 * n * 4);
    }
    if (h->env_eval) {       // evaluation envs: likewise written only once trl_set_env_eval has been called
        host("env_eval_host", 1, h->env_eval_host.data(), n * 4);
        fixed("env_eval", 1, h->env_eval, 2 * n * 4);
    }
    if (h->env_body) {       // body slots: likewise written only once one is loaded
        host("env_body_host", 1, h->env_body_host.data(), n * 4);
        fixed("env_body", 1, h->env_body, 2 * n * 4);
    }
    if (h->ranges.env_draws) {     // ranged slots: likewise written only once one is loaded
        fixed("env_bdraw", 0, h->ranges.env_bdraw, n * sizeof(BodyConst));
        fixed("env_pdraw", 0, h->ranges.env_pdraw, n * sizeof(PhysParams));
        fixed("env_draws", 0, h->ranges.env_draws, 2 * n * 8);
    }
    fixed("B.d", 3, B.d, (size_t)D_NUM_FIELDS * n * 8);
    fixed("B.i", 1, B.i, (size_t)I_NUM_PLANES * n * 4);
    fixed("B.terrain", 2, B.terrain, n * 2 * kTerrainCap * 4);
    fixed("B.poli_state", 3, B.poli_state, n * S * 8);
    fixed("B.net_out", 3, B.net_out, n * kMaxNetOut * 8);
    fixed("B.tuple_sbeg", 3, B.tuple_sbeg, n * S * 8);
    fixed("B.tuple_action", 3, B.tuple_action, n * kNumParams * 8);
    fixed("B.com_stash", 3, B.com_stash, 2 * n * 8);
    fixed("B.catchup_done", 1, B.catchup_done, (kMaxLists + 1) * 4);     // [kMaxLists]: the fault flag trl_sync reports
    dev("B.tuples", 3, B.tuples, rows * W * 8, (size_t)B.tuple_cap * W * 8);
    dev("B.tuple_flags", 1, B.tuple_flags, rows * 4, (size_t)B.tuple_cap * 4);
    dev("B.tuple_env", 1, B.tuple_env, rows * 4, (size_t)B.tuple_cap * 4);
    fixed("B.tuple_count", 1, B.tuple_count, 4);
    dev("B.dist_log", 3, B.dist_log, dists * 8, (size_t)B.dist_cap * 8);
    dev("B.dist_env", 1, B.dist_env, dists * 4, (size_t)B.dist_cap * 4);
    fixed("B.dist_count", 1, B.dist_count, 4);
    // slot 0's own blobs even under a trainer: trl_trainer_destroy hands back all but the output offset / scale
    for (size_t k = 0; k < h->net_blobs.size(); ++k) fixed("net." + std::to_string(k), 3, h->net_blobs[k], (size_t)h->net_counts[k] * 8);
    for (int p = 1; p < kMaxPolicySlots; ++p) {
        if (h->slot_blobs[p].empty() || h->slot_trainer[p]) continue;      // a slot trainer's net is in the trainer's sections
        for (size_t k = 0; k < h->slot_blobs[p].size(); ++k)
            fixed("slot" + std::to_string(p) + "." + std::to_string(k), 3, h->slot_blobs[p][k], (size_t)h->net_counts[k] * 8);
    }
    return 0;
}

trl_trainer* trainer_of(trl_handle* h, int p) { return p == 0 ? h->trainer : h->slot_trainer[p]; }

int all_state(trl_handle* h, std::vector<CkptSection>* out) {
    if (handle_state(h, out)) return 1;
    for (int p = 0; p < kMaxPolicySlots; ++p)
        if (trainer_of(h, p) && trl_trainer_state(trainer_of(h, p), "t" + std::to_string(p) + ".", out)) return 1;
    return 0;
}

struct Blob {
    std::string name;
    int dtype;
    std::vector<unsigned char> bytes;
};
template <typename T>
Blob blob_of(const std::string& name, int dtype, const T* p, size_t count) {
    const unsigned char* b = reinterpret_cast<const unsigned char*>(p);
    return Blob{name, dtype, std::vector<unsigned char>(b, b + count * sizeof(T))};
}

int save_impl(trl_handle* h, const char* path, const void* user, size_t user_bytes) {
    const std::string who = "trl_checkpoint_save";
    if (!h) return trl_fail(who + ": null handle");
    if (!path) return trl_fail(who + ": null path");
    if (user_bytes && !user) return trl_fail(who + ": null user blob");
    if (h->comm) return trl_fail(who + ": the handle has a communicator (a multi-GPU run would need every rank to agree on the cut)");
    if (h->snap_pending) return trl_fail(who + ": a trl_snapshot is pending (trl_snapshot_wait first)");
    if (trl_drain(h)) return 1;
    {
        // the last launch of an update joins every side stream, and every decision launch re-arms the list it consumed: no decision is in
        // flight between two calls, and nothing in the pending lists carries over
        int pc[kMaxLists], cd[kMaxLists + 1], dc = 0;
        CKF(cudaMemcpy(pc, h->B.pending_count, sizeof(pc), cudaMemcpyDeviceToHost), who);
        CKF(cudaMemcpy(cd, h->B.catchup_done, sizeof(cd), cudaMemcpyDeviceToHost), who);
        CKF(cudaMemcpy(&dc, h->done_count, 4, cudaMemcpyDeviceToHost), who);
        for (int l = 0; l < kMaxLists; ++l)
            if (pc[l] != 0 || cd[l] != 0) return trl_fail(who + ": pending decision list " + std::to_string(l) + " is not empty between two calls");
        if (dc != 0) return trl_fail(who + ": a decision launch has not completed");
    }
    std::vector<CkptSection> state;
    if (all_state(h, &state)) return 1;       // refuses an asynchronous trainer
    Meta m;
    std::memset(&m, 0, sizeof(m));
    m.n = h->n; m.mode = h->mode; m.rng_seed = h->mc.rng_seed;
    m.slots_active = h->slots_active; m.train_slots = h->train_slots;
    std::vector<Blob> build;
    {
        std::ostringstream os;
        if (!h->scene.write(os)) return trl_fail(who + ": scene pack serialisation failed");
        const std::string s = os.str();
        build.push_back(blob_of("scene", 0, s.data(), s.size()));
    }
    for (int p = 0; p < kMaxPolicySlots; ++p) {
        if (trl_trainer* t = trainer_of(h, p)) {
            m.trainers |= 1 << p;
            double params[10];
            if (trl_trainer_params(t, params, nullptr)) return 1;
            build.push_back(blob_of("t" + std::to_string(p) + ".params", 3, params, 10));
        }
        if (p > 0 && !h->slot_blobs[p].empty()) m.policies |= 1 << p;
    }
    for (int s = 1; s < kMaxTerrainSlots; ++s) {
        if (!h->terrain_loaded[s]) continue;
        m.terrains |= 1 << s;
        m.terrain_type[s] = h->terrain[s].type;
        build.push_back(blob_of("terrain_sets." + std::to_string(s), 3, h->terrain_sets[s].data(), h->terrain_sets[s].size()));
    }
    if (h->env_phys) {
        int32_t mask = 0;
        for (int s = 1; s < kMaxPhysSlots; ++s)
            if (h->phys_loaded[s]) mask |= 1 << s;
        build.push_back(blob_of("phys_loaded", 1, &mask, 1));
        build.push_back(blob_of("phys_table", 0, h->phys, kMaxPhysSlots));
    }
    if (h->env_eval) {
        const int32_t on = 1;
        build.push_back(blob_of("eval_envs", 1, &on, 1));
    }
    if (h->env_body) {
        int32_t mask = 0;
        for (int s = 1; s < kMaxBodySlots; ++s)
            if (h->body_loaded[s]) mask |= 1 << s;
        build.push_back(blob_of("body_loaded", 1, &mask, 1));
        build.push_back(blob_of("body_table", 0, h->body, kMaxBodySlots));
    }
    if (h->ranges.env_draws) {     // the ranged slots' hi tables (their lo tables are the slot tables above)
        const int32_t masks[2] = {(int32_t)h->ranges.body_ranged, (int32_t)h->ranges.phys_ranged};
        build.push_back(blob_of("ranges", 1, masks, 2));
        build.push_back(blob_of("range_body_hi", 0, h->ranges.body_hi, kMaxBodySlots));
        build.push_back(blob_of("range_phys_hi", 0, h->ranges.phys_hi, kMaxPhysSlots));
    }
    build.insert(build.begin() + 1, blob_of("meta", 0, &m, 1));
    build.push_back(blob_of("user", 0, (const unsigned char*)user, user_bytes));
    std::vector<CkptSection> all;
    for (Blob& b : build) all.push_back(CkptSection{b.name, b.dtype, nullptr, b.bytes.data(), b.bytes.size(), b.bytes.size()});
    const size_t n_build = all.size();
    all.insert(all.end(), state.begin(), state.end());
    std::vector<uint64_t> dig;
    if (device_digests(all, h->stream, &dig)) return 1;
    // header, table, bytes; written beside the target and renamed over it once complete
    const std::string tmp = std::string(path) + ".tmp";
    std::ofstream f(tmp, std::ios::binary | std::ios::trunc);
    if (!f) return trl_fail(who + ": cannot write " + tmp);
    const uint32_t hdr[2] = {kVersion, (uint32_t)all.size()};
    f.write(kMagic, 8);
    f.write(reinterpret_cast<const char*>(hdr), 8);
    size_t max_dev = 0;
    for (size_t k = 0; k < all.size(); ++k) {
        FileSection fs;
        std::memset(&fs, 0, sizeof(fs));
        if (all[k].name.size() >= (size_t)kNameLen) return trl_fail(who + ": section name too long: " + all[k].name);
        std::memcpy(fs.name, all[k].name.data(), all[k].name.size());
        fs.dtype = (uint32_t)all[k].dtype; fs.kind = k < n_build ? 0 : 1; fs.bytes = all[k].bytes; fs.digest = dig[k];
        f.write(reinterpret_cast<const char*>(&fs), sizeof(fs));
        if (all[k].dev) max_dev = std::max(max_dev, all[k].bytes);
    }
    PinnedBuf stage;
    const size_t chunk = std::max<size_t>(8, std::min(kStageBytes, max_dev));
    CKF(cudaMallocHost((void**)&stage.p, chunk), who);
    for (const CkptSection& s : all) {
        if (!s.dev) { f.write(reinterpret_cast<const char*>(s.host), (std::streamsize)s.bytes); continue; }
        for (size_t off = 0; off < s.bytes; off += chunk) {
            const size_t len = std::min(chunk, s.bytes - off);
            CKF(cudaMemcpyAsync(stage.p, (const unsigned char*)s.dev + off, len, cudaMemcpyDeviceToHost, h->stream), who);
            CKF(cudaStreamSynchronize(h->stream), who);
            f.write(reinterpret_cast<const char*>(stage.p), (std::streamsize)len);
        }
    }
    f.close();
    if (!f || std::rename(tmp.c_str(), path) != 0) {
        std::remove(tmp.c_str());
        return trl_fail(who + ": writing " + std::string(path) + " failed");
    }
    return 0;
}

trl_handle* load_impl(const char* path, int device, trl_trainer** trainers_out, void* user, size_t user_cap, size_t* user_bytes) {
    const std::string who = "trl_create_from_checkpoint";
    auto refuse = [&](const std::string& why) -> trl_handle* { trl_fail(who + ": " + why); return nullptr; };
    if (!path) return refuse("null path");
    std::ifstream f(path, std::ios::binary);
    if (!f) return refuse(std::string("cannot open ") + path);
    f.seekg(0, std::ios::end);
    const uint64_t size = (uint64_t)f.tellg();
    f.seekg(0, std::ios::beg);
    char magic[8];
    uint32_t hdr[2] = {0, 0};
    f.read(magic, 8);
    f.read(reinterpret_cast<char*>(hdr), 8);
    if (!f || size < 16) return refuse("truncated file (no header)");
    if (std::memcmp(magic, kMagic, 8) != 0) return refuse("not a checkpoint (bad magic)");
    if (hdr[0] != kVersion) return refuse("unsupported version " + std::to_string(hdr[0]) + " (this build reads version " + std::to_string(kVersion) + ")");
    if (hdr[1] == 0 || (uint64_t)hdr[1] > (size - 16) / sizeof(FileSection)) return refuse("truncated file (section table)");
    std::vector<FileSection> tab(hdr[1]);
    f.read(reinterpret_cast<char*>(tab.data()), (std::streamsize)(tab.size() * sizeof(FileSection)));
    if (!f) return refuse("truncated file (section table)");
    std::vector<uint64_t> offset(tab.size());
    uint64_t end = 16 + tab.size() * sizeof(FileSection);
    std::map<std::string, size_t> index;
    for (size_t k = 0; k < tab.size(); ++k) {
        if (std::memchr(tab[k].name, 0, kNameLen) == nullptr || tab[k].kind > 1) return refuse("damaged section table");
        if (tab[k].bytes > size) return refuse("truncated file (section '" + std::string(tab[k].name) + "')");
        offset[k] = end;
        end += tab[k].bytes;
        index[tab[k].name] = k;
    }
    if (end > size) return refuse("truncated file (" + std::to_string(size) + " bytes, the section table needs " + std::to_string(end) + ")");
    if (end < size) return refuse("trailing bytes after the last section");
    // kind 0: read and checked before anything is built from them
    std::map<std::string, std::vector<unsigned char>> build;
    for (size_t k = 0; k < tab.size(); ++k) {
        if (tab[k].kind != 0) continue;
        std::vector<unsigned char>& b = build[tab[k].name];
        b.resize(tab[k].bytes);
        f.seekg((std::streamoff)offset[k]);
        f.read(reinterpret_cast<char*>(b.data()), (std::streamsize)b.size());
        if (!f) return refuse("read error in section '" + std::string(tab[k].name) + "'");
        if (host_digest(b.data(), b.size()) != tab[k].digest) return refuse("digest mismatch in section '" + std::string(tab[k].name) + "'");
    }
    auto need = [&](const std::string& name, size_t bytes) -> const std::vector<unsigned char>* {
        auto it = build.find(name);
        if (it == build.end() || (bytes && it->second.size() != bytes)) return nullptr;
        return &it->second;
    };
    const auto* mb = need("meta", sizeof(Meta));
    const auto* sb = need("scene", 0);
    const auto* ub = need("user", 0);
    if (!mb || !sb || !ub) return refuse("the scene, meta or user section is missing or has the wrong size");
    Meta m;
    std::memcpy(&m, mb->data(), sizeof(m));
    const auto* eb = need("eval_envs", 0);       // evaluation envs: the slot build runs even with slot 0 alone
    if (eb && (eb->size() != 4 || m.mode != TRL_MODE_EXPLORE)) return refuse("the eval_envs section is malformed");
    if (m.n <= 0 || (m.mode != TRL_MODE_POLI_EVAL && m.mode != TRL_MODE_EXPLORE) || (m.trainers & ~0xff) || (m.policies & ~0xfe) ||
        (m.terrains & ~0xfe) || (m.slots_active != 0) != ((m.policies | (m.trainers & 0xfe)) != 0 || eb != nullptr))
        return refuse("inconsistent meta section");
    if (m.trainers && !trainers_out) return refuse("the checkpoint holds trainers: pass an array of 8 to receive them");
    auto* h = new trl_handle();
    {
        std::istringstream is(std::string(sb->begin(), sb->end()));
        std::string err;
        if (!h->scene.read(is, "the checkpoint's scene section", &err)) { delete h; return refuse(err); }
    }
    h = trl_create_common(h, m.n, device, m.mode, nullptr, m.rng_seed);
    if (!h) return nullptr;
    trl_trainer* ts[kMaxPolicySlots] = {};
    auto bail = [&](const std::string& why) -> trl_handle* {
        if (!why.empty()) trl_fail(who + ": " + why);
        const std::string msg = trl_last_error();
        trl_destroy(h);                                  // orphans the trainers: their device memory goes with the handle
        for (trl_trainer* t : ts) trl_trainer_destroy(t);
        trl_fail(msg);
        return nullptr;
    };
    // the slots, through the paths that made them
    for (int s = 1; s < kMaxTerrainSlots; ++s) {
        if (!(m.terrains & (1 << s))) continue;
        const auto* tb = need("terrain_sets." + std::to_string(s), 0);
        if (!tb || tb->size() % (kTerrainParams * 8) != 0) return bail("terrain slot " + std::to_string(s) + ": parameter sets missing or malformed");
        std::vector<double> sets(tb->size() / 8);
        std::memcpy(sets.data(), tb->data(), tb->size());
        if (trl_set_terrain_slot(h, s, m.terrain_type[s], std::move(sets))) return bail("");
    }
    if (const auto* lb = need("phys_loaded", 0)) {
        const auto* tb = need("phys_table", sizeof(PhysParams) * kMaxPhysSlots);
        int32_t mask = 0;
        if (lb->size() == 4) std::memcpy(&mask, lb->data(), 4);
        if (!tb || lb->size() != 4 || mask == 0 || (mask & ~0xfe)) return bail("physics slots: table or slot mask missing or malformed");
        PhysParams table[kMaxPhysSlots];
        std::memcpy(table, tb->data(), sizeof(table));
        for (int s = 1; s < kMaxPhysSlots; ++s) {
            if (!(mask & (1 << s))) continue;
            const PhysParams& q = table[s];
            const double p7[7] = {q.kn, q.dn, q.mu, q.v_eps, q.contact_tol, q.k_lim, q.d_lim};
            if (trl_load_physics(h, s, p7, q.vertex_contacts)) return bail("");
        }
    }
    if (const auto* lb = need("body_loaded", 0)) {     // the body slots from the stored tables (the files may be gone)
        const auto* tb = need("body_table", sizeof(BodyConst) * kMaxBodySlots);
        int32_t mask = 0;
        if (lb->size() == 4) std::memcpy(&mask, lb->data(), 4);
        // a handle whose only ranged slots are physics slots runs the body-slot build without a body slot
        if (!tb || lb->size() != 4 || (mask == 0 && !need("ranges", 0)) || (mask & ~0xfe))
            return bail("body slots: table or slot mask missing or malformed");
        std::vector<BodyConst> table(kMaxBodySlots);
        std::memcpy(table.data(), tb->data(), sizeof(BodyConst) * kMaxBodySlots);
        for (int s = 1; s < kMaxBodySlots; ++s)
            if ((mask & (1 << s)) && trl_set_body_slot(h, s, table[s])) return bail("");
    }
    if (const auto* rb = need("ranges", 0)) {         // the ranged slots: their lo tables are the slots restored above
        const auto* bh = need("range_body_hi", sizeof(BodyConst) * kMaxBodySlots);
        const auto* ph = need("range_phys_hi", sizeof(PhysParams) * kMaxPhysSlots);
        int32_t masks[2] = {0, 0};
        if (rb->size() == 8) std::memcpy(masks, rb->data(), 8);
        if (!bh || !ph || rb->size() != 8 || (masks[0] & ~0xfe) || (masks[1] & ~0xfe) || !need("body_loaded", 0))
            return bail("ranged slots: tables or slot masks missing or malformed");
        std::vector<BodyConst> body_hi(kMaxBodySlots);
        std::vector<PhysParams> phys_hi(kMaxPhysSlots);
        std::memcpy(body_hi.data(), bh->data(), bh->size());
        std::memcpy(phys_hi.data(), ph->data(), ph->size());
        if (trl_enable_ranges(h)) return bail("");
        for (int s = 1; s < kMaxBodySlots; ++s) {
            if (!(masks[0] & (1 << s))) continue;
            if (!h->body_loaded[s]) return bail("ranged body slot " + std::to_string(s) + " has no lo table");
            if (trl_set_body_range(h, s, h->body[s], body_hi[s])) return bail("");
        }
        for (int s = 1; s < kMaxPhysSlots; ++s) {
            if (!(masks[1] & (1 << s))) continue;
            if (!h->phys_loaded[s]) return bail("ranged physics slot " + std::to_string(s) + " has no lo table");
            if (trl_set_phys_range(h, s, h->phys[s], phys_hi[s])) return bail("");
        }
    }
    if ((m.policies || m.trainers || eb) && !h->mc.has_net) return bail("the scene has no policy net");
    if (eb && trl_enable_env_eval(h)) return bail("");
    for (int p = 1; p < kMaxPolicySlots; ++p)
        if ((m.policies & (1 << p)) && trl_stage_slot_model(h, p, nullptr, nullptr)) return bail("");
    for (int p = 0; p < kMaxPolicySlots; ++p) {
        if (!(m.trainers & (1 << p))) continue;
        const auto* pb = need("t" + std::to_string(p) + ".params", 80);
        if (!pb) return bail("the parameters of the trainer of slot " + std::to_string(p) + " are missing");
        double params[10];
        std::memcpy(params, pb->data(), 80);
        if (!(ts[p] = trl_trainer_create_slot(h, p, params, nullptr, nullptr))) return bail("");
    }
    h->slots_active = m.slots_active != 0;
    h->train_slots = m.train_slots != 0;
    // kind 1: the state, into the arrays of the built handle
    std::vector<CkptSection> dst;
    if (all_state(h, &dst)) return bail("");
    std::vector<size_t> state_idx;
    for (size_t k = 0; k < tab.size(); ++k)
        if (tab[k].kind == 1) state_idx.push_back(k);
    if (state_idx.size() != dst.size()) return bail("the file's state sections do not match the handle its scene and slots build");
    size_t max_dev = 0;
    for (size_t j = 0; j < dst.size(); ++j) {
        const FileSection& fs = tab[state_idx[j]];
        if (dst[j].name != fs.name) return bail("section '" + std::string(fs.name) + "' where the restored handle has '" + dst[j].name + "'");
        if (fs.bytes > dst[j].cap || (dst[j].bytes == dst[j].cap && fs.bytes != dst[j].cap))
            return bail("section '" + dst[j].name + "' has " + std::to_string(fs.bytes) + " bytes, the restored handle holds " + std::to_string(dst[j].cap));
        dst[j].bytes = fs.bytes;
        if (dst[j].dev) max_dev = std::max<size_t>(max_dev, fs.bytes);
    }
    {
        PinnedBuf stage;
        const size_t chunk = std::max<size_t>(8, std::min(kStageBytes, max_dev));
        if (cudaMallocHost((void**)&stage.p, chunk) != cudaSuccess) return bail("pinned staging allocation failed");
        for (size_t j = 0; j < dst.size(); ++j) {
            const CkptSection& s = dst[j];
            f.seekg((std::streamoff)offset[state_idx[j]]);
            if (!s.dev) { f.read(reinterpret_cast<char*>(s.host), (std::streamsize)s.bytes); if (!f) return bail("read error in section '" + s.name + "'"); continue; }
            for (size_t off = 0; off < s.bytes; off += chunk) {
                const size_t len = std::min(chunk, s.bytes - off);
                f.read(reinterpret_cast<char*>(stage.p), (std::streamsize)len);
                if (!f) return bail("read error in section '" + s.name + "'");
                if (cudaMemcpyAsync((unsigned char*)s.dev + off, stage.p, len, cudaMemcpyHostToDevice, h->stream) != cudaSuccess ||
                    cudaStreamSynchronize(h->stream) != cudaSuccess)
                    return bail("upload of section '" + s.name + "' failed");
            }
        }
    }
    // every section's digest again, on the device, over what now sits in memory
    {
        std::vector<CkptSection> all;
        std::vector<size_t> file_idx;
        for (size_t k = 0; k < tab.size(); ++k) {
            if (tab[k].kind != 0) continue;
            std::vector<unsigned char>& b = build[tab[k].name];
            all.push_back(CkptSection{tab[k].name, (int)tab[k].dtype, nullptr, b.data(), b.size(), b.size()});
            file_idx.push_back(k);
        }
        for (size_t j = 0; j < dst.size(); ++j) { all.push_back(dst[j]); file_idx.push_back(state_idx[j]); }
        std::vector<uint64_t> dig;
        if (device_digests(all, h->stream, &dig)) return bail("");
        for (size_t k = 0; k < all.size(); ++k)
            if (dig[k] != tab[file_idx[k]].digest) return bail("digest mismatch in section '" + all[k].name + "'");
    }
    // the fill levels the counters now name must be the ones the file holds
    {
        std::vector<CkptSection> again;
        if (all_state(h, &again)) return bail("");
        for (size_t j = 0; j < again.size(); ++j)
            if (again[j].bytes != dst[j].bytes) return bail("section '" + again[j].name + "' does not match the counters restored with it");
    }
    if (cudaMemcpy(h->d_ex, h->ex, sizeof(h->ex), cudaMemcpyHostToDevice) != cudaSuccess) return bail("exploration settings upload failed");
    h->slot_dirty = true;
    trl_drop_graphs(h);
    if (trl_reupload_model(h)) return bail("");
    if (user && ub->size()) std::memcpy(user, ub->data(), std::min(user_cap, ub->size()));
    if (user_bytes) *user_bytes = ub->size();
    if (trainers_out)
        for (int p = 0; p < kMaxPolicySlots; ++p) trainers_out[p] = ts[p];
    return h;
}

}  // namespace

extern "C" {

int trl_checkpoint_save(trl_handle* h, const char* path, const void* user, size_t user_bytes) {
    try {
        return save_impl(h, path, user, user_bytes);
    } catch (const std::exception& e) {
        return trl_fail(std::string("trl_checkpoint_save: ") + e.what());
    }
}

trl_handle* trl_create_from_checkpoint(const char* path, int device, trl_trainer** trainers, void* user, size_t user_cap, size_t* user_bytes) {
    try {
        return load_impl(path, device, trainers, user, user_cap, user_bytes);
    } catch (const std::exception& e) {       // bad_alloc from a damaged file must not cross the C ABI
        trl_fail(std::string("trl_create_from_checkpoint: ") + e.what());
        return nullptr;
    }
}

}  // extern "C"
