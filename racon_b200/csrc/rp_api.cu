/*
 * rp_api.cu — the C ABI (include/racon_b200.h) over the sm_90a kernels.  Product library
 * libracon_b200.so = this file alone (the C++ host layer above it, host_mirror.cpp, is a library of its own).
 * There is no CPU implementation behind these calls.
 *
 * POA batch object = racon::CUDABatchProcessor + cudapoa::Batch (src/cuda/cudabatch.cpp:23-278):
 *   add (copy into pinned staging) -> upload (H2D) -> launch (one persistent kernel) -> download (D2H).
 */
#if defined(RP_HOST_SIM)
#include "cuda_sim_runtime.h"   // TEST-ONLY build of this file (lib/simapi): see that header
#else
#include <cuda_runtime.h>
#endif

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <array>
#include <functional>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "gather_core.cuh"
#include "myers_core.cuh"
#include "poa_core.cuh"
#include "poa_pack.hpp"
#include "racon_b200.h"

namespace {

thread_local std::string g_last_error;

rp_status fail(rp_status s, const std::string& msg) {
    g_last_error = msg;
    return s;
}

#define RP_CUDA(call)                                                                                   \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess)                                                                          \
            return fail(RP_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));               \
    } while (0)

void* pinned_alloc(size_t n) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, n ? n : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    return p;
}
void pinned_free(void* p) { cudaFreeHost(p); }
const rp::HostAllocator kPinned{pinned_alloc, pinned_free};

/* growable pinned host buffer: the staging of a batch object's inputs and results */
template <typename T>
struct PinnedBuf : rp::GrowBuf<T> {
    PinnedBuf() : rp::GrowBuf<T>(&kPinned) {}
};

/* growable device buffer; frees its memory when destroyed */
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        size_t nc = n + n / 8 + 4096;          // modest head room: the object works inside a memory budget
        nc = (nc + 0xffffu) & ~static_cast<size_t>(0xffffu);
        cudaError_t e = cudaMalloc(&p, nc);
        cap = e == cudaSuccess ? nc : 0;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
};

/* Reserves `bytes` of d and binds its memory to the kernel parameter `out`. */
template <typename T>
cudaError_t reserve(DevBuf& d, size_t bytes, T*& out) {
    const cudaError_t e = d.reserve(bytes);
    out = static_cast<T*>(d.p);
    return e;
}

/* Copies a staged array into d (at least 16 bytes are reserved, also for an empty one) on the object's stream, adds its
 * bytes to the object's H2D count and binds d to the kernel parameter `out`. */
template <typename Obj, typename T>
cudaError_t upload(Obj* o, DevBuf& d, const rp::GrowBuf<T>& h, const T*& out) {
    const size_t bytes = h.bytes();
    cudaError_t e = reserve(d, bytes ? bytes : 16, out);
    if (e != cudaSuccess) return e;
    o->last_h2d += bytes;
    return bytes ? cudaMemcpyAsync(d.p, h.data, bytes, cudaMemcpyHostToDevice, o->stream) : cudaSuccess;
}

/* the device checks of every rp_*_create; makes the device current */
rp_status check_device(int device) {
    int ndev = rp_device_count();
    if (ndev <= 0) return fail(RP_ERR_NO_DEVICE, "no CUDA device");
    if (device < 0 || device >= ndev) return fail(RP_ERR_INVALID, "device index out of range");
    RP_CUDA(cudaSetDevice(device));
    return RP_OK;
}

/* The device of a batch object and the stream its work is queued on: a stream of its own, created with the object and
 * destroyed with it, until rp_*_set_stream hands it one of the caller's. */
struct StreamOwner {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = true;
    ~StreamOwner() {
        if (own_stream && stream) cudaStreamDestroy(stream);
    }
};

/* a new batch object on `device`, with a stream of its own */
template <typename Obj>
rp_status create_object(Obj*& o, int device) {
    const rp_status s = check_device(device);
    if (s != RP_OK) return s;
    o = new (std::nothrow) Obj();
    if (!o) return fail(RP_ERR_NOMEM, "host allocation failed");
    o->device = device;
    const cudaError_t e = cudaStreamCreateWithFlags(&o->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) return RP_OK;
    o->stream = nullptr;
    delete o;
    o = nullptr;
    return fail(RP_ERR_CUDA, std::string("cudaStreamCreate: ") + cudaGetErrorString(e));
}

rp_status set_stream(StreamOwner* o, void* cuda_stream) {
    if (!o) return fail(RP_ERR_INVALID, "null object");
    if (o->own_stream && o->stream) {
        cudaStreamSynchronize(o->stream);
        cudaStreamDestroy(o->stream);
    }
    o->stream = static_cast<cudaStream_t>(cuda_stream);
    o->own_stream = false;
    return RP_OK;
}

/* rp_*_query: has the work queued on the object's stream by its last run finished? (`launched`: the object's flag) */
rp_status query_stream(StreamOwner* o, bool launched) {
    if (!o) return fail(RP_ERR_INVALID, "null object");
    if (!launched) return fail(RP_ERR_STATE, "query before run");
    RP_CUDA(cudaSetDevice(o->device));
    const cudaError_t e = cudaStreamQuery(o->stream);
    if (e == cudaErrorNotReady) return RP_NOT_READY;
    RP_CUDA(e);
    return RP_OK;
}

constexpr int kWarpsPerBlock = 4;
constexpr uint32_t kBandPaysFromWindowLength = 768;   // rows of two or more 512-column chunks

/* Blocks per SM of the POA kernel, which sets its register cap, by columns per lane of a row.  Measured on the H100
 * (DESIGN.md §11b): 16 columns (the full matrix, and the 8- and 16-lane bands) run best at 3 — at 4 the 128-register cap
 * makes ptxas spill inside the DP row loop on sm_90a; the narrow 32 x 8 and 32 x 4 bands need fewer registers per row
 * and run best at 5. */
constexpr int poa_blocks_per_sm(int kb) { return kb == 16 ? 3 : 5; }

/* Persistent kernel: every GROUP of G lanes (G = 8, 16, 32; rp_warp.cuh) is an independent worker that pulls
 * windows from an atomic queue — 32/G windows in flight per warp, advancing together wherever their control
 * flow agrees.  Compiled for each layout (lanes per window x columns per lane of a row); RP_POA_GROUP /
 * RP_POA_BAND_K select one (defaults in configure). */
#if defined(RP_HOST_SIM)
/* TEST-ONLY stand-ins of the two kernels (cuda_sim_runtime.h): the same per-window / per-overlap device functions, run as
 * cooperative fibres, the queue walked by one worker after the other. */
struct SimLaunch {
    uint32_t blocks, threads;
};
template <int G, int KB>
struct SimPoaJob {
    const rp::PoaParams* P;
    uint32_t w;
    uint8_t *slot, *smem;
    static void entry(void* arg) {
        SimPoaJob* j = static_cast<SimPoaJob*>(arg);
        rp::poa_window<G, KB>(*j->P, j->w, j->slot, j->smem);
    }
};
template <int G, int KB>
void rp_poa_kernel(rp::PoaParams P, SimLaunch L) {
    const uint32_t workers = L.blocks * (L.threads / G);
    std::vector<uint8_t> smem(P.smem_per_group + 64);
    uint8_t* smem_al = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem.data()) + 15) & ~uintptr_t(15));
    for (;;) {
        const uint32_t q = (*P.queue_head)++;
        if (q >= P.n_windows) break;
        SimPoaJob<G, KB> job{&P, P.queue[q], P.scratch + static_cast<uint64_t>(q % workers) * P.lay.bytes, smem_al};
        rp::sim::run_warp(SimPoaJob<G, KB>::entry, &job, 256 * 1024, G);
    }
}
typedef void (*PoaKernel)(rp::PoaParams, SimLaunch);
struct SimGatherJob {
    const rp::GatherParams* P;
    uint32_t s;
    static void entry(void* arg) {
        SimGatherJob* j = static_cast<SimGatherJob*>(arg);
        rp::gather_sequence(*j->P, j->s);
    }
};
void rp_gather_kernel(rp::GatherParams P, SimLaunch) {
    for (uint32_t s = 0; s < P.n_seqs; ++s) {
        SimGatherJob job{&P, s};
        rp::sim::run_warp(SimGatherJob::entry, &job);
    }
}
struct SimAlnJob {
    const rp::AlnParams* P;
    uint32_t pair;
    uint8_t* slot;
    static void entry(void* arg) {
        SimAlnJob* j = static_cast<SimAlnJob*>(arg);
        rp::aln_pair(*j->P, j->pair, j->slot);
    }
};
void rp_aln_kernel(rp::AlnParams P, SimLaunch L) {
    const uint32_t workers = L.blocks * (L.threads / 32);
    for (;;) {
        const uint32_t q = (*P.queue_head)++;
        if (q >= P.n_pairs) break;
        SimAlnJob job{&P, P.queue[q], P.scratch + static_cast<uint64_t>(q % workers) * P.lay.bytes};
        rp::sim::run_warp(SimAlnJob::entry, &job);
    }
}
template <typename Params>
cudaError_t launch(void (*kernel)(Params, SimLaunch), uint32_t blocks, uint32_t threads, uint32_t, cudaStream_t,
                   const Params& P) {
    kernel(P, SimLaunch{blocks, threads});
    return cudaSuccess;
}
#else
/* kBlocksPerSm is fixed by the layout; it stays a template argument so that the kernel keeps its symbol name
 * (rp_poa_kernel<G, KB, blocks per SM>), by which tools/sass_by_line.py, the SASS tests and profiles find it */
template <int G, int KB, int kBlocksPerSm = poa_blocks_per_sm(KB)>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, kBlocksPerSm) rp_poa_kernel(rp::PoaParams P) {
    extern __shared__ __align__(16) uint8_t smem_all[];
    const uint32_t grp = threadIdx.x / G;
    const uint32_t worker = blockIdx.x * (blockDim.x / G) + grp;
    uint8_t* slot = P.scratch + static_cast<uint64_t>(worker) * P.lay.bytes;
    /* the group's shared-memory address (shared state space, 32 bits) is pinned in a register: left alone, the compiler
     * re-derives it — S2R of the CTA's shared window and of the thread index, shift, multiply — wherever a shared-memory
     * address is rebuilt inside the hot loops, at the head of every DP row's and every traceback step's dependency chain */
    uint32_t smem_s = static_cast<uint32_t>(__cvta_generic_to_shared(smem_all)) + grp * P.smem_per_group;
    RP_KEEP_IN_REGISTER(smem_s);
    uint8_t* smem = static_cast<uint8_t*>(__cvta_shared_to_generic(smem_s));
    for (;;) {
        uint32_t q = 0;
        if (rp::glane<G>() == 0) q = atomicAdd(P.queue_head, 1u);
        q = rp::gshfl<G>(q, 0);
        if (q >= P.n_windows) break;
        rp::poa_window<G, KB>(P, P.queue[q], slot, smem);
    }
}

typedef void (*PoaKernel)(rp::PoaParams);
#endif
/* lanes per window x columns per lane of a row (band_k is 16 unless group is 32) */
PoaKernel pick_kernel(int group, int band_k) {
    if (group == 8) return rp_poa_kernel<8, 16>;
    if (group == 16) return rp_poa_kernel<16, 16>;
    if (band_k == 4) return rp_poa_kernel<32, 4>;
    if (band_k == 8) return rp_poa_kernel<32, 8>;
    return rp_poa_kernel<32, 16>;
}

#if !defined(RP_HOST_SIM)
/* layer extraction (gather_core.cuh): warps stride over the packed sequences of the batch */
__global__ void __launch_bounds__(256) rp_gather_kernel(rp::GatherParams P) {
    const uint32_t warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < P.n_seqs; s += warps)
        rp::gather_sequence(P, s);
}

/* 4 blocks of 4 warps per SM */
__global__ void __launch_bounds__(kWarpsPerBlock * 32, 4) rp_aln_kernel(rp::AlnParams P) {
    const int warp = threadIdx.x >> 5;
    const uint32_t worker = blockIdx.x * (blockDim.x >> 5) + warp;
    uint8_t* slot = P.scratch + static_cast<uint64_t>(worker) * P.lay.bytes;
    for (;;) {
        uint32_t q = 0;
        if ((threadIdx.x & 31) == 0) q = atomicAdd(P.queue_head, 1u);
        q = __shfl_sync(0xffffffffu, q, 0);
        if (q >= P.n_pairs) break;
        rp::aln_pair(P, P.queue[q], slot);
    }
}

template <typename Params>
cudaError_t launch(void (*kernel)(Params), uint32_t blocks, uint32_t threads, uint32_t smem, cudaStream_t stream,
                   const Params& P) {
    kernel<<<blocks, threads, smem, stream>>>(P);
    return cudaGetLastError();
}
#endif

/* the layer-extraction grid: one warp per sequence, at most 8 blocks per SM of the device */
uint32_t gather_blocks(int device, uint32_t n_seqs) {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms < 1) sms = 1;
    return std::max<uint32_t>(1, std::min<uint32_t>(static_cast<uint32_t>(sms) * 8, (n_seqs + 7) / 8));
}

}  // namespace

/* device-resident sequences (include/racon_b200.h: rp_reads_create) */
struct rp_reads {
    int device = 0;
    std::vector<const char*> data, quality;       // the caller's host arrays (kept valid by the caller)
    std::vector<uint32_t> length;
    std::vector<uint64_t> off;                    // position of each sequence in the device arrays, n + 1
    std::vector<std::array<uint64_t, 4>> chars;   // per sequence: which byte values occur (256-bit set)
    DevBuf d_bases, d_quals;
    bool any_quality = false;
};

/* Layer extraction on `stream`: packed sequence s of the batch = the store's bytes from src_pos[s] on, written to bases
 * (and, unless weights is null, its weights from the store's qualities). */
static cudaError_t launch_gather(const rp_reads* reads, void* bases, void* weights, const uint32_t* seq_off,
                                 const uint64_t* src_pos, const uint8_t* src_flags, size_t n, cudaStream_t stream,
                                 int device) {
    rp::GatherParams G;
    G.store_bases = static_cast<const uint8_t*>(reads->d_bases.p);
    G.store_quals = weights ? static_cast<const uint8_t*>(reads->d_quals.p) : nullptr;
    G.bases = static_cast<uint8_t*>(bases);
    G.weights = static_cast<uint8_t*>(weights);
    G.seq_off = seq_off;
    G.src_pos = src_pos;
    G.src_flags = src_flags;
    G.n_seqs = static_cast<uint32_t>(n);
    return launch(rp_gather_kernel, gather_blocks(device, G.n_seqs), 256, 0, stream, G);
}

struct rp_aln : StreamOwner {
    rp::AlnParams P;
    PinnedBuf<uint8_t> bases;
    PinnedBuf<uint32_t> q_off, q_len, t_off, t_len, run_off, run_cap, queue, t_begin, q_start, bp_off, bp_cap;
    uint32_t window_length = 0;
    uint64_t bp_total = 0;
    std::vector<uint32_t> pre_status;      // per pair: soft status decided on the host (too long) or 0
    uint64_t run_total = 0;
    /* by-reference batches: both spans of every pair as slices of a device-resident store, gathered at upload */
    const rp_reads* reads = nullptr;
    bool by_ref = false;
    uint64_t n_bases = 0;              // == bases.size unless by_ref
    PinnedBuf<uint64_t> src_pos;     // two entries per pair: query, target
    PinnedBuf<uint8_t> src_flags;
    PinnedBuf<uint32_t> span_off;    // packed offsets of the 2 n spans, + total
    DevBuf d_src_pos, d_src_flags, d_span_off;
    DevBuf d_bases, d_q_off, d_q_len, d_t_off, d_t_len, d_run_off, d_run_cap, d_queue, d_runs, d_n_runs, d_dist,
        d_status, d_head, d_scratch, d_t_begin, d_q_start, d_bp_off, d_bp_cap, d_bp, d_n_bp;
    PinnedBuf<uint32_t> h_runs, h_n_runs, h_status, h_bp, h_n_bp;
    PinnedBuf<int32_t> h_dist;
    std::vector<std::string> cigars;
    std::vector<uint8_t> cigar_built;
    uint32_t workers = 0;
    int grid = 0;
    uint32_t max_len = 0;
    uint64_t max_bases = 0;
    bool uploaded = false, launched = false, downloaded = false, synced = false;
    uint64_t launches = 0, last_h2d = 0, last_d2h = 0;
    rp_aln() { std::memset(&P, 0, sizeof(P)); }
};

struct rp_poa : StreamOwner {
    rp::PackedBatch batch{&kPinned};
    rp::PoaParams P;
    /* device input buffers */
    DevBuf d_bases, d_weights, d_seq_flags, d_win_flags, d_seq_off, d_seq_begin, d_seq_end, d_win_first, d_out_off,
        d_out_cap, d_queue, d_win_alpha, d_cons, d_cov, d_len, d_status, d_head, d_stats, d_scratch;
    /* pinned results */
    PinnedBuf<uint8_t> h_cons;
    PinnedBuf<uint16_t> h_cov;
    PinnedBuf<uint32_t> h_len, h_status;
    uint64_t h_stats[8] = {0};
    uint32_t workers = 0;          // lane groups = windows in flight
    int grid = 0;
    uint32_t smem_block = 0;
    PoaKernel kernel = nullptr;
    int group = 32;                // lanes per window
    int band_k = 16;               // columns per lane of a banded row
    uint32_t groups_per_block = 4;
    bool uploaded = false, launched = false, downloaded = false, synced = false;
    bool counters = false;
    uint64_t launches = 0, last_h2d = 0, last_d2h = 0;
    int banded = 0;
    uint32_t configured_wl = 0;    // window length the scratch is sized for (0 = not yet: sized at the first upload)
    uint64_t h_band[4] = {0, 0, 0, 0};
    uint64_t band_total[3] = {0, 0, 0};   // sums of h_band over the object's life (RP_BAND_AUDIT report)
    bool band_counted = true;   // alignments tried in the band / redone with the full matrix (last launch)
    /* escalation pass for windows that exceeded a device limit (never a CPU re-run) */
    DevBuf d_scratch_big, d_queue_big;
    /* by-reference batches: the store the current batch's windows point into, and the device copy of the descriptors */
    const rp_reads* reads = nullptr;
    DevBuf d_src_pos, d_src_flags;
    uint64_t gather_launches = 0;
    rp::PoaLimits lim_big;
    rp::SlotLayout lay_big;
    uint32_t workers_big = 0;
    uint64_t escalated = 0;
    size_t mem_budget = 0;

    rp_poa() { std::memset(&P, 0, sizeof(P)); }
};

extern "C" {

static rp_status configure(rp_poa* p, uint32_t wl);
static rp_status aln_add_metadata(rp_aln* a, uint32_t ql, uint32_t tl, uint32_t t_begin, uint32_t q_start, bool too_long);

const char* rp_strerror(rp_status s) {
    switch (s) {
        case RP_OK: return "ok";
        case RP_BATCH_FULL: return "batch full";
        case RP_NOT_READY: return "not ready: the last run is still in flight";
        case RP_ERR_INVALID: return "invalid argument or malformed window";
        case RP_ERR_CUDA: return "CUDA error";
        case RP_ERR_NOMEM: return "out of memory";
        case RP_ERR_STATE: return "call order violated";
        case RP_ERR_NO_DEVICE: return "no CUDA device (this library has no CPU fallback)";
        default: return "unknown status";
    }
}

const char* rp_last_error(void) { return g_last_error.c_str(); }

const char* rp_version(void) { return "racon_b200 0.1 (sm_90a)"; }

int rp_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

rp_status rp_poa_create(rp_poa** out, int device, size_t mem_bytes, int8_t match, int8_t mismatch, int8_t gap,
                        int banded, uint32_t window_len_hint, uint32_t max_depth_hint) {
    (void)max_depth_hint;
    if (!out) return fail(RP_ERR_INVALID, "null out");
    *out = nullptr;
    if (gap > 0) return fail(RP_ERR_INVALID, "gap penalty must be non-positive (alignment_engine.cpp:47-51)");
    rp_poa* p = nullptr;
    const rp_status st = create_object(p, device);
    if (st != RP_OK) return st;
    p->banded = banded;
    rp::set_scores(p->P, match, mismatch, gap);
    p->P.banded = banded ? 1 : 0;   // the request; configure() decides whether the band layout is used (window length)
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    if (mem_bytes == 0 || mem_bytes > free_b) mem_bytes = static_cast<size_t>(free_b * 0.8);
    p->mem_budget = mem_bytes;
    /* batch limits from the budget (a quarter of it holds the batch's inputs and outputs on the device) */
    const uint64_t io_budget = mem_bytes / 4;
    p->batch.max_seq_len = 65000;
    p->batch.max_bases = std::min<uint64_t>(0xfff00000ull, std::max<uint64_t>(io_budget / 4, 1u << 16));
    p->batch.max_out = std::min<uint64_t>(0xfff00000ull, std::max<uint64_t>(io_budget / 8, 1u << 14));
    p->batch.max_windows = static_cast<uint32_t>(std::min<uint64_t>(1u << 22, std::max<uint64_t>(io_budget / 4096, 16)));
    cudaError_t e = p->d_head.reserve(256);
    if (e == cudaSuccess) e = p->d_stats.reserve(256);
    if (e != cudaSuccess) {
        rp_poa_destroy(p);
        return fail(RP_ERR_NOMEM, std::string("allocation: ") + cudaGetErrorString(e));
    }
    cudaMemsetAsync(p->d_stats.p, 0, 256, p->stream);
    /* window_len_hint == 0: the per-window scratch is sized at the first upload from the longest backbone seen
     * (racon's createCUDABatch does not pass -w, cudabatch.cpp:23-72) */
    if (window_len_hint) {
        rp_status cs = configure(p, window_len_hint);
        if (cs != RP_OK) {
            rp_poa_destroy(p);
            return cs;
        }
    }
    *out = p;
    return RP_OK;
}

/* Sizes the per-window limits, the launch shape and the workers' scratch for windows of length wl. */
static rp_status configure(rp_poa* p, uint32_t wl) {
    cudaError_t e = cudaSuccess;
    const size_t mem_bytes = p->mem_budget;
    const int banded = p->banded;
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, p->device);
    p->d_scratch.release();
    p->d_scratch_big.release();
    p->workers_big = 0;
    rp::PoaLimits lim;
    lim.nmax = std::min<uint32_t>(65000, std::max<uint32_t>(1024, 6 * wl + 64));
    lim.lmax = std::min<uint32_t>(16000, 2 * wl + 23);
    lim.lp = (lim.lmax + 1 + rp::kChunkCols - 1) / rp::kChunkCols * rp::kChunkCols;
    lim.ki = 16;
    lim.ka = 8;
    lim.stack_cap = lim.nmax * 4 + 64;
    p->P.band_margin = 16;
    if (const char* e_m = getenv("RP_BAND_MARGIN")) p->P.band_margin = static_cast<uint32_t>(atoi(e_m));
    /* tests only: recompute every accepted band result with the full matrix and count the differences */
    if (const char* e_a = getenv("RP_BAND_AUDIT")) p->P.debug_flags = atoi(e_a) ? 2u : 0u;

    /* launch shape: persistent blocks of 4 warps = 128/G lane groups, poa_blocks_per_sm blocks per SM.  Defaults measured
     * on the H100 (tools/tune_poa.py, 10 000 windows of bench config 2): full matrix: 32 lanes per window, 16 columns per
     * lane; banded (-b): 32 lanes x 8 columns = a 256-column band (the width of cudapoa's static band) — four packed
     * registers per row instead of eight.  RP_POA_BAND_K=4 selects a 128-column band (faster on clean data, refuses more
     * often). */
    int group = 32;
    if (const char* e_g = getenv("RP_POA_GROUP")) group = atoi(e_g);
    if (group != 8 && group != 16 && group != 32) group = 32;
    int band_k = (banded && group == 32) ? 8 : 16;
    if (const char* e_k = getenv("RP_POA_BAND_K")) band_k = atoi(e_k);
    if (group != 32 || (band_k != 4 && band_k != 8)) band_k = 16;
    /* -b is a request for speed with unchanged results.  Measured (profiles/README.md, round 2): for rows that fit one
     * 512-column chunk the full matrix is the faster kernel (a DP row's cost is mostly width-independent), the band
     * pays from two chunks per row on (w = 1000: 1.35x).  So a banded object uses the band when its windows are long
     * enough, or when the band layout is asked for explicitly (RP_POA_BAND_K / RP_POA_GROUP: tests, bench config 3). */
    const bool band_forced = getenv("RP_POA_BAND_K") != nullptr || getenv("RP_POA_GROUP") != nullptr;
    p->P.banded = (banded && (band_forced || wl >= kBandPaysFromWindowLength)) ? 1 : 0;
    if (!p->P.banded) band_k = 16;
    p->group = group;
    p->band_k = band_k;
    p->groups_per_block = kWarpsPerBlock * 32 / group;
    p->kernel = pick_kernel(group, band_k);
    uint32_t smem_per_sm = static_cast<uint32_t>(prop.sharedMemPerMultiprocessor);
    uint32_t per_block = smem_per_sm / poa_blocks_per_sm(band_k) - 1024;       // 1 KB reserved per block
    if (per_block > prop.sharedMemPerBlockOptin) per_block = static_cast<uint32_t>(prop.sharedMemPerBlockOptin);
    uint32_t per_group = (per_block / p->groups_per_block) & ~255u;
    p->P.smem_per_group = per_group;
    p->smem_block = per_group * p->groups_per_block;
    e = cudaFuncSetAttribute(p->kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(p->smem_block));
    int occ = 0;
    if (e == cudaSuccess)
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, p->kernel, kWarpsPerBlock * 32, p->smem_block);
    if (e != cudaSuccess || occ < 1)
        return fail(RP_ERR_CUDA, std::string("kernel configuration: ") + cudaGetErrorString(e));
    /* Device-memory budget of this object (cudabatch.cpp:23-72 passes 0.9 * free / batches): half for the
     * per-window scratch of the workers, a quarter for the lazily allocated escalation pass, a quarter for the
     * batch itself (inputs + outputs) — the batch limits below are what makes add_window return RP_BATCH_FULL. */
    const uint64_t max_workers = static_cast<uint64_t>(prop.multiProcessorCount) * occ * p->groups_per_block;
    const uint64_t scratch_budget = mem_bytes / 2;
    /* score-matrix scratch per window: the whole (nmax + 1) x padded-lmax matrix when the budget allows it for
     * every worker, otherwise down to what a window 4x deeper than its length needs (larger windows are re-run
     * by the escalation pass); only then fewer workers */
    const uint64_t hcap_full = static_cast<uint64_t>(lim.nmax + 1) * lim.lp;
    const uint64_t hcap_min = std::min<uint64_t>(
        hcap_full, static_cast<uint64_t>(4 * wl + 64) *
                       (((wl + wl / 4 + wl / 32 + 1) + 16 * group - 1) / (16 * group) * (16 * group)));
    lim.hcap = 0;
    const uint64_t fixed_bytes = rp::make_layout(lim).bytes;
    uint64_t hcap = hcap_full;
    if (max_workers * (fixed_bytes + hcap * 2) > scratch_budget) {
        const uint64_t per = scratch_budget / max_workers;
        hcap = per > fixed_bytes + 4096 ? (per - fixed_bytes - 4096) / 2 : 0;
        hcap = std::max(hcap_min, std::min(hcap, hcap_full));
    }
    lim.hcap = static_cast<uint32_t>(std::min<uint64_t>(hcap, 0xfffffff0ull));
    p->P.lim = lim;
    p->P.lay = rp::make_layout(lim);
    uint64_t fit = scratch_budget / p->P.lay.bytes;
    if (fit < p->groups_per_block) return fail(RP_ERR_NOMEM, "memory budget too small for one block of POA workers");
    uint64_t workers = std::min(max_workers, fit) / p->groups_per_block * p->groups_per_block;
    p->workers = static_cast<uint32_t>(workers);
    p->grid = static_cast<int>(workers / p->groups_per_block);
    e = p->d_scratch.reserve(workers * p->P.lay.bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(RP_ERR_NOMEM, std::string("scratch allocation: ") + cudaGetErrorString(e));
    }
    p->lim_big = lim;
    p->lim_big.nmax = std::min<uint32_t>(65000, lim.nmax * 8);
    p->lim_big.lmax = std::min<uint32_t>(16000, lim.lmax * 4);
    p->lim_big.lp = (p->lim_big.lmax + 1 + rp::kChunkCols - 1) / rp::kChunkCols * rp::kChunkCols;
    p->lim_big.ki = 96;
    p->lim_big.ka = 8;
    p->lim_big.stack_cap = p->lim_big.nmax * 6 + 64;
    p->lim_big.hcap = static_cast<uint32_t>(
        std::min<uint64_t>(0xfffffff0ull, static_cast<uint64_t>(p->lim_big.nmax + 1) * p->lim_big.lp));
    p->lay_big = rp::make_layout(p->lim_big);
    p->configured_wl = wl;
    return RP_OK;
}

void rp_poa_destroy(rp_poa* p) {
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->stream) cudaStreamSynchronize(p->stream);
    if (p->banded && getenv("RP_BAND_AUDIT"))   // test mode: what the band did over this object's life
        fprintf(stderr, "[racon_b200] band %u columns: %llu alignments tried, %llu redone with the full matrix, %llu accepted "
                        "band alignments differ from the full-matrix alignment (audit)\n",
                static_cast<unsigned>(p->group * p->band_k), static_cast<unsigned long long>(p->band_total[0]),
                static_cast<unsigned long long>(p->band_total[1]), static_cast<unsigned long long>(p->band_total[2]));
    delete p;   // frees the device buffers, then destroys the object's own stream
}

rp_status rp_poa_set_stream(rp_poa* p, void* cuda_stream) { return set_stream(p, cuda_stream); }

static rp_status map_pack(int r) {
    switch (r) {
        case rp::kPackOk: return RP_OK;
        case rp::kPackFull: return RP_BATCH_FULL;
        case rp::kPackNoMem: return fail(RP_ERR_NOMEM, "pinned staging allocation failed");
        default: return fail(RP_ERR_INVALID, "malformed window (see Window::add_layer checks, window.cpp:42-63)");
    }
}

rp_status rp_poa_add_window(rp_poa* p, uint32_t n_seq, const char* const* seq, const uint32_t* len,
                            const char* const* qual, const uint32_t* begin, const uint32_t* end, int window_type,
                            int trim) {
    if (!p) return fail(RP_ERR_INVALID, "null object");
    if (p->uploaded) return fail(RP_ERR_STATE, "batch already uploaded; reset first");
    if (p->batch.by_ref) return fail(RP_ERR_STATE, "this batch holds windows added by reference; reset first");
    return map_pack(p->batch.add(n_seq, seq, len, qual, begin, end, window_type, trim));
}

rp_status rp_reads_create(rp_reads** out, int device, uint32_t n_seqs, const char* const* data,
                          const char* const* quality, const uint32_t* length) {
    if (!out) return fail(RP_ERR_INVALID, "null out");
    *out = nullptr;
    if (!data || !length) return fail(RP_ERR_INVALID, "null argument");
    const rp_status s = check_device(device);
    if (s != RP_OK) return s;
    rp_reads* r = new (std::nothrow) rp_reads();
    if (!r) return fail(RP_ERR_NOMEM, "host allocation failed");
    r->device = device;
    r->data.assign(data, data + n_seqs);
    r->quality.assign(n_seqs, nullptr);
    r->length.assign(length, length + n_seqs);
    r->off.assign(n_seqs + 1, 0);
    r->chars.assign(n_seqs, std::array<uint64_t, 4>{0, 0, 0, 0});
    for (uint32_t i = 0; i < n_seqs; ++i) {
        if (length[i] && !data[i]) {
            delete r;
            return fail(RP_ERR_INVALID, "null sequence");
        }
        if (quality && quality[i] && length[i]) {
            r->quality[i] = quality[i];
            r->any_quality = true;
        }
        r->off[i + 1] = r->off[i] + length[i];
        uint8_t seen[256];
        std::memset(seen, 0, sizeof(seen));
        rp::PackedBatch::scan_alphabet(reinterpret_cast<const uint8_t*>(data[i]), length[i], seen);
        if (seen[0]) {
            delete r;
            return fail(RP_ERR_INVALID, "NUL byte in a sequence");
        }
        for (uint32_t c = 1; c < 256; ++c)
            if (seen[c]) r->chars[i][c >> 6] |= 1ull << (c & 63);
    }
    const uint64_t total = r->off[n_seqs];
    cudaError_t e = r->d_bases.reserve(total + 16);
    if (e == cudaSuccess && r->any_quality) e = r->d_quals.reserve(total + 16);
    /* the caller's sequences are separate pageable strings: stage them through pinned memory in large pieces */
    const size_t stage_bytes = static_cast<size_t>(std::min<uint64_t>(std::max<uint64_t>(total, 1), 64ull << 20));
    void* stage = nullptr;
    if (e == cudaSuccess) e = cudaHostAlloc(&stage, stage_bytes, cudaHostAllocDefault);
    if (e != cudaSuccess) {
        cudaGetLastError();
        delete r;
        return fail(RP_ERR_NOMEM, std::string("read store allocation: ") + cudaGetErrorString(e));
    }
    cudaStream_t st = nullptr;
    e = cudaStreamCreate(&st);
    for (int pass = 0; pass < 2 && e == cudaSuccess; ++pass) {
        if (pass == 1 && !r->any_quality) break;
        uint8_t* dst = static_cast<uint8_t*>(pass == 0 ? r->d_bases.p : r->d_quals.p);
        uint64_t flushed = 0, filled = 0;   // device positions: [flushed, filled) sits in the staging buffer
        auto flush = [&]() {
            if (filled > flushed) {
                e = cudaMemcpyAsync(dst + flushed, stage, filled - flushed, cudaMemcpyHostToDevice, st);
                if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            }
            flushed = filled;
        };
        for (uint32_t i = 0; i < n_seqs && e == cudaSuccess; ++i) {
            const char* src = pass == 0 ? r->data[i] : r->quality[i];
            uint64_t done = 0;
            while (done < length[i] && e == cudaSuccess) {
                if (filled - flushed == stage_bytes) flush();
                const uint64_t n = std::min<uint64_t>(length[i] - done, stage_bytes - (filled - flushed));
                if (src) {
                    std::memcpy(static_cast<uint8_t*>(stage) + (filled - flushed), src + done, n);
                } else {
                    std::memset(static_cast<uint8_t*>(stage) + (filled - flushed), '!', n);
                }
                filled += n;
                done += n;
            }
        }
        if (e == cudaSuccess) flush();
    }
    if (st) cudaStreamDestroy(st);
    cudaFreeHost(stage);
    if (e != cudaSuccess) {
        delete r;
        return fail(RP_ERR_CUDA, std::string("read store upload: ") + cudaGetErrorString(e));
    }
    *out = r;
    return RP_OK;
}

void rp_reads_destroy(rp_reads* r) {
    if (!r) return;
    cudaSetDevice(r->device);
    delete r;
}

uint64_t rp_reads_bytes(const rp_reads* r) { return r ? r->d_bases.cap + r->d_quals.cap : 0; }

rp_status rp_poa_add_window_refs(rp_poa* p, const rp_reads* reads, uint32_t n_seq, const uint32_t* seq_id,
                                 const uint32_t* offset, const uint32_t* length, const uint8_t* reverse,
                                 const uint32_t* begin, const uint32_t* end, int window_type, int trim) {
    if (!p || !reads || !seq_id || !offset || !length || !begin || !end) return fail(RP_ERR_INVALID, "null argument");
    if (p->uploaded) return fail(RP_ERR_STATE, "batch already uploaded; reset first");
    if (reads->device != p->device) return fail(RP_ERR_INVALID, "the read store lives on another device");
    rp::PackedBatch& b = p->batch;
    if (b.n_added() > 0 && (!b.by_ref || p->reads != reads))
        return fail(RP_ERR_STATE, "a batch holds windows added by pointer or by reference into ONE store; reset first");
    if (n_seq == 0) return fail(RP_ERR_INVALID, "malformed window (see Window::add_layer checks, window.cpp:42-63)");
    const uint32_t n_store = static_cast<uint32_t>(reads->length.size());
    for (uint32_t k = 0; k < n_seq; ++k) {
        if (seq_id[k] >= n_store || static_cast<uint64_t>(offset[k]) + length[k] > reads->length[seq_id[k]])
            return fail(RP_ERR_INVALID, "window piece outside its sequence");
    }
    if (reverse && reverse[0]) return fail(RP_ERR_INVALID, "the backbone cannot be a reverse-complement piece");
    rp::PackedBatch::Prep pr;
    rp::PackedBatch::prepare_layout(pr, n_seq, nullptr, length, begin, end, b.max_seq_len);
    if (pr.status == rp::kPackOk && pr.kind == 0) {
        /* alphabet: union of the characters of the pieces' sequences (a superset of the window's own, which only matters
         * when it has more than the 8 codes the device holds: then the pieces themselves are scanned) */
        std::array<uint64_t, 4> set{0, 0, 0, 0};
        auto swap_bits = [](std::array<uint64_t, 4>& m, uint8_t a, uint8_t c) {
            const bool ha = m[a >> 6] >> (a & 63) & 1, hc = m[c >> 6] >> (c & 63) & 1;
            if (ha != hc) {
                m[a >> 6] ^= 1ull << (a & 63);
                m[c >> 6] ^= 1ull << (c & 63);
            }
        };
        for (uint32_t k : pr.order) {
            std::array<uint64_t, 4> m = reads->chars[seq_id[k]];
            if (reverse && reverse[k]) {
                swap_bits(m, 'A', 'T');
                swap_bits(m, 'C', 'G');
            }
            for (int i = 0; i < 4; ++i) set[i] |= m[i];
        }
        uint8_t seen[256];
        int distinct = 0;
        for (uint32_t c = 0; c < 256; ++c) distinct += seen[c] = set[c >> 6] >> (c & 63) & 1;
        if (distinct > 8) {
            std::memset(seen, 0, sizeof(seen));
            for (uint32_t k : pr.order) {
                const uint32_t len_k = reads->length[seq_id[k]];
                const bool rev = reverse && reverse[k];
                const uint8_t* piece = reinterpret_cast<const uint8_t*>(reads->data[seq_id[k]]) +
                                       (rev ? len_k - offset[k] - length[k] : offset[k]);
                uint8_t local[256];
                std::memset(local, 0, sizeof(local));
                rp::PackedBatch::scan_alphabet(piece, length[k], local);
                for (uint32_t c = 0; c < 256; ++c)
                    if (local[c]) seen[rev ? rp::complement_base(static_cast<uint8_t>(c)) : c] = 1;
            }
        }
        rp::PackedBatch::alphabet_from_seen(pr, seen);
    }
    const bool was_empty = b.n_added() == 0;
    if (was_empty) b.by_ref = true;
    const char* backbone = reads->data[seq_id[0]] + offset[0];
    const int rc = b.commit(pr, &backbone, length, begin, end, window_type, trim);
    if (rc != rp::kPackOk) {
        if (was_empty) b.by_ref = false;
        return map_pack(rc);
    }
    p->reads = reads;
    if (pr.kind == 0) {
        for (size_t i = 0; i < pr.order.size(); ++i) {
            const uint32_t k = pr.order[i];
            const uint32_t id = seq_id[k];
            const bool rev = reverse && reverse[k];
            b.src_pos.push(reads->off[id] + (rev ? reads->length[id] - 1 - offset[k] : offset[k]));
            b.src_flags.push(static_cast<uint8_t>((rev ? rp::kSrcReverse : 0) | (reads->quality[id] ? rp::kSrcHasQuality : 0) |
                                                  (i == 0 ? rp::kSrcBackbone : 0)));
        }
    }
    return RP_OK;
}

rp_status rp_poa_add_window_set_refs(rp_poa* p, const rp_reads* reads, uint32_t first, uint32_t count,
                                     const uint32_t* seq_id, const uint32_t* offset, const uint32_t* length,
                                     const uint8_t* reverse, const uint32_t* begin, const uint32_t* end,
                                     const uint32_t* win_first, const uint8_t* win_type, int trim, uint32_t* added) {
    if (!win_first || !seq_id || !offset || !length || !begin || !end) return fail(RP_ERR_INVALID, "null argument");
    if (added) *added = 0;
    uint32_t n = 0;
    rp_status st = RP_OK;
    for (; n < count; ++n) {
        const uint32_t s0 = win_first[first + n], s1 = win_first[first + n + 1];
        st = rp_poa_add_window_refs(p, reads, s1 - s0, seq_id + s0, offset + s0, length + s0, reverse ? reverse + s0 : nullptr,
                                    begin + s0, end + s0, win_type ? win_type[first + n] : 1, trim);
        if (st != RP_OK) break;
    }
    if (added) *added = n;
    return st == RP_BATCH_FULL && n > 0 ? RP_OK : st;
}

rp_status rp_poa_add_window_set(rp_poa* p, uint32_t first, uint32_t count, const char* bases, const char* quals,
                                const uint64_t* seq_off, const uint8_t* seq_has_qual, const uint32_t* seq_begin,
                                const uint32_t* seq_end, const uint32_t* win_first, const uint8_t* win_type, int trim,
                                uint32_t* added) {
    if (!p || !bases || !seq_off || !win_first || !seq_begin || !seq_end)
        return fail(RP_ERR_INVALID, "null argument");
    if (p->uploaded) return fail(RP_ERR_STATE, "batch already uploaded; reset first");
    if (p->batch.by_ref) return fail(RP_ERR_STATE, "this batch holds windows added by reference; reset first");
    if (added) *added = 0;
    if (count == 0) return RP_OK;
    /* per-window pointer tables (the flat set stores offsets) */
    const uint32_t sbase = win_first[first];
    const uint32_t nseq = win_first[first + count] - sbase;
    std::vector<const char*> sp(nseq), qp(nseq);
    std::vector<uint32_t> ln(nseq);
    const bool any_q = quals && seq_has_qual;
    /* host threads for the byte-heavy packing steps: the machine's threads are shared by every rank of the node
     * (LOCAL_WORLD_SIZE, set by torchrun) and by every batch object a caller drives concurrently — more packers than
     * hardware threads only slow each other down (round 1: 8 ranks x 32 packers on 128 threads) */
    unsigned hw = std::thread::hardware_concurrency();
    unsigned share = 1;
    if (const char* lw = getenv("LOCAL_WORLD_SIZE")) share = std::max(1, atoi(lw));
    unsigned cap = 32;
    if (const char* pt = getenv("RP_PACK_THREADS")) cap = std::max(1, atoi(pt));
    const unsigned fair = std::max(1u, (hw ? hw : 1u) / share / 2);
    const unsigned nthreads = std::max(1u, std::min(std::min(fair, cap), count / 64 + 1));
    std::vector<rp::PackedBatch::Prep> preps(count);
    const uint32_t max_len = p->batch.max_seq_len;
    auto prep_range = [&](uint32_t a, uint32_t b) {
        for (uint32_t w = a; w < b; ++w) {
            const uint32_t s0 = win_first[first + w], s1 = win_first[first + w + 1];
            for (uint32_t s = s0; s < s1; ++s) {
                sp[s - sbase] = bases + seq_off[s];
                qp[s - sbase] = (any_q && seq_has_qual[s]) ? quals + seq_off[s] : nullptr;
                ln[s - sbase] = static_cast<uint32_t>(seq_off[s + 1] - seq_off[s]);
            }
            rp::PackedBatch::prepare(preps[w], s1 - s0, sp.data() + (s0 - sbase), ln.data() + (s0 - sbase),
                                     seq_begin + s0, seq_end + s0, max_len);
        }
    };
    auto run_parallel = [&](const std::function<void(uint32_t, uint32_t)>& fn, uint32_t n) {
        if (nthreads <= 1 || n < 128) {
            fn(0, n);
            return;
        }
        std::vector<std::thread> pool;
        const uint32_t step = (n + nthreads - 1) / nthreads;
        for (uint32_t a = 0; a < n; a += step) pool.emplace_back(fn, a, std::min(n, a + step));
        for (auto& t : pool) t.join();
    };
    run_parallel(prep_range, count);
    /* serial commit: reserves space, writes metadata; stops at the first window that does not fit */
    uint32_t n = 0;
    rp_status st = RP_OK;
    for (; n < count; ++n) {
        const uint32_t s0 = win_first[first + n];
        st = map_pack(p->batch.commit(preps[n], sp.data() + (s0 - sbase), ln.data() + (s0 - sbase), seq_begin + s0,
                                      seq_end + s0, win_type ? win_type[first + n] : 1, trim));
        if (st != RP_OK) break;
    }
    auto fill_range = [&](uint32_t a, uint32_t b) {
        for (uint32_t w = a; w < b; ++w) {
            const uint32_t s0 = win_first[first + w];
            p->batch.fill(preps[w], sp.data() + (s0 - sbase), ln.data() + (s0 - sbase), qp.data() + (s0 - sbase));
        }
    };
    run_parallel(fill_range, n);
    if (added) *added = n;
    return st == RP_BATCH_FULL && n > 0 ? RP_OK : st;
}

uint32_t rp_poa_size(const rp_poa* p) { return p ? p->batch.n_added() : 0; }

rp_status rp_poa_upload(rp_poa* p) {
    if (!p) return fail(RP_ERR_INVALID, "null object");
    RP_CUDA(cudaSetDevice(p->device));
    rp::PackedBatch& b = p->batch;
    if (!b.build_queue()) return fail(RP_ERR_NOMEM, "queue allocation failed");
    const uint32_t n = b.n_gpu();
    if (!p->configured_wl) {
        uint32_t wl = 0;
        for (uint32_t w = 0; w < n; ++w) {
            const uint32_t s0 = b.win_first.data[w];
            wl = std::max(wl, b.seq_off.data[s0 + 1] - b.seq_off.data[s0]);
        }
        wl = std::max<uint32_t>(100, (wl + 99) / 100 * 100);
        rp_status cs = configure(p, wl);
        if (cs != RP_OK) return cs;
    }
    rp::PoaParams& P = p->P;
    const uint64_t* src_pos = nullptr;
    const uint8_t* src_flags = nullptr;
    p->last_h2d = 0;
    if (b.by_ref) {
        RP_CUDA(reserve(p->d_bases, b.n_bases + 16, P.bases));
        RP_CUDA(reserve(p->d_weights, b.n_bases + 16, P.weights));
        RP_CUDA(upload(p, p->d_src_pos, b.src_pos, src_pos));
        RP_CUDA(upload(p, p->d_src_flags, b.src_flags, src_flags));
    } else {
        RP_CUDA(upload(p, p->d_bases, b.bases, P.bases));
        RP_CUDA(upload(p, p->d_weights, b.weights, P.weights));
    }
    RP_CUDA(upload(p, p->d_seq_off, b.seq_off, P.seq_off));
    RP_CUDA(upload(p, p->d_seq_begin, b.seq_begin, P.seq_begin));
    RP_CUDA(upload(p, p->d_seq_end, b.seq_end, P.seq_end));
    RP_CUDA(upload(p, p->d_seq_flags, b.seq_flags, P.seq_flags));
    RP_CUDA(upload(p, p->d_win_first, b.win_first, P.win_first));
    RP_CUDA(upload(p, p->d_win_flags, b.win_flags, P.win_flags));
    RP_CUDA(upload(p, p->d_win_alpha, b.win_alpha, P.win_alpha));
    RP_CUDA(upload(p, p->d_out_off, b.out_off, P.out_off));
    RP_CUDA(upload(p, p->d_out_cap, b.out_cap, P.out_cap));
    RP_CUDA(upload(p, p->d_queue, b.queue, P.queue));
    RP_CUDA(reserve(p->d_cons, b.out_total + 16, P.cons));
    RP_CUDA(reserve(p->d_cov, (b.out_total + 16) * 2, P.cons_cov));
    RP_CUDA(reserve(p->d_len, (n + 1) * 4, P.cons_len));
    RP_CUDA(reserve(p->d_status, (n + 1) * 4, P.status));
    if (!p->h_cons.reserve(b.out_total + 16) || !p->h_cov.reserve(b.out_total + 16) || !p->h_len.reserve(n + 1) ||
        !p->h_status.reserve(n + 1))
        return fail(RP_ERR_NOMEM, "pinned result allocation failed");
    P.n_windows = n;
    P.queue_head = static_cast<uint32_t*>(p->d_head.p);
    P.stats = p->counters ? static_cast<uint64_t*>(p->d_stats.p) : nullptr;
    P.scratch = static_cast<uint8_t*>(p->d_scratch.p);
    if (b.by_ref && b.src_pos.size > 0) {
        /* layer extraction on the device: fills d_bases / d_weights from the store, on this object's stream, ahead of the
         * POA kernel */
        RP_CUDA(launch_gather(p->reads, p->d_bases.p, p->d_weights.p, P.seq_off, src_pos, src_flags, b.src_pos.size,
                              p->stream, p->device));
        p->gather_launches += 1;
    }
    p->uploaded = true;
    p->launched = p->downloaded = p->synced = false;
    return RP_OK;
}

rp_status rp_poa_launch(rp_poa* p) {
    if (!p) return fail(RP_ERR_INVALID, "null object");
    if (!p->uploaded) return fail(RP_ERR_STATE, "launch before upload");
    RP_CUDA(cudaSetDevice(p->device));
    if (p->P.n_windows > 0) {
        RP_CUDA(cudaMemsetAsync(p->d_head.p, 0, 4, p->stream));
        /* the DP counters [0, 64) and the band counters [128, 160) count this launch alone */
        RP_CUDA(cudaMemsetAsync(p->d_stats.p, 0, 160, p->stream));
        p->P.stats = p->counters ? static_cast<uint64_t*>(p->d_stats.p) : nullptr;
        p->P.band_stats = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(p->d_stats.p) + 128);
        const uint32_t need_blocks = (p->P.n_windows + p->groups_per_block - 1) / p->groups_per_block;
        const uint32_t blocks = std::min<uint32_t>(static_cast<uint32_t>(p->grid), need_blocks);
        RP_CUDA(launch(p->kernel, blocks, kWarpsPerBlock * 32, p->smem_block, p->stream, p->P));
        p->launches += 1;
    }
    p->launched = true;
    p->downloaded = p->synced = false;
    return RP_OK;
}

/* queues the copies of the results of the batch's n GPU windows (consensus, coverage, lengths, statuses) to pinned memory */
static rp_status read_results(rp_poa* p, uint32_t n) {
    const size_t tot = p->batch.out_total;
    RP_CUDA(cudaMemcpyAsync(p->h_cons.data, p->d_cons.p, tot, cudaMemcpyDeviceToHost, p->stream));
    RP_CUDA(cudaMemcpyAsync(p->h_cov.data, p->d_cov.p, tot * 2, cudaMemcpyDeviceToHost, p->stream));
    RP_CUDA(cudaMemcpyAsync(p->h_len.data, p->d_len.p, n * 4, cudaMemcpyDeviceToHost, p->stream));
    RP_CUDA(cudaMemcpyAsync(p->h_status.data, p->d_status.p, n * 4, cudaMemcpyDeviceToHost, p->stream));
    return RP_OK;
}

rp_status rp_poa_download(rp_poa* p) {
    if (!p) return fail(RP_ERR_INVALID, "null object");
    if (!p->launched) return fail(RP_ERR_STATE, "download before launch");
    RP_CUDA(cudaSetDevice(p->device));
    const uint32_t n = p->P.n_windows;
    uint64_t d2h = 0;
    if (n > 0) {
        const rp_status s = read_results(p, n);
        if (s != RP_OK) return s;
        d2h = p->batch.out_total * 3 + static_cast<uint64_t>(n) * 8;
    }
    if (p->counters && n > 0)
        RP_CUDA(cudaMemcpyAsync(p->h_stats, p->d_stats.p, 64, cudaMemcpyDeviceToHost, p->stream));
    else
        std::memset(p->h_stats, 0, sizeof(p->h_stats));
    if (p->banded && n > 0)
    {
        RP_CUDA(cudaMemcpyAsync(p->h_band, static_cast<uint8_t*>(p->d_stats.p) + 128, 32, cudaMemcpyDeviceToHost,
                                p->stream));
        p->band_counted = false;
    }
    p->last_d2h = d2h;
    p->downloaded = true;
    p->synced = false;
    return RP_OK;
}

rp_status rp_poa_run(rp_poa* p) {
    rp_status s = rp_poa_upload(p);
    if (s != RP_OK) return s;
    s = rp_poa_launch(p);
    if (s != RP_OK) return s;
    return rp_poa_download(p);
}

/* Windows whose graph outgrew the default per-window limits (very deep coverage, very long layers) are run
 * again ON THE GPU with 8x the node budget (lim_big.nmax, the only node limit of this pass in every layout: add_alignment
 * keeps its order counters in HBM when the group's shared memory is too small), 4x the layer length and 96 in-edge
 * slots, on a smaller set of workers (the reference hands such windows to the CPU, cudapolisher.cpp:354-370; this library has no CPU path). */
static rp_status escalate(rp_poa* p) {
    const uint32_t n = p->P.n_windows;
    std::vector<uint32_t> redo;
    for (uint32_t w = 0; w < n; ++w) {
        uint32_t st = p->h_status.data[w];
        if (st == rp::kWinNodeLimit || st == rp::kWinEdgeLimit || st == rp::kWinSeqTooLong ||
            st == rp::kWinStackLimit || st == rp::kWinMatrixLimit)
            redo.push_back(w);
    }
    if (redo.empty()) return RP_OK;
    if (p->workers_big == 0) {
        uint64_t fit = (p->mem_budget / 4) / p->lay_big.bytes;
        uint64_t workers = std::min<uint64_t>(p->workers, fit) / p->groups_per_block * p->groups_per_block;
        if (workers < p->groups_per_block) return RP_OK;  // no room: the soft status stays
        cudaError_t e = p->d_scratch_big.reserve(workers * p->lay_big.bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return RP_OK;
        }
        p->workers_big = static_cast<uint32_t>(workers);
    }
    RP_CUDA(p->d_queue_big.reserve(redo.size() * 4));
    RP_CUDA(cudaMemcpyAsync(p->d_queue_big.p, redo.data(), redo.size() * 4, cudaMemcpyHostToDevice, p->stream));
    RP_CUDA(cudaMemsetAsync(p->d_head.p, 0, 4, p->stream));
    rp::PoaParams P = p->P;
    P.n_windows = static_cast<uint32_t>(redo.size());
    P.queue = static_cast<const uint32_t*>(p->d_queue_big.p);
    P.scratch = static_cast<uint8_t*>(p->d_scratch_big.p);
    P.lim = p->lim_big;
    P.lay = p->lay_big;
    P.stats = nullptr;
    P.banded = 0;
    P.band_stats = nullptr;
    uint32_t blocks = std::min<uint32_t>(p->workers_big / p->groups_per_block,
                                         (static_cast<uint32_t>(redo.size()) + p->groups_per_block - 1) / p->groups_per_block);
    RP_CUDA(launch(p->kernel, blocks, kWarpsPerBlock * 32, p->smem_block, p->stream, P));
    p->launches += 1;
    p->escalated += redo.size();
    const rp_status s = read_results(p, n);
    if (s != RP_OK) return s;
    RP_CUDA(cudaStreamSynchronize(p->stream));
    return RP_OK;
}

rp_status rp_poa_sync(rp_poa* p) {
    if (!p) return fail(RP_ERR_INVALID, "null object");
    RP_CUDA(cudaSetDevice(p->device));
    RP_CUDA(cudaStreamSynchronize(p->stream));
    if (p->downloaded && !p->synced) {
        rp_status s = escalate(p);
        if (s != RP_OK) return s;
        p->synced = true;
        if (p->banded && !p->band_counted) {
            for (int k = 0; k < 3; ++k) p->band_total[k] += p->h_band[k];
            p->band_counted = true;
        }
    }
    return RP_OK;
}

rp_status rp_poa_query(rp_poa* p) { return query_stream(p, p && p->launched); }

static rp_status ensure_results(rp_poa* p) {
    if (!p) return fail(RP_ERR_INVALID, "null object");
    if (!p->downloaded) return fail(RP_ERR_STATE, "fetch before run/download");
    if (!p->synced) return rp_poa_sync(p);
    return RP_OK;
}

rp_status rp_poa_fetch(rp_poa* p, uint32_t i, const char** consensus, uint32_t* len, const uint16_t** coverage,
                       int* polished) {
    rp_status s = ensure_results(p);
    if (s != RP_OK) return s;
    if (i >= p->batch.n_added()) return fail(RP_ERR_INVALID, "window index out of range");
    int32_t gi = p->batch.gpu_index[i];
    if (gi < 0) {
        const std::string& c = p->batch.trivial[i];
        if (consensus) *consensus = c.data();
        if (len) *len = static_cast<uint32_t>(c.size());
        if (coverage) *coverage = nullptr;
        if (polished) *polished = 0;
        return RP_OK;
    }
    uint32_t off = p->batch.out_off.data[gi];
    bool ok = p->h_status.data[gi] == rp::kWinOk;
    if (consensus) *consensus = reinterpret_cast<const char*>(p->h_cons.data + off);
    if (len) *len = ok ? p->h_len.data[gi] : 0;
    if (coverage) *coverage = p->h_cov.data + off;
    if (polished) *polished = ok ? 1 : 0;
    return RP_OK;
}

rp_status rp_poa_window_status(rp_poa* p, uint32_t i, uint32_t* status) {
    rp_status s = ensure_results(p);
    if (s != RP_OK) return s;
    if (i >= p->batch.n_added() || !status) return fail(RP_ERR_INVALID, "window index out of range");
    int32_t gi = p->batch.gpu_index[i];
    *status = gi == -1 ? RP_WIN_OK : (gi == -2 ? RP_WIN_ALPHABET_LIMIT : p->h_status.data[gi]);
    return RP_OK;
}

rp_status rp_poa_fetch_all(rp_poa* p, char* out, uint32_t stride, uint32_t* lens, uint8_t* polished,
                           uint32_t* status) {
    rp_status s = ensure_results(p);
    if (s != RP_OK) return s;
    const uint32_t n = p->batch.n_added();
    for (uint32_t i = 0; i < n; ++i) {
        const char* c = nullptr;
        uint32_t l = 0;
        int pol = 0;
        uint32_t st = 0;
        rp_poa_fetch(p, i, &c, &l, nullptr, &pol);
        rp_poa_window_status(p, i, &st);
        if (out) {
            if (l > stride) return fail(RP_ERR_INVALID, "stride too small for a consensus");
            std::memcpy(out + static_cast<uint64_t>(i) * stride, c, l);
        }
        if (lens) lens[i] = l;
        if (polished) polished[i] = static_cast<uint8_t>(pol);
        if (status) status[i] = st;
    }
    return RP_OK;
}

rp_status rp_poa_reset(rp_poa* p) {
    if (!p) return fail(RP_ERR_INVALID, "null object");
    cudaSetDevice(p->device);
    if (p->stream) RP_CUDA(cudaStreamSynchronize(p->stream));
    p->batch.reset();
    p->uploaded = p->launched = p->downloaded = p->synced = false;
    return RP_OK;
}

rp_status rp_poa_info(rp_poa* p, uint64_t info[8]) {
    if (!p || !info) return fail(RP_ERR_INVALID, "null argument");
    info[0] = p->launches;
    info[1] = p->last_h2d;
    info[2] = p->last_d2h;
    info[3] = p->workers;
    info[4] = p->P.lay.bytes;
    info[5] = p->h_stats[0];
    info[6] = p->h_stats[1];
    info[7] = p->h_stats[3];
    return RP_OK;
}

rp_status rp_poa_band_info(rp_poa* p, uint64_t info[8]) {
    if (!p || !info) return fail(RP_ERR_INVALID, "null argument");
    rp_status s = ensure_results(p);
    if (s != RP_OK) return s;
    std::memset(info, 0, 8 * sizeof(uint64_t));
    info[0] = p->banded ? 1 : 0;
    info[5] = p->P.banded ? 1 : 0;   // the band layout is in use for this object's window length
    info[1] = p->h_band[0];
    info[2] = p->h_band[1];
    info[3] = static_cast<uint64_t>(p->group) * p->band_k;
    info[4] = p->h_band[2];
    return RP_OK;
}

rp_status rp_poa_enable_counters(rp_poa* p, int on) {
    if (!p) return fail(RP_ERR_INVALID, "null object");
    p->counters = on != 0;
    return RP_OK;
}


/* ---------------------------------------------------------------------------------------------------------
 * pre-alignment batch (racon::CUDABatchAligner shape)
 * --------------------------------------------------------------------------------------------------------- */
rp_status rp_aln_create(rp_aln** out, int device, size_t mem_bytes, uint32_t max_len) {
    if (!out) return fail(RP_ERR_INVALID, "null out");
    *out = nullptr;
    rp_aln* a = nullptr;
    const rp_status st = create_object(a, device);
    if (st != RP_OK) return st;
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    if (mem_bytes == 0 || mem_bytes > free_b) mem_bytes = static_cast<size_t>(free_b * 0.4);
    a->max_len = max_len ? max_len : 65536;
    a->P.lim.max_len = a->max_len;
    a->P.lim.store_words = 53000;  // > 1 MiB / 20 B: the largest base case edlib's rule allows
    a->P.lay = rp::make_aln_layout(a->P.lim);
    int occ = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rp_aln_kernel, kWarpsPerBlock * 32, 0);
    if (e != cudaSuccess || occ < 1) {
        rp_aln_destroy(a);
        return fail(RP_ERR_CUDA, std::string("kernel configuration: ") + cudaGetErrorString(e));
    }
    uint64_t max_workers = static_cast<uint64_t>(prop.multiProcessorCount) * occ * kWarpsPerBlock;
    uint64_t fit = (mem_bytes / 2) / a->P.lay.bytes;
    uint64_t workers = std::min(max_workers, fit) / kWarpsPerBlock * kWarpsPerBlock;
    if (workers < kWarpsPerBlock) {
        rp_aln_destroy(a);
        return fail(RP_ERR_NOMEM, "memory budget too small for one block of aligner workers");
    }
    a->workers = static_cast<uint32_t>(workers);
    a->grid = static_cast<int>(workers / kWarpsPerBlock);
    a->max_bases = std::min<uint64_t>(0xfff00000ull, mem_bytes / 8);
    e = a->d_scratch.reserve(workers * a->P.lay.bytes);
    if (e == cudaSuccess) e = a->d_head.reserve(256);
    if (e != cudaSuccess) {
        rp_aln_destroy(a);
        return fail(RP_ERR_NOMEM, std::string("scratch allocation: ") + cudaGetErrorString(e));
    }
    *out = a;
    return RP_OK;
}

void rp_aln_destroy(rp_aln* a) {
    if (!a) return;
    cudaSetDevice(a->device);
    if (a->stream) cudaStreamSynchronize(a->stream);
    delete a;   // frees the device buffers, then destroys the object's own stream
}

rp_status rp_aln_set_stream(rp_aln* a, void* cuda_stream) { return set_stream(a, cuda_stream); }

rp_status rp_aln_set_window_length(rp_aln* a, uint32_t window_length) {
    if (!a) return fail(RP_ERR_INVALID, "null object");
    if (!a->pre_status.empty()) return fail(RP_ERR_STATE, "window length must be set on an empty batch");
    a->window_length = window_length;
    return RP_OK;
}

rp_status rp_aln_add(rp_aln* a, const char* q, uint32_t ql, const char* t, uint32_t tl) {
    return rp_aln_add_overlap(a, q, ql, t, tl, 0, 0);
}

rp_status rp_aln_add_overlap(rp_aln* a, const char* q, uint32_t ql, const char* t, uint32_t tl, uint32_t t_begin,
                             uint32_t q_start) {
    if (!a || (!q && ql) || (!t && tl)) return fail(RP_ERR_INVALID, "null argument");
    if (static_cast<uint64_t>(t_begin) + tl > 0xffffffffull || static_cast<uint64_t>(q_start) + ql > 0xffffffffull)
        return fail(RP_ERR_INVALID, "coordinates exceed 32 bits");
    if (a->uploaded) return fail(RP_ERR_STATE, "batch already uploaded; reset first");
    if (a->by_ref) return fail(RP_ERR_STATE, "this batch holds overlaps added by reference; reset first");
    const bool too_long = ql > a->max_len || tl > a->max_len;
    const uint64_t add = too_long ? 0 : static_cast<uint64_t>(ql) + tl;
    if (a->n_bases + add > a->max_bases) return RP_BATCH_FULL;
    if (!too_long) {
        uint8_t* b = a->bases.extend(add);
        if (!b) return fail(RP_ERR_NOMEM, "pinned staging allocation failed");
        std::memcpy(b, q, ql);
        std::memcpy(b + ql, t, tl);
    }
    return aln_add_metadata(a, ql, tl, t_begin, q_start, too_long);
}

rp_status rp_aln_add_overlap_ref(rp_aln* a, const rp_reads* reads, uint32_t q_id, uint32_t q_start, uint32_t q_len,
                                 int q_reverse, uint32_t t_id, uint32_t t_begin, uint32_t t_len) {
    if (!a || !reads) return fail(RP_ERR_INVALID, "null argument");
    if (a->uploaded) return fail(RP_ERR_STATE, "batch already uploaded; reset first");
    if (reads->device != a->device) return fail(RP_ERR_INVALID, "the read store lives on another device");
    if (!a->pre_status.empty() && (!a->by_ref || a->reads != reads))
        return fail(RP_ERR_STATE, "a batch holds overlaps added by pointer or by reference into ONE store; reset first");
    const uint32_t n_store = static_cast<uint32_t>(reads->length.size());
    if (q_id >= n_store || t_id >= n_store || static_cast<uint64_t>(q_start) + q_len > reads->length[q_id] ||
        static_cast<uint64_t>(t_begin) + t_len > reads->length[t_id])
        return fail(RP_ERR_INVALID, "overlap span outside its sequence");
    const bool too_long = q_len > a->max_len || t_len > a->max_len;
    const uint64_t add = too_long ? 0 : static_cast<uint64_t>(q_len) + t_len;
    if (a->n_bases + add > a->max_bases) return RP_BATCH_FULL;
    if (!a->src_pos.reserve(a->src_pos.size + 2) || !a->src_flags.reserve(a->src_flags.size + 2) ||
        !a->span_off.reserve(a->span_off.size + 3))
        return fail(RP_ERR_NOMEM, "pinned staging allocation failed");
    if (a->span_off.size == 0) a->span_off.push(0);
    const uint32_t at = static_cast<uint32_t>(a->n_bases);
    a->src_pos.push(reads->off[q_id] + (q_reverse ? reads->length[q_id] - 1 - q_start : q_start));
    a->src_flags.push(q_reverse ? rp::kSrcReverse : 0);
    a->span_off.push(at + (too_long ? 0 : q_len));
    a->src_pos.push(reads->off[t_id] + t_begin);
    a->src_flags.push(0);
    a->span_off.push(at + static_cast<uint32_t>(add));
    a->by_ref = true;
    a->reads = reads;
    return aln_add_metadata(a, q_len, t_len, t_begin, q_start, too_long);
}

/* the part of adding an overlap that does not touch its bases */
static rp_status aln_add_metadata(rp_aln* a, uint32_t ql, uint32_t tl, uint32_t t_begin, uint32_t q_start, bool too_long) {
    const uint64_t add = too_long ? 0 : static_cast<uint64_t>(ql) + tl;
    const uint32_t off = static_cast<uint32_t>(a->n_bases);
    a->n_bases += add;
    const uint32_t cap = too_long ? 0 : (ql + tl) / 3 + 64;
    if (!a->q_off.push(off) || !a->q_len.push(too_long ? 0 : ql) || !a->t_off.push(off + (too_long ? 0 : ql)) ||
        !a->t_len.push(too_long ? 0 : tl) || !a->run_off.push(static_cast<uint32_t>(a->run_total)) ||
        !a->run_cap.push(cap))
        return fail(RP_ERR_NOMEM, "pinned staging allocation failed");
    a->run_total += cap;
    uint32_t bcap = 0;
    if (a->window_length && !too_long && tl > 0) {
        const uint64_t w = a->window_length;
        bcap = static_cast<uint32_t>(2 * ((static_cast<uint64_t>(t_begin) + tl - 1) / w - t_begin / w + 1));
    }
    if (!a->t_begin.push(t_begin) || !a->q_start.push(q_start) ||
        !a->bp_off.push(static_cast<uint32_t>(a->bp_total)) || !a->bp_cap.push(bcap))
        return fail(RP_ERR_NOMEM, "pinned staging allocation failed");
    a->bp_total += bcap;
    a->pre_status.push_back(too_long ? RP_ALN_TOO_LONG : RP_ALN_OK);
    return RP_OK;
}

uint32_t rp_aln_size(const rp_aln* a) { return a ? static_cast<uint32_t>(a->pre_status.size()) : 0; }

rp_status rp_aln_upload(rp_aln* a) {
    if (!a) return fail(RP_ERR_INVALID, "null object");
    RP_CUDA(cudaSetDevice(a->device));
    const uint32_t n = rp_aln_size(a);
    /* longest pairs first */
    std::vector<uint32_t> idx(n);
    for (uint32_t i = 0; i < n; ++i) idx[i] = i;
    std::stable_sort(idx.begin(), idx.end(), [&](uint32_t x, uint32_t y) {
        return static_cast<uint64_t>(a->q_len.data[x]) * a->t_len.data[x] >
               static_cast<uint64_t>(a->q_len.data[y]) * a->t_len.data[y];
    });
    a->queue.clear();
    if (!a->queue.reserve(n ? n : 1)) return fail(RP_ERR_NOMEM, "queue allocation failed");
    for (uint32_t i = 0; i < n; ++i) a->queue.push(idx[i]);
    rp::AlnParams& P = a->P;
    a->last_h2d = 0;
    if (a->by_ref) {
        const uint64_t* src_pos = nullptr;
        const uint8_t* src_flags = nullptr;
        const uint32_t* span_off = nullptr;
        RP_CUDA(reserve(a->d_bases, a->n_bases + 16, P.bases));
        RP_CUDA(upload(a, a->d_src_pos, a->src_pos, src_pos));
        RP_CUDA(upload(a, a->d_src_flags, a->src_flags, src_flags));
        RP_CUDA(upload(a, a->d_span_off, a->span_off, span_off));
        /* both spans of every pair are cut out of the store on the device (reverse complement included) */
        if (a->src_pos.size > 0)
            RP_CUDA(launch_gather(a->reads, a->d_bases.p, nullptr, span_off, src_pos, src_flags, a->src_pos.size,
                                  a->stream, a->device));
    } else {
        RP_CUDA(upload(a, a->d_bases, a->bases, P.bases));
    }
    RP_CUDA(upload(a, a->d_q_off, a->q_off, P.q_off));
    RP_CUDA(upload(a, a->d_q_len, a->q_len, P.q_len));
    RP_CUDA(upload(a, a->d_t_off, a->t_off, P.t_off));
    RP_CUDA(upload(a, a->d_t_len, a->t_len, P.t_len));
    RP_CUDA(upload(a, a->d_run_off, a->run_off, P.run_off));
    RP_CUDA(upload(a, a->d_run_cap, a->run_cap, P.run_cap));
    RP_CUDA(upload(a, a->d_queue, a->queue, P.queue));
    if (a->window_length) {
        RP_CUDA(upload(a, a->d_t_begin, a->t_begin, P.t_begin));
        RP_CUDA(upload(a, a->d_q_start, a->q_start, P.q_start));
        RP_CUDA(upload(a, a->d_bp_off, a->bp_off, P.bp_off));
        RP_CUDA(upload(a, a->d_bp_cap, a->bp_cap, P.bp_cap));
        RP_CUDA(reserve(a->d_bp, (a->bp_total + 4) * 8, P.bp));
        RP_CUDA(reserve(a->d_n_bp, (n + 1) * 4, P.n_bp));
        if (!a->h_bp.reserve(2 * a->bp_total + 8) || !a->h_n_bp.reserve(n + 1))
            return fail(RP_ERR_NOMEM, "pinned result allocation failed");
    }
    RP_CUDA(reserve(a->d_runs, (a->run_total + 16) * 4, P.runs));
    RP_CUDA(reserve(a->d_n_runs, (n + 1) * 4, P.n_runs));
    RP_CUDA(reserve(a->d_dist, (n + 1) * 4, P.dist));
    RP_CUDA(reserve(a->d_status, (n + 1) * 4, P.status));
    if (!a->h_runs.reserve(a->run_total + 16) || !a->h_n_runs.reserve(n + 1) || !a->h_status.reserve(n + 1) ||
        !a->h_dist.reserve(n + 1))
        return fail(RP_ERR_NOMEM, "pinned result allocation failed");
    P.n_pairs = n;
    P.queue_head = static_cast<uint32_t*>(a->d_head.p);
    P.scratch = static_cast<uint8_t*>(a->d_scratch.p);
    P.window_length = a->window_length;
    a->uploaded = true;
    a->launched = a->downloaded = a->synced = false;
    return RP_OK;
}

rp_status rp_aln_launch(rp_aln* a) {
    if (!a) return fail(RP_ERR_INVALID, "null object");
    if (!a->uploaded) return fail(RP_ERR_STATE, "launch before upload");
    RP_CUDA(cudaSetDevice(a->device));
    if (a->P.n_pairs > 0) {
        RP_CUDA(cudaMemsetAsync(a->d_head.p, 0, 4, a->stream));
        RP_CUDA(launch(rp_aln_kernel, static_cast<uint32_t>(a->grid), kWarpsPerBlock * 32, 0, a->stream, a->P));
        a->launches += 1;
    }
    a->launched = true;
    a->downloaded = a->synced = false;
    return RP_OK;
}

rp_status rp_aln_download(rp_aln* a) {
    if (!a) return fail(RP_ERR_INVALID, "null object");
    if (!a->launched) return fail(RP_ERR_STATE, "download before launch");
    RP_CUDA(cudaSetDevice(a->device));
    const uint32_t n = a->P.n_pairs;
    uint64_t d2h = 0;
    if (n > 0) {
        RP_CUDA(cudaMemcpyAsync(a->h_n_runs.data, a->d_n_runs.p, n * 4, cudaMemcpyDeviceToHost, a->stream));
        RP_CUDA(cudaMemcpyAsync(a->h_dist.data, a->d_dist.p, n * 4, cudaMemcpyDeviceToHost, a->stream));
        RP_CUDA(cudaMemcpyAsync(a->h_status.data, a->d_status.p, n * 4, cudaMemcpyDeviceToHost, a->stream));
        RP_CUDA(cudaMemcpyAsync(a->h_runs.data, a->d_runs.p, a->run_total * 4, cudaMemcpyDeviceToHost, a->stream));
        d2h = a->run_total * 4 + static_cast<uint64_t>(n) * 12;
        if (a->window_length) {
            RP_CUDA(cudaMemcpyAsync(a->h_n_bp.data, a->d_n_bp.p, n * 4, cudaMemcpyDeviceToHost, a->stream));
            if (a->bp_total)
                RP_CUDA(cudaMemcpyAsync(a->h_bp.data, a->d_bp.p, a->bp_total * 8, cudaMemcpyDeviceToHost, a->stream));
            d2h += a->bp_total * 8 + static_cast<uint64_t>(n) * 4;
        }
    }
    a->last_d2h = d2h;
    a->cigars.assign(n, std::string());
    a->cigar_built.assign(n, 0);
    a->downloaded = true;
    a->synced = false;
    return RP_OK;
}

rp_status rp_aln_run(rp_aln* a) {
    rp_status s = rp_aln_upload(a);
    if (s != RP_OK) return s;
    s = rp_aln_launch(a);
    if (s != RP_OK) return s;
    return rp_aln_download(a);
}

rp_status rp_aln_sync(rp_aln* a) {
    if (!a) return fail(RP_ERR_INVALID, "null object");
    RP_CUDA(cudaSetDevice(a->device));
    RP_CUDA(cudaStreamSynchronize(a->stream));
    if (a->downloaded) a->synced = true;
    return RP_OK;
}

rp_status rp_aln_query(rp_aln* a) { return query_stream(a, a && a->launched); }

rp_status rp_aln_fetch_cigar(rp_aln* a, uint32_t i, const char** cigar, uint32_t* len, int32_t* edit_distance,
                             uint32_t* status) {
    if (!a) return fail(RP_ERR_INVALID, "null object");
    if (!a->downloaded) return fail(RP_ERR_STATE, "fetch before run/download");
    if (!a->synced) {
        rp_status s = rp_aln_sync(a);
        if (s != RP_OK) return s;
    }
    if (i >= rp_aln_size(a)) return fail(RP_ERR_INVALID, "overlap index out of range");
    uint32_t st = a->pre_status[i] ? a->pre_status[i] : a->h_status.data[i];
    /* the text is built on the first call that asks for it: a caller after the status alone (the polisher, which takes
     * the breaking points) pays nothing per run */
    if ((cigar || len) && !a->cigar_built[i]) {
        std::string& c = a->cigars[i];
        if (st == RP_ALN_OK) {
            const uint32_t* r = a->h_runs.data + a->run_off.data[i];
            const uint32_t nr = a->h_n_runs.data[i];
            char tmp[16];
            for (uint32_t k = 0; k < nr; ++k) {
                int w = snprintf(tmp, sizeof(tmp), "%u%c", r[k] >> 8, static_cast<char>(r[k] & 0xff));
                c.append(tmp, static_cast<size_t>(w));
            }
        }
        a->cigar_built[i] = 1;
    }
    if (cigar) *cigar = a->cigars[i].c_str();
    if (len) *len = static_cast<uint32_t>(a->cigars[i].size());
    if (edit_distance) *edit_distance = st == RP_ALN_OK ? a->h_dist.data[i] : -1;
    if (status) *status = st;
    return RP_OK;
}

rp_status rp_aln_fetch_breaking_points(rp_aln* a, uint32_t i, const uint32_t** points, uint32_t* n_points) {
    if (!a || !points || !n_points) return fail(RP_ERR_INVALID, "null argument");
    if (!a->downloaded) return fail(RP_ERR_STATE, "fetch before run/download");
    if (!a->window_length) return fail(RP_ERR_STATE, "no window length set: breaking points were not computed");
    if (!a->synced) {
        rp_status s = rp_aln_sync(a);
        if (s != RP_OK) return s;
    }
    if (i >= rp_aln_size(a)) return fail(RP_ERR_INVALID, "overlap index out of range");
    const uint32_t st = a->pre_status[i] ? a->pre_status[i] : a->h_status.data[i];
    *points = a->h_bp.data + 2ull * a->bp_off.data[i];
    *n_points = st == RP_ALN_OK ? a->h_n_bp.data[i] : 0;
    return RP_OK;
}

rp_status rp_aln_reset(rp_aln* a) {
    if (!a) return fail(RP_ERR_INVALID, "null object");
    cudaSetDevice(a->device);
    if (a->stream) RP_CUDA(cudaStreamSynchronize(a->stream));
    a->bases.clear(); a->q_off.clear(); a->q_len.clear(); a->t_off.clear(); a->t_len.clear();
    a->run_off.clear(); a->run_cap.clear(); a->queue.clear();
    a->t_begin.clear(); a->q_start.clear(); a->bp_off.clear(); a->bp_cap.clear();
    a->src_pos.clear(); a->src_flags.clear(); a->span_off.clear();
    a->by_ref = false;
    a->n_bases = 0;
    a->pre_status.clear();
    a->run_total = 0;
    a->bp_total = 0;
    a->cigars.clear();
    a->cigar_built.clear();
    a->uploaded = a->launched = a->downloaded = a->synced = false;
    return RP_OK;
}

rp_status rp_aln_info(rp_aln* a, uint64_t info[8]) {
    if (!a || !info) return fail(RP_ERR_INVALID, "null argument");
    std::memset(info, 0, 8 * sizeof(uint64_t));
    info[0] = a->launches;
    info[1] = a->last_h2d;
    info[2] = a->last_d2h;
    info[3] = a->workers;
    info[4] = a->P.lay.bytes;
    return RP_OK;
}

}  // extern "C"
