/*
 * rp_warp.cuh — the warp-level vocabulary the POA/Myers device code is written in.
 *
 * Two builds of the SAME device code:
 *   nvcc (sm_90a)          : thin wrappers over __shfl_sync / __ballot_sync / DPX packed-int16 ops
 *                            (VIADDMNMX.S16x2 via __viaddmax_s16x2, PRMT via __byte_perm).
 *   g++ -DRP_HOST_SIM=1    : TEST-ONLY simulation — one simulated warp = 32 cooperative fibres
 *                            (ucontext) that meet at every collective.  It lets tests/ run the device
 *                            logic under ASan/gdb on the CPU container (no GPU there).  It is never
 *                            part of libracon_b200.so: the product has no CPU path.
 */
#pragma once
#include <stdint.h>

#if defined(RP_HOST_SIM)
#include <ucontext.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#define RP_DEV inline
#define RP_DEV_NOINLINE
#define RP_HD inline
#define RP_GLOBAL
#define RP_KEEP_IN_REGISTER(x) do { } while (0)
template <typename T> inline T* keep_smem_ptr(T* p) { return p; }
#else
#include <cuda_runtime.h>
#define RP_DEV __device__ __forceinline__
#define RP_DEV_NOINLINE __device__ __noinline__
#define RP_HD __host__ __device__ __forceinline__
/* makes a 32-bit value opaque to the compiler at this point: it then has to keep it in a register instead of
 * re-deriving it (from the thread index, the parameter block ...) inside a loop.  No instruction is emitted. */
#define RP_KEEP_IN_REGISTER(x) asm volatile("" : "+r"(x))
/* the same for a pointer into shared memory: its 32-bit shared-window address is pinned, so that an address derived from
 * it inside a loop costs one add, and the accesses stay LDS/STS */
template <typename T> __device__ __forceinline__ T* keep_smem_ptr(T* p) {
    uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
    RP_KEEP_IN_REGISTER(a);
    return static_cast<T*>(__cvta_shared_to_generic(a));
}
#endif

namespace rp {

constexpr uint32_t kFull = 0xffffffffu;

#if defined(RP_HOST_SIM)
/* ------------------------------------------------------------------ host simulation */
namespace sim {
struct Warp {
    ucontext_t main;
    ucontext_t ctx[32];
    char* stacks = nullptr;
    bool done[32];
    uint64_t slot[32];
    uint64_t result[32];
    int arrived = 0;
    uint64_t gen = 0;
    int cur = 0;
    int n = 32;          // lanes of this simulated warp (32, or one 8/16-lane group of the POA kernel)
    void (*fn)(void*) = nullptr;
    void* arg = nullptr;
};
inline Warp*& current() {
    static thread_local Warp* w = nullptr;
    return w;
}
inline void yield_() {
    Warp* w = current();
    swapcontext(&w->ctx[w->cur], &w->main);
}
inline void trampoline() {
    Warp* w = current();
    w->fn(w->arg);
    w->done[w->cur] = true;
    swapcontext(&w->ctx[w->cur], &w->main);
}
/* Runs fn(arg) as n (default 32) lock-step-at-collectives fibres. */
inline void run_warp(void (*fn)(void*), void* arg, size_t stack_bytes = 256 * 1024, int n = 32) {
    Warp w;
    w.fn = fn;
    w.arg = arg;
    w.n = n;
    w.stacks = static_cast<char*>(malloc(stack_bytes * 32));
    Warp* saved = current();
    current() = &w;
    for (int l = 0; l < n; ++l) {
        w.done[l] = false;
        getcontext(&w.ctx[l]);
        w.ctx[l].uc_stack.ss_sp = w.stacks + static_cast<size_t>(l) * stack_bytes;
        w.ctx[l].uc_stack.ss_size = stack_bytes;
        w.ctx[l].uc_link = &w.main;
        makecontext(&w.ctx[l], reinterpret_cast<void (*)()>(trampoline), 0);
    }
    for (;;) {
        int alive = 0;
        for (int l = 0; l < n; ++l) {
            if (w.done[l]) continue;
            ++alive;
            w.cur = l;
            swapcontext(&w.main, &w.ctx[l]);
        }
        if (!alive) break;
        int finished = 0;
        for (int l = 0; l < n; ++l) finished += w.done[l] ? 1 : 0;
        if (finished > 0 && finished < n && w.arrived > 0 && w.arrived + finished == n) {
            fprintf(stderr, "[rp::sim] deadlock: %d lanes wait at a collective, %d lanes already returned\n",
                    w.arrived, finished);
            abort();
        }
    }
    current() = saved;
    free(w.stacks);
}
inline uint64_t collective(uint64_t v, int src_or_neg /* -1: return own slot table ptr semantic */) {
    Warp* w = current();
    int me = w->cur;
    w->slot[me] = v;
    uint64_t my_gen = w->gen;
    if (++w->arrived == w->n) {
        memcpy(w->result, w->slot, sizeof(w->slot));
        w->arrived = 0;
        w->gen++;
    } else {
        while (w->gen == my_gen) yield_();
    }
    (void)src_or_neg;
    return 0;
}
inline uint64_t result_of(int lane) { return current()->result[lane & (current()->n - 1)]; }
inline int lanes() { return current()->n; }
}  // namespace sim

inline int lane_id() { return sim::current()->cur; }
inline void syncwarp() { sim::collective(0, 0); }
/* 16-byte asynchronous global -> shared copy (cp.async on the device): here an ordinary copy, nothing to wait for */
inline void copy16_async(void* smem_dst, const void* gsrc) { std::memcpy(smem_dst, gsrc, 16); }
inline void copy_async_wait() {}
inline uint32_t ballot(bool p) {
    sim::collective(p ? 1 : 0, 0);
    uint32_t m = 0;
    for (int l = 0; l < sim::lanes(); ++l) m |= (sim::result_of(l) ? 1u : 0u) << l;
    return m;
}
template <typename T>
inline T shfl(T v, int src) {
    uint64_t raw = 0;
    static_assert(sizeof(T) <= 8, "shfl payload");
    memcpy(&raw, &v, sizeof(T));
    sim::collective(raw, 0);
    uint64_t r = sim::result_of(src);
    T out;
    memcpy(&out, &r, sizeof(T));
    return out;
}
template <typename T>
inline T shfl_up(T v, int d) {
    int me = lane_id();
    T got = shfl(v, me - d < 0 ? me : me - d);
    return got;
}
template <typename T>
inline T shfl_down(T v, int d) {
    int me = lane_id();
    T got = shfl(v, me + d > sim::lanes() - 1 ? me : me + d);
    return got;
}
inline uint32_t atomic_add(uint32_t* p, uint32_t v) {
    uint32_t o = *p;
    *p = o + v;
    return o;
}
inline uint32_t atomic_add_u16(uint16_t* p, uint32_t v) {
    uint32_t o = *p;
    *p = static_cast<uint16_t>(o + v);
    return o;
}
/* adds v to a 64-bit statistics counter (atomic on the device; here the workers run one after the other) */
template <typename T>
inline void count_add(T* p, unsigned long long v) { *p += v; }
inline int popc(uint32_t x) { return __builtin_popcount(x); }
inline int ffs_(uint32_t x) { return __builtin_ffs(static_cast<int>(x)); }

/* packed int16x2 helpers (wrapping arithmetic like the hardware) */
inline int16_t lo16(uint32_t a) { return static_cast<int16_t>(a & 0xffff); }
inline int16_t hi16(uint32_t a) { return static_cast<int16_t>(a >> 16); }
inline uint32_t pack16(int32_t lo, int32_t hi) {
    return (static_cast<uint32_t>(lo) & 0xffffu) | (static_cast<uint32_t>(hi) << 16);
}
inline uint32_t viaddmax_s16x2(uint32_t a, uint32_t b, uint32_t c) {
    int16_t l = static_cast<int16_t>(lo16(a) + lo16(b));
    int16_t h = static_cast<int16_t>(hi16(a) + hi16(b));
    return pack16(l > lo16(c) ? l : lo16(c), h > hi16(c) ? h : hi16(c));
}
inline int32_t viaddmax_s32(int32_t a, int32_t b, int32_t c) {
    int32_t s = a + b;
    return s > c ? s : c;
}
inline uint32_t vmax_s16x2(uint32_t a, uint32_t b) {
    return pack16(lo16(a) > lo16(b) ? lo16(a) : lo16(b), hi16(a) > hi16(b) ? hi16(a) : hi16(b));
}
inline uint32_t byte_perm(uint32_t a, uint32_t b, uint32_t sel) {
    uint64_t all = (static_cast<uint64_t>(b) << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) {
        uint32_t s = (sel >> (4 * i)) & 7;
        r |= static_cast<uint32_t>((all >> (8 * s)) & 0xff) << (8 * i);
    }
    return r;
}

#else
/* ------------------------------------------------------------------ sm_90a */
RP_DEV int lane_id() { return static_cast<int>(threadIdx.x & 31); }
RP_DEV void syncwarp() { __syncwarp(); }
/* 16-byte asynchronous global -> shared copy (LDGSTS): the data goes from HBM / L2 into shared memory without passing
 * through registers, and any number of copies can be in flight per lane; both addresses 16-byte aligned.
 * copy_async_wait(): every copy this lane has issued has landed (a __syncwarp then publishes them to the other lanes). */
RP_DEV void copy16_async(void* smem_dst, const void* gsrc) {
    const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
RP_DEV void copy_async_wait() {
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}
RP_DEV uint32_t ballot(bool p) { return __ballot_sync(kFull, p); }
template <typename T>
RP_DEV T shfl(T v, int src) {
    return __shfl_sync(kFull, v, src);
}
template <typename T>
RP_DEV T shfl_up(T v, int d) {
    return __shfl_up_sync(kFull, v, d);
}
template <typename T>
RP_DEV T shfl_down(T v, int d) {
    return __shfl_down_sync(kFull, v, d);
}
RP_DEV uint32_t atomic_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
template <typename T>
RP_DEV void count_add(T* p, unsigned long long v) {
    static_assert(sizeof(T) == sizeof(unsigned long long), "64-bit counter");
    atomicAdd(reinterpret_cast<unsigned long long*>(p), v);
}
RP_DEV int popc(uint32_t x) { return __popc(x); }
RP_DEV int ffs_(uint32_t x) { return __ffs(static_cast<int>(x)); }
RP_DEV int16_t lo16(uint32_t a) { return static_cast<int16_t>(a & 0xffff); }
RP_DEV int16_t hi16(uint32_t a) { return static_cast<int16_t>(a >> 16); }
RP_DEV uint32_t pack16(int32_t lo, int32_t hi) {
    return __byte_perm(static_cast<uint32_t>(lo), static_cast<uint32_t>(hi), 0x5410);
}
/* DPX: per-halfword max(a + b, c) — one VIADDMNMX.S16x2 on sm_90+ */
RP_DEV uint32_t viaddmax_s16x2(uint32_t a, uint32_t b, uint32_t c) { return __viaddmax_s16x2(a, b, c); }
RP_DEV int32_t viaddmax_s32(int32_t a, int32_t b, int32_t c) { return __viaddmax_s32(a, b, c); }
RP_DEV uint32_t vmax_s16x2(uint32_t a, uint32_t b) { return __vmaxs2(a, b); }  // VIMNMX.S16x2
RP_DEV uint32_t byte_perm(uint32_t a, uint32_t b, uint32_t sel) { return __byte_perm(a, b, sel); }
#endif

RP_DEV uint32_t lanemask_lt() { return (1u << lane_id()) - 1u; }

/* exclusive prefix count of a predicate over the warp; *total = popcount */
RP_DEV uint32_t warp_rank(bool p, uint32_t* total) {
    uint32_t m = ballot(p);
    *total = static_cast<uint32_t>(popc(m));
    return static_cast<uint32_t>(popc(m & lanemask_lt()));
}

/* inclusive warp scans */
RP_DEV uint32_t warp_incl_sum(uint32_t v) {
    int l = lane_id();
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t o = shfl_up(v, d);
        if (l >= d) v += o;
    }
    return v;
}
RP_DEV int32_t warp_incl_max(int32_t v) {
    int l = lane_id();
    for (int d = 1; d < 32; d <<= 1) {
        int32_t o = shfl_up(v, d);
        if (l >= d && o > v) v = o;
    }
    return v;
}

/* ------------------------------------------------------------------ lane groups
 * The POA kernel runs one window per GROUP of G lanes (G = 8, 16 or 32), 32/G independent windows per warp:
 * the groups of a warp execute the same instruction stream, so one issued instruction advances 32/G windows
 * wherever their control flow agrees (SIMT), and every collective below only names the lanes of its own group,
 * which keeps it legal when the groups have diverged.  In the host simulation a group is simply a simulated
 * warp of G fibres. */
#if defined(RP_HOST_SIM)
template <int G> RP_DEV int glane() { return lane_id(); }
template <int G> RP_DEV void gsync() { syncwarp(); }
template <int G> RP_DEV uint32_t gballot(bool p) { return ballot(p); }
template <int G, typename T> RP_DEV T gshfl(T v, int src) { return shfl(v, src); }
template <int G, typename T> RP_DEV T gshfl_up(T v, int d) { return shfl_up(v, d); }
template <int G, typename T> RP_DEV T gshfl_down(T v, int d) { return shfl_down(v, d); }
/* true when any group that currently executes together with this one votes yes (a hint, never needed for
 * correctness): the simulation knows only its own group */
template <int G> RP_DEV bool any_converged_peer(bool p) { return ballot(p) != 0; }
#else
template <int G> RP_DEV int glane() { return static_cast<int>(threadIdx.x & (G - 1)); }
template <int G> RP_DEV uint32_t gbase() { return (threadIdx.x & 31u) & ~static_cast<uint32_t>(G - 1); }
template <int G> RP_DEV uint32_t gmask() {
    return G == 32 ? kFull : (((1u << (G & 31)) - 1u) << gbase<G>());
}
template <int G> RP_DEV void gsync() { __syncwarp(gmask<G>()); }
template <int G> RP_DEV uint32_t gballot(bool p) {
    return (__ballot_sync(gmask<G>(), p) >> gbase<G>()) & (G == 32 ? kFull : ((1u << (G & 31)) - 1u));
}
template <int G, typename T> RP_DEV T gshfl(T v, int src) { return __shfl_sync(gmask<G>(), v, src, G); }
template <int G, typename T> RP_DEV T gshfl_up(T v, int d) { return __shfl_up_sync(gmask<G>(), v, d, G); }
template <int G, typename T> RP_DEV T gshfl_down(T v, int d) { return __shfl_down_sync(gmask<G>(), v, d, G); }
template <int G> RP_DEV bool any_converged_peer(bool p) {
    const uint32_t act = __activemask();        // whoever happens to execute this together with me
    return __ballot_sync(act, p) != 0;
}
#endif

template <int G> RP_DEV uint32_t grank(bool p, uint32_t* total) {
    const uint32_t m = gballot<G>(p);
    *total = static_cast<uint32_t>(popc(m));
    return static_cast<uint32_t>(popc(m & ((1u << glane<G>()) - 1u)));
}
template <int G> RP_DEV uint32_t gincl_sum(uint32_t v) {
    const int l = glane<G>();
#pragma unroll
    for (int d = 1; d < G; d <<= 1) {
        uint32_t o = gshfl_up<G>(v, d);
        if (l >= d) v += o;
    }
    return v;
}
template <int G> RP_DEV int32_t gincl_max(int32_t v) {
    const int l = glane<G>();
#pragma unroll
    for (int d = 1; d < G; d <<= 1) {
        int32_t o = gshfl_up<G>(v, d);
        if (l >= d && o > v) v = o;
    }
    return v;
}

}  // namespace rp
