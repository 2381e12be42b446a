/*
 * poa_core.cuh — CUDA-native (sm_90a) per-window partial-order-alignment consensus (device code).
 *
 * What the reference does per window (Window::generate_consensus, /root/reference/src/window.cpp:65-149,
 * driving spoa: vendor/spoa/src/graph.cpp and sisd/simd alignment engines) is done here by ONE WARP per
 * window, many windows in flight per SM, in one persistent kernel launch:
 *
 *   for every layer:   [subgraph marking]  ->  DP "program" build  ->  NW-linear graph x read DP
 *                      ->  traceback  ->  graph merge  ->  incremental topological order update
 *   then:              spoa-order DFS sort -> heaviest-bundle consensus -> coverage -> TGS trim
 *
 * Design (not a port; see DESIGN.md):
 *   * The POA graph lives in HBM as flat per-node slot arrays (in-edge slots with weights, aligned-node
 *     slots, per-node sequence counters instead of per-edge label lists).  Every graph phase is a
 *     lane-strided data-parallel loop, so HBM latency is overlapped 32-wide.
 *   * The DP keeps a whole 512-column row chunk in registers: lane l owns 16 consecutive columns as
 *     8 packed int16x2 registers; predecessor rows come from a shared-memory ring of the most recent
 *     rows (conflict-free swizzled 128-bit loads) or, for far predecessors, from the HBM copy; the cell
 *     update is two DPX VIADDMNMX.S16x2 per predecessor per register; the in-row gap recurrence is a
 *     lane-local max-plus chain plus a 5-step warp shuffle scan.
 *   * Rows are processed in an incrementally maintained topological order (aligned clusters kept
 *     contiguous).  Cell values and the traceback do not depend on which valid topological order is
 *     used; spoa's own DFS order (graph.cpp:249-303) is only needed to break ties between equally
 *     scoring sink rows and for the final consensus, and is computed on demand.
 *   * H rows are streamed once to HBM (coalesced 1 KB row stores) for the traceback.
 *
 * Exact semantics reproduced (SURVEY.md Appendix A): A.1 DP / sink choice / traceback priority,
 * A.2 graph merge, A.3 topological order (on demand), A.4 heaviest bundle + branch completion,
 * A.5 coverage + trim, A.6 subgraph.
 */
#pragma once
#include "rp_warp.cuh"

namespace rp {

constexpr uint16_t kNone = 0xffffu;
constexpr int kChunkCols = 512;          // padding unit of the row length limit (the widest chunk: 32 lanes x 16)
constexpr int32_t kBandFloor = -32768 + 1024;   // banded rows: "minus infinity" of excluded cells = spoa's int16 legal minimum
constexpr int32_t kNegDiag = -32640;     // "column -1" sentinel: + any int8 profile value stays >= INT16_MIN and
                                         // below every legal score (legal >= INT16_MIN + 1024, the int16 criterion)
constexpr int32_t kNeg32 = -(1 << 28);
constexpr int32_t kMaxGapInt16 = 64;     // |gap| bound of the packed-int16 path (sentinel + 16*gap must not wrap)

/* window status codes (soft, per window; mirrored in include/racon_b200.h) */
enum : uint32_t {
    kWinOk = 0,
    kWinNodeLimit = 1,
    kWinEdgeLimit = 2,
    kWinAlignedLimit = 3,
    kWinNeedsInt32 = 4,
    kWinSeqTooLong = 5,
    kWinStackLimit = 6,
    kWinAlphabetLimit = 7,
    kWinInternal = 8,
    kWinMatrixLimit = 9,   // score matrix larger than the per-window scratch (re-run by the escalation pass)
};

struct PoaLimits {
    uint32_t nmax;   // max graph nodes per window
    uint32_t lmax;   // max layer length
    uint32_t lp;     // padded row length in int16 cells: multiple of kCC, >= lmax + 1
    uint32_t ki;     // in-edge slots per node
    uint32_t ka;     // aligned-node slots per node
    uint32_t stack_cap;
    uint32_t hcap;   // int16 cells of score-matrix scratch per window ((rows + 1) x padded row length must fit)
};

struct SlotLayout {
    uint64_t code, flags, in_cnt, al_cnt, cov, in_tail, in_w, al, order_a, order_b, rank_of, dp_order, dp_rank,
        rec, pred_ovf, H, aln, cur, member, has_out_sub, score, cpred, sorder, srank, marks, stack,
        newlist, ccarry, bpos, bs, delta, bytes;
};

RP_HD uint64_t align_up(uint64_t x, uint64_t a) { return (x + a - 1) / a * a; }

RP_HD SlotLayout make_layout(const PoaLimits& L) {
    SlotLayout s;
    uint64_t o = 0;
    auto take = [&](uint64_t bytes) {
        uint64_t r = o;
        o = align_up(o + bytes, 256);
        return r;
    };
    uint64_t n = L.nmax;
    s.code = take(n);
    s.flags = take(n);
    s.in_cnt = take(n);
    s.al_cnt = take(n);
    s.cov = take(n * 2);
    s.in_tail = take(n * L.ki * 2);
    s.in_w = take(n * L.ki * 4);
    s.al = take(n * L.ka * 2);
    s.order_a = take((n + 2 + 64) * 2);
    s.order_b = take((n + 2 + 64) * 2);
    s.rank_of = take(n * 2);
    s.dp_order = take((n + 2 + 64) * 2);
    s.dp_rank = take(n * 2);
    s.rec = take((n + 1 + 160) * 16);
    s.pred_ovf = take((n + 1) * L.ki * 2);
    s.H = take(static_cast<uint64_t>(L.hcap) * 2 + 64);
    s.aln = take((static_cast<uint64_t>(L.lmax) + 1) * 2);
    s.cur = take((static_cast<uint64_t>(L.lmax) + 1) * 2);
    s.member = take(n);
    s.has_out_sub = take(n);
    s.score = take(n * 8);
    s.cpred = take(n * 2);
    s.sorder = take(n * 2);
    s.srank = take(n * 2);
    s.marks = take(n);
    s.stack = take(static_cast<uint64_t>(L.stack_cap) * 2);
    s.newlist = take((static_cast<uint64_t>(L.lmax) + 1) * 4);
    s.ccarry = take((n + 2) * 2 * 2);
    s.bpos = take(n * 2);
    s.bs = take(n + 2 + 64);
    s.delta = take((n + 4) * 2);
    s.bytes = align_up(o, 4096);
    return s;
}

/* Launch-wide parameters (plain pointers into HBM). */
struct PoaParams {
    int32_t match, mismatch, gap;
    /* per-register constants of a full-matrix DP row, derived from `gap` by set_scores(): [r] = (0, (r+1)g) bridge
     * offsets, [8+r] = ((r+1)g, (r+9)g) carry offsets, [16] = (g, g).  Kept in the parameter block so that the row loop
     * takes them straight from the constant bank as instruction operands — as loop-invariant registers they do not
     * survive the kernel's register cap and were rebuilt (about 35 instructions) in every row. */
    uint32_t row_consts[17];
    uint32_t n_windows;
    /* inputs, packed by the host in processing order (backbone first, layers sorted as window.cpp:85-86) */
    const uint8_t* bases;
    const uint8_t* weights;       // per base: quality - 33, or 1 (layers without quality), 0 (dummy backbone)
    const uint32_t* seq_off;      // n_seq + 1
    const uint32_t* seq_begin;
    const uint32_t* seq_end;
    const uint8_t* seq_flags;     // bit0: full-span layer (window.cpp:92-93 test evaluated on the host)
    const uint32_t* win_first;    // n_windows + 1
    const uint8_t* win_flags;     // bit0: trim (type == kTGS && trim)
    const uint64_t* win_alpha;    // up to 8 distinct characters of the window, low byte first
    const uint32_t* queue;        // processing order of windows (longest first)
    uint32_t* queue_head;         // atomic cursor
    /* outputs */
    uint8_t* cons;                // window w at cons + out_off[w], capacity out_cap[w]
    uint16_t* cons_cov;           // same offsets (per-base coverage of the returned consensus)
    const uint32_t* out_off;
    const uint32_t* out_cap;
    uint32_t* cons_len;
    uint32_t* status;
    uint64_t* stats;              // optional device counters (may be null): [0] alignments, [1] dp cells, ...
    /* scratch */
    uint8_t* scratch;
    PoaLimits lim;
    SlotLayout lay;
    uint32_t smem_per_group;      // bytes of shared memory owned by each lane group (= one window in flight)
    uint32_t tile_rows;           // traceback tile height in ranks (0 = as many as fit, at most 96)
    uint32_t debug_flags;         // tests only: bit0 = use the HBM-resident variants of the order DFS / bundle
    uint32_t banded;              // 1: every alignment is first tried inside a diagonal band of 16*G columns
                                  // (racon -b); a band result that cannot be trusted is redone with the full matrix
    uint32_t band_margin;         // columns the traceback must keep from a cut band edge to be trusted
    unsigned long long* band_stats;  // [0] alignments tried in the band, [1] redone with the full matrix (may be null)
};

/* scores + everything derived from them (host side, both the product and the test builds fill PoaParams through this) */
inline void set_scores(PoaParams& P, int32_t match, int32_t mismatch, int32_t gap) {
    P.match = match;
    P.mismatch = mismatch;
    P.gap = gap;
    auto pk = [](int32_t lo, int32_t hi) {
        return (static_cast<uint32_t>(lo) & 0xffffu) | (static_cast<uint32_t>(hi) << 16);
    };
    for (int r = 0; r < 8; ++r) {
        P.row_consts[r] = pk(0, (r + 1) * gap);
        P.row_consts[8 + r] = pk((r + 1) * gap, (r + 9) * gap);
    }
    P.row_consts[16] = pk(gap, gap);
}

/* Row layout.  A lane owns 16 consecutive columns; inside that 32-byte block register r (0..7) packs
 * column r in its low half and column 8+r in its high half, so the in-row gap recurrence runs as two
 * packed 8-long chains and the diagonal operand of register r is simply register r-1 of the predecessor.
 * perm(): logical column -> element index in a row stored in that register order (HBM copy);
 * swz(): additionally XOR-swizzles 16-byte granules so the two LDS.128 of a lane are bank-conflict free. */
RP_DEV uint32_t perm(uint32_t c) { return (c & ~15u) | ((c & 7u) << 1) | ((c >> 3) & 1u); }
RP_DEV uint32_t swz_e(uint32_t e) {
    uint32_t q = e >> 3;
    return ((q ^ ((q >> 3) & 1u)) << 3) | (e & 7u);
}
RP_DEV uint32_t swz(uint32_t c) { return swz_e(perm(c)); }

struct Row8 {
    uint32_t r[8];
};

/* One DP program record per row: a = code index (8) | in-degree (7) | sink (1) | pred0 | pred1 | pred2,
 * b = pred3..pred6 (DP ranks, 0 = virtual root row).  In-degrees above 7 spill to pred_ovf. */
struct alignas(16) Rec {
    uint64_t a, b;
};
RP_DEV uint32_t rec_pred(const Rec& r, uint32_t k) {  // k < 7
    return k < 3 ? (static_cast<uint32_t>(r.a >> (16 + 16 * k)) & 0xffffu)
                 : (static_cast<uint32_t>(r.b >> (16 * (k - 3))) & 0xffffu);
}

struct alignas(16) U4 {
    uint32_t x, y, z, w;
};
struct alignas(8) U2 {
    uint32_t x, y;
};

/* A lane's 16 columns = two 16-byte granules 2*lane, 2*lane+1 of the row (chunk or band) it belongs to */
RP_DEV Row8 load_row_smem(const int16_t* row, int lane) {
    uint32_t q0 = 2u * static_cast<uint32_t>(lane);
    uint32_t p0 = q0 ^ ((q0 >> 3) & 1u);
    uint32_t p1 = (q0 + 1u) ^ (((q0 + 1u) >> 3) & 1u);
    const U4* b = reinterpret_cast<const U4*>(row);
    U4 a = b[p0], c = b[p1];
    Row8 o;
    o.r[0] = a.x; o.r[1] = a.y; o.r[2] = a.z; o.r[3] = a.w;
    o.r[4] = c.x; o.r[5] = c.y; o.r[6] = c.z; o.r[7] = c.w;
    return o;
}
/* the same with the lane's two (swizzled) granule indices handed in: dp() derives them once per alignment */
RP_DEV Row8 load_row_smem_at(const int16_t* row, uint32_t p0, uint32_t p1) {
    const U4* b = reinterpret_cast<const U4*>(row);
    U4 a = b[p0], c = b[p1];
    Row8 o;
    o.r[0] = a.x; o.r[1] = a.y; o.r[2] = a.z; o.r[3] = a.w;
    o.r[4] = c.x; o.r[5] = c.y; o.r[6] = c.z; o.r[7] = c.w;
    return o;
}
RP_DEV void store_row_smem_at(int16_t* row, uint32_t p0, uint32_t p1, const Row8& v) {
    U4* b = reinterpret_cast<U4*>(row);
    b[p0] = U4{v.r[0], v.r[1], v.r[2], v.r[3]};
    b[p1] = U4{v.r[4], v.r[5], v.r[6], v.r[7]};
}
RP_DEV void store_row_smem(int16_t* row, int lane, const Row8& v) {
    uint32_t q0 = 2u * static_cast<uint32_t>(lane);
    uint32_t p0 = q0 ^ ((q0 >> 3) & 1u);
    uint32_t p1 = (q0 + 1u) ^ (((q0 + 1u) >> 3) & 1u);
    U4* b = reinterpret_cast<U4*>(row);
    b[p0] = U4{v.r[0], v.r[1], v.r[2], v.r[3]};
    b[p1] = U4{v.r[4], v.r[5], v.r[6], v.r[7]};
}
RP_DEV Row8 load_row_gmem(const int16_t* row, int lane) {
    const U4* b = reinterpret_cast<const U4*>(row) + 2u * static_cast<uint32_t>(lane);
    U4 a = b[0], c = b[1];
    Row8 o;
    o.r[0] = a.x; o.r[1] = a.y; o.r[2] = a.z; o.r[3] = a.w;
    o.r[4] = c.x; o.r[5] = c.y; o.r[6] = c.z; o.r[7] = c.w;
    return o;
}
/* A row that has left the shared-memory ring (2 % of the predecessors), fetched from the HBM copy by an out-of-line helper,
 * 8 bytes per call: kept out of line on purpose — inlined, the compiler turns the rare branch into ~18 predicated-off
 * instructions that every predecessor of every row then issues. */
static RP_DEV_NOINLINE uint64_t load_far_u64(const int16_t* row, uint32_t idx) {
    return reinterpret_cast<const uint64_t*>(row)[idx];
}
RP_DEV Row8 load_row_far(const int16_t* row, int lane) {
    Row8 o;
#pragma unroll
    for (uint32_t k = 0; k < 4; ++k) {
        const uint64_t v = load_far_u64(row, 4u * static_cast<uint32_t>(lane) + k);
        o.r[2 * k] = static_cast<uint32_t>(v);
        o.r[2 * k + 1] = static_cast<uint32_t>(v >> 32);
    }
    return o;
}
RP_DEV void store_row_gmem(int16_t* row, int lane, const Row8& v) {
    U4* b = reinterpret_cast<U4*>(row) + 2u * static_cast<uint32_t>(lane);
    b[0] = U4{v.r[0], v.r[1], v.r[2], v.r[3]};
    b[1] = U4{v.r[4], v.r[5], v.r[6], v.r[7]};
}

/* One lane group's view of its scratch slot + shared memory (G lanes = one window; rp_warp.cuh "lane groups").
 * All scalar members are group-uniform.  The collectives the code below calls unqualified (syncwarp, ballot, shfl,
 * ...) are the member versions declared here: they span the G lanes of this group only. */
template <int G, int KB = 16>
struct PoaWarp {
    static constexpr uint32_t kCC = 16u * G;   // full matrix: columns of a register-resident row chunk (16 per lane)
    /* banded rows: KB columns per lane (16, 8 or 4) => a band of G*KB columns = NB blocks of 16 columns, each block
     * spread over LPB neighbouring lanes, R packed int16x2 registers per lane */
    static constexpr uint32_t kBW = static_cast<uint32_t>(G) * KB;
    static constexpr uint32_t NB = kBW / 16u;
    static constexpr uint32_t LPB = 16u / KB;
    static constexpr int R = KB / 2;
    static_assert(KB == 16 || KB == 8 || KB == 4, "columns per lane of a banded row");
    static_assert(NB >= 2 && (NB & (NB - 1)) == 0, "blocks per band must be a power of two");

    /* element index, inside a band row, of logical column c (low 4 bits: place inside its 16-column block): lane q of
     * the block holds columns q*KB .. q*KB+KB-1 as registers r = k mod R, half = k div R (k = column inside the lane) */
    static RP_DEV uint32_t perm_band(uint32_t c) {
        if (KB == 16) return perm(c);
        const uint32_t ib = c & 15u, q = ib / KB, k = ib % KB;
        return (c & ~15u) | (q * KB + ((k % R) << 1) + (k / R));
    }
    static RP_DEV uint32_t unperm_band(uint32_t el) {   // inverse of perm_band inside one block (el = 0..15)
        const uint32_t q = el / KB, w = el % KB;
        return q * KB + (w >> 1) + (w & 1u) * R;
    }
    struct RowB {
        uint32_t r[R];
    };
    /* a lane's R registers of a band row in shared memory / HBM (lane-contiguous; 16-column lanes use the swizzled
     * two-granule layout of the full rows) */
    static RP_DEV RowB load_band_smem(const int16_t* row, int lane) {
        RowB o;
        if constexpr (R == 8) {
            const Row8 t = load_row_smem(row, lane);
#pragma unroll
            for (int r = 0; r < R; ++r) o.r[r] = t.r[r];
        } else if constexpr (R == 4) {
            const U4 t = reinterpret_cast<const U4*>(row)[lane];
            o.r[0] = t.x; o.r[1] = t.y; o.r[2] = t.z; o.r[3] = t.w;
        } else {
            const U2 t = reinterpret_cast<const U2*>(row)[lane];
            o.r[0] = t.x; o.r[1] = t.y;
        }
        return o;
    }
    static RP_DEV void store_band_smem(int16_t* row, int lane, const RowB& v) {
        if constexpr (R == 8) {
            Row8 t;
#pragma unroll
            for (int r = 0; r < R; ++r) t.r[r] = v.r[r];
            store_row_smem(row, lane, t);
        } else if constexpr (R == 4) {
            reinterpret_cast<U4*>(row)[lane] = U4{v.r[0], v.r[1], v.r[2], v.r[3]};
        } else {
            reinterpret_cast<U2*>(row)[lane] = U2{v.r[0], v.r[1]};
        }
    }
    static RP_DEV RowB load_band_gmem(const int16_t* row, int lane) {
        RowB o;
        if constexpr (R == 8) {
            const Row8 t = load_row_gmem(row, lane);
#pragma unroll
            for (int r = 0; r < R; ++r) o.r[r] = t.r[r];
        } else if constexpr (R == 4) {
            const U4 t = reinterpret_cast<const U4*>(row)[lane];
            o.r[0] = t.x; o.r[1] = t.y; o.r[2] = t.z; o.r[3] = t.w;
        } else {
            const U2 t = reinterpret_cast<const U2*>(row)[lane];
            o.r[0] = t.x; o.r[1] = t.y;
        }
        return o;
    }
    static RP_DEV void store_band_gmem(int16_t* row, int lane, const RowB& v) {
        if constexpr (R == 8) {
            Row8 t;
#pragma unroll
            for (int r = 0; r < R; ++r) t.r[r] = v.r[r];
            store_row_gmem(row, lane, t);
        } else if constexpr (R == 4) {
            reinterpret_cast<U4*>(row)[lane] = U4{v.r[0], v.r[1], v.r[2], v.r[3]};
        } else {
            reinterpret_cast<U2*>(row)[lane] = U2{v.r[0], v.r[1]};
        }
    }
    /* where column c of a band row sits in a shared-memory ring row */
    static RP_DEV uint32_t band_elem_smem(uint32_t c) {
        const uint32_t e = (((c >> 4) & (NB - 1)) << 4) | (perm_band(c) & 15u);
        return KB == 16 ? swz_e(e) : e;
    }
    static RP_DEV void syncwarp() { gsync<G>(); }
    static RP_DEV uint32_t ballot(bool p) { return gballot<G>(p); }
    template <typename T> static RP_DEV T shfl(T v, int src) { return gshfl<G, T>(v, src); }
    template <typename T> static RP_DEV T shfl_up(T v, int d) { return gshfl_up<G, T>(v, d); }
    template <typename T> static RP_DEV T shfl_down(T v, int d) { return gshfl_down<G, T>(v, d); }
    static RP_DEV uint32_t warp_rank(bool p, uint32_t* total) { return grank<G>(p, total); }
    static RP_DEV uint32_t warp_incl_sum(uint32_t v) { return gincl_sum<G>(v); }
    static RP_DEV int32_t warp_incl_max(int32_t v) { return gincl_max<G>(v); }

    const PoaParams* P;
    int lane;
    /* graph (HBM) */
    uint8_t *code, *flags, *in_cnt, *al_cnt, *member, *has_out_sub, *marks;
    uint16_t *cov, *in_tail, *al, *order, *order_nxt, *rank_of, *dp_order, *dp_rank, *pred_ovf, *aln, *cur, *cpred,
        *sorder, *srank, *stack;
    int32_t* in_w;
    Rec* rec;
    int16_t* H;
    int64_t* score;
    uint32_t* newlist;
    int16_t* ccarry;
    uint16_t* bpos;      // per node: backbone coordinate it sits at (band centre line)
    uint8_t* bs;         // per DP row: first 16-column block of the row's band
    /* shared memory */
    int16_t* ring;       // ring_rows x lp_a
    int16_t* prof;       // ncodes x lp_a
    uint8_t* smem;
    uint32_t smem_bytes;
    /* state */
    uint32_t N;          // nodes
    uint32_t ki, ka, nmax;
    uint32_t status;
    uint64_t alpha;
    uint32_t ncodes;
    uint32_t n_added;    // sequences merged so far (incl. backbone)

    RP_DEV void bind(const PoaParams* p, uint8_t* slot, uint8_t* sm, uint32_t sm_bytes) {
        P = p;
        lane = glane<G>();
        const SlotLayout& y = p->lay;
        code = slot + y.code;
        flags = slot + y.flags;
        in_cnt = slot + y.in_cnt;
        al_cnt = slot + y.al_cnt;
        cov = reinterpret_cast<uint16_t*>(slot + y.cov);
        in_tail = reinterpret_cast<uint16_t*>(slot + y.in_tail);
        in_w = reinterpret_cast<int32_t*>(slot + y.in_w);
        al = reinterpret_cast<uint16_t*>(slot + y.al);
        order = reinterpret_cast<uint16_t*>(slot + y.order_a);
        order_nxt = reinterpret_cast<uint16_t*>(slot + y.order_b);
        rank_of = reinterpret_cast<uint16_t*>(slot + y.rank_of);
        dp_order = reinterpret_cast<uint16_t*>(slot + y.dp_order);
        dp_rank = reinterpret_cast<uint16_t*>(slot + y.dp_rank);
        rec = reinterpret_cast<Rec*>(slot + y.rec);
        pred_ovf = reinterpret_cast<uint16_t*>(slot + y.pred_ovf);
        H = reinterpret_cast<int16_t*>(slot + y.H);
        aln = reinterpret_cast<uint16_t*>(slot + y.aln);
        cur = reinterpret_cast<uint16_t*>(slot + y.cur);
        member = slot + y.member;
        has_out_sub = slot + y.has_out_sub;
        score = reinterpret_cast<int64_t*>(slot + y.score);
        cpred = reinterpret_cast<uint16_t*>(slot + y.cpred);
        sorder = reinterpret_cast<uint16_t*>(slot + y.sorder);
        srank = reinterpret_cast<uint16_t*>(slot + y.srank);
        marks = slot + y.marks;
        stack = reinterpret_cast<uint16_t*>(slot + y.stack);
        newlist = reinterpret_cast<uint32_t*>(slot + y.newlist);
        ccarry = reinterpret_cast<int16_t*>(slot + y.ccarry);
        bpos = reinterpret_cast<uint16_t*>(slot + y.bpos);
        bs = slot + y.bs;
        smem = sm;
        smem_bytes = sm_bytes;
        ki = p->lim.ki;
        ka = p->lim.ka;
        nmax = p->lim.nmax;
    }

    RP_DEV void fail(uint32_t st) {
        if (status == kWinOk) status = st;
    }

    RP_DEV uint32_t code_index(uint8_t c) const {  // position of character c in the window alphabet
        uint32_t k = 0;
        for (; k < ncodes; ++k)
            if (static_cast<uint8_t>(alpha >> (8 * k)) == c) break;
        return k;
    }

    /* ---------------------------------------------------------------- backbone (graph.cpp:186-190, 93-110) */
    RP_DEV void init_backbone(const uint8_t* seq, const uint8_t* w, uint32_t len) {
        for (uint32_t v = lane; v < len; v += G) {
            code[v] = seq[v];
            al_cnt[v] = 0;
            flags[v] = (v + 1 < len) ? 1 : 0;
            cov[v] = len >= 2 ? 1 : 0;
            if (v > 0) {
                in_cnt[v] = 1;
                in_tail[v * ki] = static_cast<uint16_t>(v - 1);
                in_w[v * ki] = static_cast<int32_t>(w[v - 1]) + static_cast<int32_t>(w[v]);
            } else {
                in_cnt[v] = 0;
            }
            order[v + 1] = static_cast<uint16_t>(v);
            rank_of[v] = static_cast<uint16_t>(v + 1);
            bpos[v] = static_cast<uint16_t>(v);
        }
        if (lane == 0) order[0] = kNone;
        N = len;
        n_added = 1;
        syncwarp();
    }

    /* ---------------------------------------------------------------- subgraph (graph.cpp:518-539) */
    /* Backward DFS from backbone node `end` over in-edges and aligned nodes, keeping ids >= begin.
     * Serial (lane 0); only partial-span layers take this path. */
    RP_DEV void mark_subgraph(uint32_t begin, uint32_t end) {
        const uint32_t npad = (N + 15) & ~15u;
        bool staged = ki <= 31 && ka == 8 && 2 * npad + 512 <= smem_bytes && !(P->debug_flags & 1);
        if (staged && !mark_subgraph_staged(begin, end, npad)) staged = false;  // stack outgrew shared memory
        if (!staged) {  /* HBM-resident variant */
            for (uint32_t v = lane; v < N; v += G) member[v] = 0;
            syncwarp();
            if (lane == 0) {
                uint32_t sp = 0;
                const uint32_t cap = P->lim.stack_cap;
                stack[sp++] = static_cast<uint16_t>(end);
                while (sp > 0) {
                    uint32_t c = stack[--sp];
                    if (member[c] || c < begin) continue;
                    uint32_t ni = in_cnt[c], na = al_cnt[c];
                    if (sp + ni + na > cap) {
                        fail(kWinStackLimit);
                        break;
                    }
                    for (uint32_t k = 0; k < ni; ++k) stack[sp++] = in_tail[c * ki + k];
                    for (uint32_t k = 0; k < na; ++k) stack[sp++] = al[c * ka + k];
                    member[c] = 1;
                }
            }
            status = shfl(status, 0);
            syncwarp();
        }
    }

    /* membership bytes, per-node degrees, the first two in-edge tails of every node and the stack live in
     * shared memory: a node costs an HBM round trip only if it has more than two in-edges or aligned nodes.
     * Returns false (nothing decided) when the stack does not fit. */
    RP_DEV bool mark_subgraph_staged(uint32_t begin, uint32_t end, uint32_t npad) {
        uint8_t* smb = smem;
        uint8_t* sme = smem + npad;
        const bool have_t2 = 6 * npad + 1024 <= smem_bytes;
        uint32_t* st2 = reinterpret_cast<uint32_t*>(smem + 2 * npad);
        const uint32_t fixed = have_t2 ? 6 * npad : 2 * npad;
        uint16_t* sst = reinterpret_cast<uint16_t*>(smem + fixed);
        const uint32_t cap = (smem_bytes - fixed) / 2;
        for (uint32_t v = lane; v < N; v += G) {
            smb[v] = 0;
            sme[v] = static_cast<uint8_t>(in_cnt[v] | (al_cnt[v] << 5));
            if (have_t2) st2[v] = *reinterpret_cast<const uint32_t*>(in_tail + v * ki);
        }
        syncwarp();
        uint32_t ovf = 0;
        if (lane == 0) {
            uint32_t sp = 0;
            sst[sp++] = static_cast<uint16_t>(end);
            while (sp > 0) {
                const uint32_t c = sst[--sp];
                if (smb[c] || c < begin) continue;
                const uint32_t ni = sme[c] & 31u, na = sme[c] >> 5;
                uint64_t t4 = have_t2 ? st2[c] : 0;
                if (!have_t2 || ni > 2) t4 = *reinterpret_cast<const uint64_t*>(in_tail + c * ki);
                uint64_t a_lo = 0, a_hi = 0;
                if (na) {
                    const U4 a8 = *reinterpret_cast<const U4*>(al + c * ka);
                    a_lo = a8.x | (static_cast<uint64_t>(a8.y) << 32);
                    a_hi = a8.z | (static_cast<uint64_t>(a8.w) << 32);
                }
                if (sp + ni + na > cap) {
                    ovf = 1;
                    break;
                }
                for (uint32_t k = 0; k < ni; ++k) {
                    const uint32_t t = k < 4 ? (static_cast<uint32_t>(t4 >> (16 * k)) & 0xffffu) : in_tail[c * ki + k];
                    if (!smb[t] && t >= begin) sst[sp++] = static_cast<uint16_t>(t);
                }
                for (uint32_t k = 0; k < na; ++k) {
                    const uint32_t a = static_cast<uint32_t>((k < 4 ? a_lo : a_hi) >> (16 * (k & 3))) & 0xffffu;
                    if (!smb[a] && a >= begin) sst[sp++] = static_cast<uint16_t>(a);
                }
                smb[c] = 1;
            }
        }
        ovf = shfl(ovf, 0);
        syncwarp();
        if (ovf) return false;
        for (uint32_t v = lane; v < N; v += G) member[v] = smb[v];
        syncwarp();
        return true;
    }

    /* Compact DP order over the member nodes (rank order preserved). Returns number of DP rows. */
    RP_DEV uint32_t build_dp_order_subgraph() {
        uint32_t base = 0;
        for (uint32_t r0 = 1; r0 <= N; r0 += G) {
            uint32_t r = r0 + lane;
            uint32_t v = r <= N ? order[r] : 0;
            bool in = r <= N && member[v];
            uint32_t tot;
            uint32_t pos = warp_rank(in, &tot);
            if (in) {
                dp_order[base + pos + 1] = static_cast<uint16_t>(v);
                dp_rank[v] = static_cast<uint16_t>(base + pos + 1);
            }
            base += tot;
        }
        for (uint32_t v = lane; v < N; v += G) has_out_sub[v] = 0;
        syncwarp();
        /* sinks of the subgraph: members without an out-edge to another member (graph.cpp:575-580) */
        for (uint32_t v = lane; v < N; v += G) {
            if (!member[v]) continue;
            uint32_t ni = in_cnt[v];
            for (uint32_t k = 0; k < ni; ++k) {
                uint32_t t = in_tail[v * ki + k];
                if (member[t]) has_out_sub[t] = 1;
            }
        }
        syncwarp();
        return base;
    }

    /* ---------------------------------------------------------------- DP program (one 8-byte record per row)
     * byte0 code index, byte1 = npred(7 bits) | sink<<7, bytes2..7 = first three predecessor DP ranks
     * (0 = virtual root row).  Further predecessors spill to pred_ovf. */
    /* With `band`, also the first 16-column block bs[r] of every row's band: the band (16*G columns) is centred on
     * the column the node's backbone coordinate maps to, (bpos - b0) * (len + 1) / span, and never moves left
     * along the processing order. */
    RP_DEV uint32_t build_program(uint32_t nrows, bool sub, bool band, uint32_t len, uint32_t b0, uint32_t span) {
        const uint16_t* ord = sub ? dp_order : order;
        const uint16_t* rk = sub ? dp_rank : rank_of;
        uint32_t pred_rows = 0;
        const uint32_t nblk = (len + 16) >> 4;            // blocks holding columns 0..len
        const int32_t smax = static_cast<int32_t>(nblk) - static_cast<int32_t>(NB);
        int32_t brun = 0;
        /* The graph lives in HBM, so every level of the chain row -> node -> in-edges -> ranks costs a full
         * memory latency.  Rows are handled kU per lane at a time with all loads of one level issued together. */
        constexpr int kU = 4;
        for (uint32_t r0 = 1; r0 <= nrows; r0 += G * kU) {
            uint32_t r[kU], v[kU], ni[kU], cd[kU], fl[kU], bp[kU];
            uint64_t t4[kU];
            uint32_t pk[kU][3];
            bool use[kU][3];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                r[u] = r0 + u * G + lane;
                v[u] = r[u] <= nrows ? ord[r[u]] : ord[1];
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                ni[u] = in_cnt[v[u]];
                cd[u] = code[v[u]];
                fl[u] = sub ? has_out_sub[v[u]] : (flags[v[u]] & 1u);
                t4[u] = *reinterpret_cast<const uint64_t*>(in_tail + v[u] * ki);  // first four in-edge tails
                bp[u] = band ? bpos[v[u]] : 0u;
            }
            if (band) {
#pragma unroll
                for (int u = 0; u < kU; ++u) {
                    uint32_t x = bp[u] > b0 ? bp[u] - b0 : 0u;
                    if (x >= span) x = span - 1;
                    const int32_t cc = static_cast<int32_t>((x * (len + 1)) / span);
                    int32_t t = (cc + 8) / 16 - static_cast<int32_t>(NB) / 2;
                    t = t > smax ? smax : t;
                    t = t < 0 ? 0 : t;
                    if (r[u] > nrows) t = 0;
                    int32_t inc = warp_incl_max(t);
                    inc = inc < brun ? brun : inc;
                    if (r[u] <= nrows) bs[r[u]] = static_cast<uint8_t>(inc);
                    brun = shfl(inc, G - 1);
                }
            }
#pragma unroll
            for (int u = 0; u < kU; ++u)
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    uint32_t t = static_cast<uint32_t>(t4[u] >> (16 * k)) & 0xffffu;
                    use[u][k] = static_cast<uint32_t>(k) < ni[u] && (!sub || member[t]);
                    pk[u][k] = t;
                }
#pragma unroll
            for (int u = 0; u < kU; ++u)
#pragma unroll
                for (int k = 0; k < 3; ++k) pk[u][k] = use[u][k] ? rk[pk[u][k]] : 0u;
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                if (r[u] > nrows) continue;
                uint32_t np = 0;
                uint64_t pa = 0, pb = 0;
                auto put = [&](uint32_t pr) {
                    if (np < 3)
                        pa |= static_cast<uint64_t>(pr) << (16 + 16 * np);
                    else if (np < 7)
                        pb |= static_cast<uint64_t>(pr) << (16 * (np - 3));
                    else
                        pred_ovf[r[u] * ki + np] = static_cast<uint16_t>(pr);
                    ++np;
                };
#pragma unroll
                for (int k = 0; k < 3; ++k)
                    if (use[u][k]) put(pk[u][k]);
                for (uint32_t k = 3; k < ni[u]; ++k) {  // less common: in-degree > 3
                    uint32_t t = in_tail[v[u] * ki + k];
                    if (sub && !member[t]) continue;
                    put(rk[t]);
                }
                bool sink = !fl[u];
                Rec rc;
                rc.a = static_cast<uint64_t>(code_index(static_cast<uint8_t>(cd[u]))) |
                       (static_cast<uint64_t>(np & 0x7f) << 8) | (static_cast<uint64_t>(sink ? 1 : 0) << 15) | pa;
                rc.b = pb;
                rec[r[u]] = rc;
                pred_rows += np ? np : 1;
            }
        }
        if (lane == 0) {
            rec[0] = Rec{0, 0};
            bs[0] = 0;
        }
        syncwarp();
        return pred_rows;  // per-lane partial sum (only summed when the device counters are on)
    }

    /* ---------------------------------------------------------------- the DP (sisd :292-360, simd :760-906)
     * Column c of a row holds H[row][c] for c = 0..len (column 0 is spoa's first_column); column -1 is
     * -infinity, which makes column 0 follow the general recurrence.  Returns the best sink row
     * (first strictly greater in processing order) in *best_row, its score, and the number of sink rows
     * that reach that score. */
    /* one 512-column chunk of the match/mismatch profile (sisd :123-131) into shared memory */
    RP_DEV void build_profile(const uint8_t* seq, uint32_t len, uint32_t ch) {
        int32_t m = P->match, x = P->mismatch;
        for (uint32_t k = 0; k < ncodes; ++k) {
            uint8_t c = static_cast<uint8_t>(alpha >> (8 * k));
            int16_t* row = prof + k * kCC;
            for (uint32_t cc = lane; cc < kCC; cc += G) {
                uint32_t col = ch * kCC + cc;
                int16_t v = static_cast<int16_t>(x);
                if (col >= 1 && col <= len && seq[col - 1] == c) v = static_cast<int16_t>(m);
                row[swz(cc)] = v;
            }
        }
    }

    /* True iff no cell of the finished matrix can have left the range int16 arithmetic is exact in.  Every cell
     * satisfies H[i][j] >= H[i][0] + j*g (the horizontal move is always a candidate), column 0 falls by exactly |g|
     * per level along a shortest path (so it cannot jump over the limit unnoticed), and the largest value is bounded
     * by max(match, mismatch) * min(rows, columns), checked by the caller.  Limit: spoa's own margin, -32768 + 1024. */
    RP_DEV bool matrix_in_range(uint32_t nrows, uint32_t len, uint32_t lpa) {
        int32_t mn = 0;
        const uint32_t e0 = perm(0);
        for (uint32_t i = 1 + lane; i <= nrows; i += G) {
            const int32_t v = H[static_cast<uint64_t>(i) * lpa + e0];
            mn = v < mn ? v : mn;
        }
        mn = -warp_incl_max(-mn);
        mn = shfl(mn, G - 1);
        return mn + static_cast<int32_t>(len) * P->gap >= -32768 + 1024;
    }

    RP_DEV void dp(const uint8_t* seq, uint32_t nrows, uint32_t len, uint32_t lpa, uint32_t ring_rows,
                   uint32_t* best_row, int32_t* best_score, uint32_t* n_best) {
        /* rows of one 512-column chunk (every window of up to 511 bases: the common case) get a copy of the row loop
         * without the chunk-carry code, which otherwise rides along as ~14 predicated-off instructions per row */
        if (lpa / kCC > 1)
            dp_rows<true>(seq, nrows, len, lpa, ring_rows, best_row, best_score, n_best);
        else
            dp_rows<false>(seq, nrows, len, lpa, ring_rows, best_row, best_score, n_best);
    }

    template <bool CHUNKS>
    RP_DEV void dp_rows(const uint8_t* seq, uint32_t nrows, uint32_t len, uint32_t lpa, uint32_t ring_rows,
                        uint32_t* best_row, int32_t* best_score, uint32_t* n_best) {
        /* Row-synchronous: the whole warp computes one row (512-column chunk) at a time; lane l owns columns
         * 16l..16l+15.  Rows longer than 512 columns are done chunk by chunk (one pass over all rows per chunk,
         * the carry between chunks goes through a small per-row array), so shared memory only ever holds one
         * chunk: the profile chunk and a ring of the last `ring_rows` rows. */
        const int32_t g = P->gap;
        const uint32_t g2 = P->row_consts[16];
        const uint32_t nch = CHUNKS ? lpa / kCC : 1u;
        const int32_t negsafe = -32768 - 16 * g;  // see kMaxGapInt16
        const uint32_t* gb = P->row_consts;       // bridge / carry offsets per register (constant bank, see PoaParams)
        const uint32_t* gc = P->row_consts + 8;
        for (uint32_t col = lane; col < lpa; col += G) H[perm(col)] = static_cast<int16_t>(static_cast<int32_t>(col) * g);
        const uint32_t sink_ch = len / kCC, sink_e = swz(len % kCC);
        int32_t best = kNeg32;
        uint32_t bi = 0, nb = 0;
        int16_t* cc_prev = ccarry;        // last column of the previous chunk, per row (multi-chunk rows only)
        int16_t* cc_cur = ccarry + (nmax + 2);
        const uint32_t lanem = static_cast<uint32_t>(lane);
        /* this lane's two granules of a shared-memory row (load_row_smem's swizzle), pinned in registers for the row
         * loop: re-derived per row they start every row's dependency chain with an S2R of the thread index */
        uint32_t sw0 = (2u * lanem) ^ (((2u * lanem) >> 3) & 1u);
        uint32_t sw1 = (2u * lanem + 1u) ^ (((2u * lanem + 1u) >> 3) & 1u);
        RP_KEEP_IN_REGISTER(sw0);
        RP_KEEP_IN_REGISTER(sw1);
        for (uint32_t ch = 0; ch < nch; ++ch) {
            build_profile(seq, len, ch);
            for (uint32_t c = lane; c < kCC; c += G)  // root row (rank 0) -> ring slot 0
                ring[swz(c)] = static_cast<int16_t>(static_cast<int32_t>(ch * kCC + c) * g);
            syncwarp();
            const bool multi = CHUNKS && ch > 0;
            /* columns beyond the read's last one are computed but never read by anything that matters (dependencies run
             * left to right and the walk starts at column len): lanes that only hold such columns do not vote */
            const bool scan_lane = ch * kCC + lanem * 16u <= len;
            uint32_t rec_a_lo = 0, rec_a_hi = 0, rec_b_lo = 0, rec_b_hi = 0;
            int16_t* hrow = H + static_cast<uint64_t>(ch) * kCC;  // row i of this chunk = hrow + i*lpa
            uint32_t myslot = 0;  // i % ring_rows, kept incrementally (any ring size, no division)
            /* where this lane stores its 16 columns of row i in the HBM copy: a running pointer (rows come in order), so
             * that the row loop carries one 64-bit add instead of rebuilding the address from the parameter block */
            U4* hst = reinterpret_cast<U4*>(hrow + lpa) + 2u * lanem;
            Row8 prev;            // the row computed last (this lane's registers of it)
#pragma unroll
            for (int r = 0; r < 8; ++r) prev.r[r] = 0;
            /* rows in blocks of G: lane l fetches the record of row i0 + l once per block (a loop level of its own, so that
             * the row loop carries no predicated-off copy of the fetch), every row then takes its record by shuffle */
            Rec nxt = rec[1 + lane];  // rec[] is padded (SlotLayout: + 160 records)
            for (uint32_t i0 = 1; i0 <= nrows; i0 += G) {
              {
                  /* this block's records were requested one block ago: their HBM latency ran under 32 rows of work */
                  rec_a_lo = static_cast<uint32_t>(nxt.a);
                  rec_a_hi = static_cast<uint32_t>(nxt.a >> 32);
                  rec_b_lo = static_cast<uint32_t>(nxt.b);
                  rec_b_hi = static_cast<uint32_t>(nxt.b >> 32);
                  nxt = rec[i0 + G + lane];
              }
              const uint32_t i_last = i0 + G - 1 < nrows ? i0 + G - 1 : nrows;
              uint32_t lo_next = shfl(rec_a_lo, 0);
              for (uint32_t i = i0; i <= i_last; ++i) {
                myslot = myslot + 1 == ring_rows ? 0u : myslot + 1;
                const uint32_t ti = i - i0;
                /* the record word of the NEXT row is shuffled out now: its latency runs under this row */
                const uint32_t lo = lo_next;
                lo_next = shfl(rec_a_lo, (ti + 1) & (G - 1));
                const uint32_t cidx = lo & 0xff;
                const uint32_t np = (lo >> 8) & 0x7f;
                const bool sink = (lo >> 15) & 1;
                const Row8 pf = load_row_smem_at(prof + cidx * kCC, sw0, sw1);
                /* max over predecessors distributes over both terms of the recurrence:
                 *   max_p(H[p][c-1] + s(c), H[p][c] + g) = max(max_p H[p][c-1] + s(c), max_p H[p][c] + g),
                 * so predecessor rows are first combined with a packed max (8 ops per extra predecessor) and the
                 * diagonal/vertical update (16 DPX ops, one shuffle) runs once per row */
                Row8 pm;
                int32_t lvm = kNegDiag;
                auto load_pred = [&](uint32_t p, Row8& pr) {
                    const uint32_t dist = i - p;
                    if (__builtin_expect(dist < ring_rows, 1)) {  // warp-uniform; 98 % of the predecessors
                        const uint32_t slot = myslot >= dist ? myslot - dist : myslot + ring_rows - dist;
                        pr = load_row_smem_at(ring + slot * kCC, sw0, sw1);
                    } else
                        pr = load_row_far(hrow + static_cast<uint64_t>(p) * lpa, lane);
                    if (multi) {
                        int32_t lv = cc_prev[p];
                        lvm = lv > lvm ? lv : lvm;
                    }
                };
                auto more = [&](uint32_t p) {
                    Row8 pr;
                    load_pred(p, pr);
#pragma unroll
                    for (int r = 0; r < 8; ++r) pm.r[r] = vmax_s16x2(pm.r[r], pr.r[r]);
                };
                /* the first predecessor is loaded by every group of the warp together; only the groups whose row has
                 * more predecessors enter the nested part */
                {
                    const uint32_t p0 = np ? (lo >> 16) : 0u;
                    if (p0 + 1 == i && p0 != 0) {  // group-uniform
                        /* the first predecessor is the row just computed (4 of 10 rows): it still is in registers — no
                         * trip through the shared-memory ring, whose store -> load latency would start this row */
                        pm = prev;
                        if (multi) {
                            int32_t lv = cc_prev[p0];
                            lvm = lv > lvm ? lv : lvm;
                        }
                    } else {
                        load_pred(p0, pm);
                    }
                }
                if (np > 1) {
                    const uint32_t hi = shfl(rec_a_hi, ti);
                    more(hi & 0xffff);
                    if (np > 2) {
                        more(hi >> 16);
                        if (np > 3) {
                            const uint32_t blo = shfl(rec_b_lo, ti), bhi = shfl(rec_b_hi, ti);
                            more(blo & 0xffff);
                            if (np > 4) more(blo >> 16);
                            if (np > 5) more(bhi & 0xffff);
                            if (np > 6) more(bhi >> 16);
                            for (uint32_t k = 7; k < np; ++k) more(pred_ovf[i * ki + k]);
                        }
                    }
                }
                uint32_t acc[8];
                {
                    uint32_t left = shfl_up(pm.r[7], 1);  // hi half = previous lane's last column
                    left = lanem == 0 ? (static_cast<uint32_t>(lvm) << 16) : left;
                    /* diagonal operand of register 0 = (column -1 of the block, column 7) */
                    const uint32_t d0 = byte_perm(left, pm.r[7], 0x5432);
                    acc[0] = viaddmax_s16x2(pm.r[0], g2, viaddmax_s16x2(d0, pf.r[0], 0x80008000u));
#pragma unroll
                    for (int r = 1; r < 8; ++r)
                        acc[r] = viaddmax_s16x2(pm.r[r], g2, viaddmax_s16x2(pm.r[r - 1], pf.r[r], 0x80008000u));
                }
                /* in-row gap recurrence H[c] = max(H[c], H[c-1] + g), all in packed int16:
                 * two 8-long chains (low halves = columns 0..7, high halves = columns 8..15 of the block) */
#pragma unroll
                for (int r = 1; r < 8; ++r) acc[r] = viaddmax_s16x2(acc[r - 1], g2, acc[r]);
                /* bridge: column 7 feeds columns 8..15 */
                const uint32_t bridge = byte_perm(acc[7], 0x80008000u, 0x1076);  // lo = INT16_MIN, hi = acc[7].lo
#pragma unroll
                for (int r = 0; r < 8; ++r) acc[r] = viaddmax_s16x2(bridge, gb[r], acc[r]);
                /* warp max-plus scan of the lane totals (column 15 of each block), decay 16*g per lane */
                int32_t chunk_carry = kNeg32;
                if (multi) chunk_carry = cc_prev[i];
                int32_t t = hi16(acc[7]);
                /* Short cut: if no lane's total is raised by what its left neighbour hands over (neighbour's total +
                 * 16 gaps), no carry travels further than one lane and the carry into a lane is simply the neighbour's
                 * total — one shuffle and a vote instead of the five dependent scan steps.  (Right of the alignment
                 * path the gap-extended values tie with the diagonal ones already in the row, so this is the common
                 * case; the scan stays for the rows where a long gap run really wins.) */
                int32_t carry = shfl_up(t, 1);
                carry = lanem == 0 ? chunk_carry : carry;
                if (ballot(scan_lane && carry + 16 * g > t)) {  // group-uniform
                    t = viaddmax_s32(lanem == 0 ? chunk_carry : kNeg32, 16 * g, t);
#pragma unroll
                    for (int dd = 1; dd < G; dd <<= 1) {
                        int32_t o = shfl_up(t, dd);
                        t = viaddmax_s32(lanem >= static_cast<uint32_t>(dd) ? o : kNeg32, dd * 16 * g, t);
                    }
                    carry = shfl_up(t, 1);
                    carry = lanem == 0 ? chunk_carry : carry;
                }
                carry = carry < negsafe ? negsafe : carry;
                const uint32_t c2 = pack16(carry, carry);
#pragma unroll
                for (int r = 0; r < 8; ++r) acc[r] = viaddmax_s16x2(c2, gc[r], acc[r]);
                Row8 out;
#pragma unroll
                for (int r = 0; r < 8; ++r) out.r[r] = acc[r];
                prev = out;
                int16_t* myrow_s = ring + myslot * kCC;
                store_row_smem_at(myrow_s, sw0, sw1, out);
                hst[0] = U4{out.r[0], out.r[1], out.r[2], out.r[3]};
                hst[1] = U4{out.r[4], out.r[5], out.r[6], out.r[7]};
                hst += CHUNKS ? lpa / 8u : kCC / 8u;   // next row (a U4 holds 8 cells; one chunk: lpa == kCC)
                if (CHUNKS && lanem == G - 1) cc_cur[i] = static_cast<int16_t>(hi16(acc[7]));
                syncwarp();
                if (sink && ch == sink_ch) {  // warp-uniform
                    int32_t sc = myrow_s[sink_e];
                    if (sc > best) {
                        best = sc;
                        bi = i;
                        nb = 1;
                    } else if (sc == best) {
                        ++nb;
                    }
                }
              }
            }
            if (CHUNKS) {
                if (lane == 0) cc_cur[0] = static_cast<int16_t>((ch + 1) * kCC * g - g);  // root row, last column
                int16_t* tmp = cc_prev;
                cc_prev = cc_cur;
                cc_cur = tmp;
                syncwarp();
            }
        }
        *best_row = bi;
        *best_score = best;
        *n_best = nb;
        syncwarp();
    }

    /* ---------------------------------------------------------------- banded DP (racon -b)
     * Row i only computes the 16*G columns of its band, blocks [bs[i], bs[i] + G).  A 16-column block cb always
     * lives in lane cb mod G — in registers, in the shared-memory ring and in the HBM copy (row pitch = band
     * width) — so when the band slides right only the lane whose block left the band changes its columns, and a
     * predecessor row lines up with the current row without any data movement.  Cells outside a row's band count
     * as minus infinity (kBandFloor, also the floor of every stored cell, so excluded regions cannot wrap around
     * int16): banded values are <= the full matrix's and equal to them on every cell of an optimal path that lies
     * inside the band.  traceback<true> decides whether the result can be trusted. */
    RP_DEV void build_profile_block(const uint8_t* seq, uint32_t len, uint32_t col0) {
        const int32_t m = P->match, x = P->mismatch;
        uint8_t ch[KB];
#pragma unroll
        for (int c = 0; c < KB; ++c) {
            const uint32_t col = col0 + c;
            ch[c] = (col >= 1 && col <= len) ? seq[col - 1] : 0;   // 0 never is a window character
        }
        for (uint32_t k = 0; k < ncodes; ++k) {
            const uint8_t c = static_cast<uint8_t>(alpha >> (8 * k));
            RowB v;
#pragma unroll
            for (int r = 0; r < R; ++r) v.r[r] = pack16(ch[r] == c ? m : x, ch[R + r] == c ? m : x);
            store_band_smem(prof + k * kBW, lane, v);
        }
    }

    RP_DEV void dp_band(const uint8_t* seq, uint32_t nrows, uint32_t len, uint32_t ring_rows, uint32_t* best_row,
                        int32_t* best_score, uint32_t* n_best) {
        const int32_t g = P->gap;
        const uint32_t g2 = pack16(g, g);
        const int32_t negsafe = -32768 - KB * g;
        const uint32_t floor2 = pack16(kBandFloor, kBandFloor);
        uint32_t gb[R], gc[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            gb[r] = pack16(0, (r + 1) * g);
            gc[r] = pack16((r + 1) * g, (r + 1 + R) * g);
        }
        const uint32_t lanem = static_cast<uint32_t>(lane);
        const uint32_t lane_left = (lanem + G - 1) & (G - 1);   // the lane that holds the columns to the left
        const uint32_t sub_lane = lanem & (LPB - 1);            // which KB-column part of its block the lane holds
        const uint32_t sink_blk = len >> 4;
        const uint32_t sink_e = band_elem_smem(len);
        int32_t best = kNeg32;
        uint32_t bi = 0, nb = 0;
        /* rows with the same band start form a segment; predecessors from before the segment need a validity test */
        uint32_t s_cur = 0xffffffffu, seg_i0 = 1, s_prev = 0, prev_i0 = 1;
        uint32_t cb = 0, bo = 0;           // this lane's block and its place in band order (0 = leftmost lane)
        uint32_t pcb = 0xffffffffu;        // block whose profile this lane's profile slot holds
        uint32_t rec_a_lo = 0, rec_a_hi = 0, rec_b_lo = 0, rec_b_hi = 0, bsv = 0;
        uint32_t myslot = 0;
        syncwarp();
        for (uint32_t i = 1; i <= nrows; ++i) {
            myslot = myslot + 1 == ring_rows ? 0u : myslot + 1;
            const uint32_t ti = (i - 1) & (G - 1);
            if (ti == 0) {
                Rec t = rec[i + lane];  // rec[] and bs[] are padded
                rec_a_lo = static_cast<uint32_t>(t.a);
                rec_a_hi = static_cast<uint32_t>(t.a >> 32);
                rec_b_lo = static_cast<uint32_t>(t.b);
                rec_b_hi = static_cast<uint32_t>(t.b >> 32);
                bsv = bs[i + lane];
            }
            const uint32_t lo = shfl(rec_a_lo, ti);
            const uint32_t s_i = shfl(bsv, ti);
            if (s_i != s_cur) {  // group-uniform: the band slides
                s_prev = s_cur;
                prev_i0 = seg_i0;
                s_cur = s_i;
                seg_i0 = i;
                const uint32_t pos = ((lanem / LPB) - s_cur) & (NB - 1);   // block position inside the band
                cb = s_cur + pos;
                bo = pos * LPB + sub_lane;
                if (cb != pcb) {  // only the lanes whose block changed
                    build_profile_block(seq, len, cb * 16u + sub_lane * KB);
                    pcb = cb;
                }
            }
            const uint32_t cidx = lo & 0xff;
            const uint32_t np = (lo >> 8) & 0x7f;
            const bool sink = (lo >> 15) & 1;
            const RowB pf = load_band_smem(prof + cidx * kBW, lane);
            RowB pm;
            auto load_pred = [&](uint32_t p, RowB& pr) {
                if (p == 0) {  // virtual root row: H[0][j] = j * g
                    const int32_t base = static_cast<int32_t>(cb * 16u + sub_lane * KB) * g;
#pragma unroll
                    for (int r = 0; r < R; ++r) pr.r[r] = pack16(base + r * g, base + (R + r) * g);
                    return;
                }
                const uint32_t dist = i - p;
                if (dist < ring_rows) {  // group-uniform
                    const uint32_t slot = myslot >= dist ? myslot - dist : myslot + ring_rows - dist;
                    pr = load_band_smem(ring + slot * kBW, lane);
                } else {
                    pr = load_band_gmem(H + static_cast<uint64_t>(p) * kBW, lane);
                }
                if (p < seg_i0) {  // from an earlier segment: its band may not hold this lane's block
                    const uint32_t sp = p >= prev_i0 ? s_prev : static_cast<uint32_t>(bs[p]);
                    if (cb - sp >= NB) {
#pragma unroll
                        for (int r = 0; r < R; ++r) pr.r[r] = floor2;
                    }
                }
            };
            auto more = [&](uint32_t p) {
                RowB pr;
                load_pred(p, pr);
#pragma unroll
                for (int r = 0; r < R; ++r) pm.r[r] = vmax_s16x2(pm.r[r], pr.r[r]);
            };
            load_pred(np ? (lo >> 16) : 0u, pm);
            if (np > 1) {
                const uint32_t hi = shfl(rec_a_hi, ti);
                more(hi & 0xffff);
                if (np > 2) {
                    more(hi >> 16);
                    if (np > 3) {
                        const uint32_t blo = shfl(rec_b_lo, ti), bhi = shfl(rec_b_hi, ti);
                        more(blo & 0xffff);
                        if (np > 4) more(blo >> 16);
                        if (np > 5) more(bhi & 0xffff);
                        if (np > 6) more(bhi >> 16);
                        for (uint32_t k = 7; k < np; ++k) more(pred_ovf[i * ki + k]);
                    }
                }
            }
            uint32_t acc[R];
            {
                uint32_t left = shfl(pm.r[R - 1], lane_left);  // hi half = last column of the lane to the left
                left = bo == 0 ? floor2 : left;                // leftmost lane of the band: nothing to its left
                const uint32_t d0 = byte_perm(left, pm.r[R - 1], 0x5432);
                acc[0] = viaddmax_s16x2(pm.r[0], g2, viaddmax_s16x2(d0, pf.r[0], floor2));
#pragma unroll
                for (int r = 1; r < R; ++r)
                    acc[r] = viaddmax_s16x2(pm.r[r], g2, viaddmax_s16x2(pm.r[r - 1], pf.r[r], floor2));
            }
#pragma unroll
            for (int r = 1; r < R; ++r) acc[r] = viaddmax_s16x2(acc[r - 1], g2, acc[r]);
            const uint32_t bridge = byte_perm(acc[R - 1], 0x80008000u, 0x1076);  // lo = INT16_MIN, hi = acc[R-1].lo
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] = viaddmax_s16x2(bridge, gb[r], acc[r]);
            /* max-plus scan of the lane totals in band order (the band starts at lane s_cur * LPB mod G) */
            int32_t t = hi16(acc[R - 1]);
            int32_t carry = shfl(t, lane_left);   // same short cut as in dp(): usually no carry travels beyond one lane
            carry = bo == 0 ? kNeg32 : carry;
            if (ballot(cb * 16u + sub_lane * KB <= len && carry + KB * g > t)) {  // group-uniform; see dp()
#pragma unroll
                for (int dd = 1; dd < G; dd <<= 1) {
                    const int32_t o = shfl(t, (lanem - dd) & (G - 1));
                    t = viaddmax_s32(bo >= static_cast<uint32_t>(dd) ? o : kNeg32, dd * KB * g, t);
                }
                carry = shfl(t, lane_left);
                carry = bo == 0 ? kNeg32 : carry;
            }
            carry = carry < negsafe ? negsafe : carry;
            const uint32_t c2 = pack16(carry, carry);
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] = viaddmax_s16x2(c2, gc[r], acc[r]);
            RowB out;
#pragma unroll
            for (int r = 0; r < R; ++r) out.r[r] = acc[r];
            int16_t* myrow_s = ring + myslot * kBW;
            store_band_smem(myrow_s, lane, out);
            store_band_gmem(H + static_cast<uint64_t>(i) * kBW, lane, out);
            syncwarp();
            if (sink && sink_blk - s_cur < NB) {  // group-uniform
                const int32_t sc = myrow_s[sink_e];
                if (sc > best) {
                    best = sc;
                    bi = i;
                    nb = 1;
                } else if (sc == best) {
                    ++nb;
                }
            }
        }
        *best_row = bi;
        *best_score = best;
        *n_best = nb;
        syncwarp();
    }

    /* H[r][c] of the last DP, whichever layout it used (full rows of pitch lpa, or band rows) */
    template <bool BAND>
    RP_DEV int32_t hcell(uint32_t lpa, uint32_t r, uint32_t c) const {
        return hcell_at<BAND>(H, bs, P->gap, lpa, r, c);
    }

    /* ---------------------------------------------------------------- spoa's DFS order (graph.cpp:249-303)
     * Serial (lane 0).  With `sub`, runs on the subgraph exactly as spoa would on Graph::Subgraph():
     * nodes in ascending id, in-edges/aligned nodes filtered to members, original list orders kept. */
    RP_DEV void spoa_sort_hbm(bool sub) {
        for (uint32_t v = lane; v < N; v += G) marks[v] = 0;  // bits0-1 mark, bit2 ignored
        syncwarp();
        if (lane == 0) {
            const uint32_t cap = P->lim.stack_cap;
            uint32_t out = 0, sp = 0;
            for (uint32_t root = 0; root < N && status == kWinOk; ++root) {
                if (sub && !member[root]) continue;
                if ((marks[root] & 3) != 0) continue;
                stack[sp++] = static_cast<uint16_t>(root);
                while (sp > 0) {
                    uint32_t c = stack[sp - 1];
                    bool valid = true;
                    uint8_t mk = marks[c];
                    if ((mk & 3) != 2) {
                        uint32_t ni = in_cnt[c], na = al_cnt[c];
                        if (sp + ni + na > cap) {
                            fail(kWinStackLimit);
                            break;
                        }
                        for (uint32_t k = 0; k < ni; ++k) {
                            uint32_t t = in_tail[c * ki + k];
                            if (sub && !member[t]) continue;
                            if ((marks[t] & 3) != 2) {
                                stack[sp++] = static_cast<uint16_t>(t);
                                valid = false;
                            }
                        }
                        if (!(mk & 4)) {
                            for (uint32_t k = 0; k < na; ++k) {
                                uint32_t a = al[c * ka + k];
                                if (sub && !member[a]) continue;
                                if ((marks[a] & 3) != 2) {
                                    stack[sp++] = static_cast<uint16_t>(a);
                                    marks[a] |= 4;
                                    valid = false;
                                }
                            }
                        }
                        if (valid) {
                            marks[c] = static_cast<uint8_t>((marks[c] & 4) | 2);
                            if (!(marks[c] & 4)) {
                                srank[c] = static_cast<uint16_t>(out);
                                sorder[out++] = static_cast<uint16_t>(c);
                                for (uint32_t k = 0; k < na; ++k) {
                                    uint32_t a = al[c * ka + k];
                                    if (sub && !member[a]) continue;
                                    srank[a] = static_cast<uint16_t>(out);
                                    sorder[out++] = static_cast<uint16_t>(a);
                                }
                            }
                        } else {
                            marks[c] = static_cast<uint8_t>((marks[c] & 4) | 1);
                        }
                    }
                    if (valid) --sp;
                }
            }
        }
        status = shfl(status, 0);
        syncwarp();
    }

    /* Same DFS with the per-node state the walk touches on every step (marks, in-degree, aligned count) and
     * the stack staged in shared memory (idle outside the DP): one HBM round trip per examined node (its
     * in-edge tails and aligned list are fetched together) instead of five dependent ones. */
    RP_DEV void spoa_sort(bool sub) {
        const uint32_t npad = (N + 15) & ~15u;
        if (ki > 31 || ka != 8 || 2 * npad + 512 > smem_bytes || (P->debug_flags & 1) ||
            !spoa_sort_staged(sub, npad))
            spoa_sort_hbm(sub);
    }

    RP_DEV bool spoa_sort_staged(bool sub, uint32_t npad) {
        uint8_t* smk = smem;          // bits0-1 mark, bit2 ignored, bit3 member
        uint8_t* sme = smem + npad;   // in_cnt | al_cnt << 5
        /* the first two in-edge tails of every node too, when they fit: a node then costs an HBM round trip
         * only if it has more than two in-edges or aligned nodes */
        const bool have_t2 = 6 * npad + 1536 <= smem_bytes;
        uint32_t* st2 = reinterpret_cast<uint32_t*>(smem + 2 * npad);
        const uint32_t fixed = have_t2 ? 6 * npad : 2 * npad;
        uint16_t* sst = reinterpret_cast<uint16_t*>(smem + fixed);
        const uint32_t cap = (smem_bytes - fixed) / 2;
        for (uint32_t v = lane; v < N; v += G) {
            smk[v] = (!sub || member[v]) ? 8 : 0;
            sme[v] = static_cast<uint8_t>(in_cnt[v] | (al_cnt[v] << 5));
            if (have_t2) st2[v] = *reinterpret_cast<const uint32_t*>(in_tail + v * ki);
        }
        syncwarp();
        uint32_t ovf = 0;
        if (lane == 0) {
            uint32_t out = 0, sp = 0;
            for (uint32_t root = 0; root < N && !ovf; ++root) {
                if (smk[root] != 8) continue;  // not a member, or already marked
                sst[sp++] = static_cast<uint16_t>(root);
                while (sp > 0) {
                    const uint32_t c = sst[sp - 1];
                    bool valid = true;
                    const uint8_t mk = smk[c];
                    if ((mk & 3) != 2) {
                        const uint32_t ni = sme[c] & 31u, na = sme[c] >> 5;
                        uint64_t t4 = have_t2 ? st2[c] : 0;
                        if (!have_t2 || ni > 2) t4 = *reinterpret_cast<const uint64_t*>(in_tail + c * ki);
                        uint64_t a_lo = 0, a_hi = 0;
                        if (na) {
                            const U4 a8 = *reinterpret_cast<const U4*>(al + c * ka);
                            a_lo = a8.x | (static_cast<uint64_t>(a8.y) << 32);
                            a_hi = a8.z | (static_cast<uint64_t>(a8.w) << 32);
                        }
                        if (sp + ni + na > cap) {
                            ovf = 1;
                            break;
                        }
                        for (uint32_t k = 0; k < ni; ++k) {
                            const uint32_t t = k < 4 ? (static_cast<uint32_t>(t4 >> (16 * k)) & 0xffffu)
                                                     : in_tail[c * ki + k];
                            const uint8_t mt = smk[t];
                            if (!(mt & 8)) continue;
                            if ((mt & 3) != 2) {
                                sst[sp++] = static_cast<uint16_t>(t);
                                valid = false;
                            }
                        }
                        if (!(mk & 4)) {
                            for (uint32_t k = 0; k < na; ++k) {
                                const uint32_t a = static_cast<uint32_t>((k < 4 ? a_lo : a_hi) >> (16 * (k & 3))) & 0xffffu;
                                const uint8_t ma = smk[a];
                                if (!(ma & 8)) continue;
                                if ((ma & 3) != 2) {
                                    sst[sp++] = static_cast<uint16_t>(a);
                                    smk[a] = ma | 4;
                                    valid = false;
                                }
                            }
                        }
                        if (valid) {
                            const uint8_t now = smk[c];
                            smk[c] = static_cast<uint8_t>((now & 12) | 2);
                            if (!(now & 4)) {
                                srank[c] = static_cast<uint16_t>(out);
                                sorder[out++] = static_cast<uint16_t>(c);
                                for (uint32_t k = 0; k < na; ++k) {
                                    const uint32_t a = static_cast<uint32_t>((k < 4 ? a_lo : a_hi) >> (16 * (k & 3))) & 0xffffu;
                                    if (!(smk[a] & 8)) continue;
                                    srank[a] = static_cast<uint16_t>(out);
                                    sorder[out++] = static_cast<uint16_t>(a);
                                }
                            }
                        } else {
                            smk[c] = static_cast<uint8_t>((smk[c] & 12) | 1);
                        }
                    }
                    if (valid) --sp;
                }
            }
        }
        ovf = shfl(ovf, 0);
        syncwarp();
        return !ovf;
    }

    /* Among sink rows whose last-column score equals `best`, the one spoa visits first (sisd :353-355). */
    template <bool BAND>
    RP_DEV uint32_t resolve_sink_tie(uint32_t nrows, uint32_t len, uint32_t lpa, int32_t best, bool sub) {
        spoa_sort(sub);
        const uint16_t* ord = sub ? dp_order : order;
        uint32_t bestkey = 0xffffffffu;
        for (uint32_t r = 1 + lane; r <= nrows; r += G) {
            uint64_t rc = rec[r].a;
            if (!((rc >> 15) & 1)) continue;
            if (hcell<BAND>(lpa, r, len) != best) continue;
            uint32_t key = (static_cast<uint32_t>(srank[ord[r]]) << 16) | r;
            if (key < bestkey) bestkey = key;
        }
        for (int d = G / 2; d > 0; d >>= 1) {
            uint32_t o = shfl_down(bestkey, d);
            if (o < bestkey) bestkey = o;
        }
        bestkey = shfl(bestkey, 0);
        return bestkey & 0xffffu;
    }

    /* ---------------------------------------------------------------- traceback (sisd :366-459)
     * Priority: diagonal over predecessors in in-edge order, then vertical in the same order, then
     * horizontal.  Lanes test predecessors in parallel; the lowest lane that matches wins.
     * The walk is a chain of dependent reads of H, so it runs out of a shared-memory TILE: the group
     * copies tile_rows ranks x 32 columns of H (plus those rows' program records) from HBM with one
     * coalesced burst, walks until the path leaves the tile, and re-anchors.  Predecessors below the tile
     * (rare long edges) are read from HBM directly.
     * Output: aln[j] = node aligned to read position j, or kNone (new node).
     *
     * BAND: the matrix is the banded one (dp_band).  The result is accepted — the function returns true — only if
     * every cell of the path (i) keeps `band_margin` columns away from every band edge that really cuts the matrix
     * (an edge at column 0 or at the last column cuts nothing; the cells of the predecessor rows the walk compares with
     * must keep the same distance inside THEIR bands), (ii) holds a value a real alignment can have (>= worst: anything
     * derived from an excluded cell is below that, see poa_window), and (iii) the path is not a long stretch of
     * mismatches and gaps (the true path then probably lies outside the band: kBandJunkLimit).  Otherwise false is
     * returned and the caller repeats the alignment with the full matrix.  Why an accepted result equals the
     * full-matrix result: banded values never exceed the full ones and are equal wherever an optimal path lies
     * inside the band, so every equality test of the walk has the same outcome as in the full matrix as long as
     * the optimal paths stay inside; the margin test is the (heuristic) evidence that they do. */
    /* > G predecessors (escalated windows only): every diagonal candidate of every batch outranks any
     * vertical one.  Reads straight from the HBM copy; kept out of line so the common loop stays small. */
    /* static + explicit arguments: a non-inlined MEMBER would take `this`, forcing the whole PoaWarp into local memory */
    template <bool BAND>
    static RP_DEV int32_t hcell_at(const int16_t* H, const uint8_t* bs, int32_t g, uint32_t lpa, uint32_t r, uint32_t c) {
        if (!BAND) return H[static_cast<uint64_t>(r) * lpa + perm(c)];
        if (r == 0) return static_cast<int32_t>(c) * g;
        const uint32_t cbk = c >> 4;
        const uint32_t sr = bs[r];   // independent of the cell's address: the two loads overlap
        const int32_t v = H[static_cast<uint64_t>(r) * kBW + ((cbk & (NB - 1)) << 4) + (perm_band(c) & 15u)];
        return cbk - sr >= NB ? kBandFloor : v;
    }

    template <bool BAND>
    /* returns (move << 16) | predecessor rank, 0 when no predecessor matches — a packed value, not an output pointer: the
     * caller's variable would then live in local memory, on the dependency chain of every step of the walk */
    static RP_DEV_NOINLINE uint32_t traceback_step_wide(const int16_t* H, const uint8_t* bs, const Rec* rec,
                                                        const uint16_t* pred_ovf, uint32_t ki, int lane, int32_t g,
                                                        uint32_t i, uint32_t j, uint32_t npe, int32_t hij, int32_t mc,
                                                        uint32_t lpa) {
        for (int pass = 1; pass <= 2; ++pass) {
            if (pass == 1 && j == 0) continue;
            for (uint32_t k0 = 0; k0 < npe; k0 += G) {
                const uint32_t k = k0 + lane;
                uint32_t p = 0;
                bool ok = false;
                if (k < npe) {
                    p = k < 7 ? rec_pred(rec[i], k) : pred_ovf[i * ki + k];
                    ok = pass == 1 ? (hij == hcell_at<BAND>(H, bs, g, lpa, p, j - 1) + mc)
                                   : (hij == hcell_at<BAND>(H, bs, g, lpa, p, j) + g);
                }
                const uint32_t msk = gballot<G>(ok);
                if (msk) return (static_cast<uint32_t>(pass) << 16) | (gshfl<G>(p, ffs_(msk) - 1) & 0xffffu);
            }
        }
        return 0;
    }

    /* banded walk, more predecessors than lanes: true when some candidate cell is closer than the margin to an edge
     * that cuts its own row's band (see traceback) */
    static RP_DEV_NOINLINE bool wide_candidates_unsure(const uint8_t* bs, const Rec* rec, const uint16_t* pred_ovf,
                                                       uint32_t ki, int lane, uint32_t i, uint32_t j, uint32_t npe,
                                                       uint32_t nblk, uint32_t margin) {
        bool unsure = false;
        for (uint32_t k0 = 0; k0 < npe; k0 += G) {
            const uint32_t k = k0 + lane;
            if (k < npe) {
                const uint32_t p = k < 7 ? rec_pred(rec[i], k) : pred_ovf[i * ki + k];
                if (p != 0) {
                    const uint32_t sp = bs[p];
                    const int32_t dlp = static_cast<int32_t>(j) - 1 - static_cast<int32_t>(16u * sp);
                    const int32_t drp = static_cast<int32_t>(16u * (sp + NB)) - 1 - static_cast<int32_t>(j);
                    unsure |= (sp > 0 && dlp < static_cast<int32_t>(margin)) ||
                              (sp + NB < nblk && drp < static_cast<int32_t>(margin));
                }
            }
        }
        return gballot<G>(unsure) != 0;
    }

    static constexpr uint32_t kTileCols = 32;
    static constexpr uint32_t kBandJunkLimit = 48;   // see traceback<true>, check (iii)
    static constexpr uint32_t kTileRowBytes = kTileCols * 2 + 16 + 1;   // H cells | record | band start

    template <bool BAND>
    RP_DEV bool traceback(uint32_t best_row, uint32_t len, uint32_t lpa, const uint8_t* seq, bool sub, int32_t worst) {
        const int32_t g = P->gap, m = P->match, x = P->mismatch;
        const uint16_t* ord = sub ? dp_order : order;
        uint32_t kTileRows = (smem_bytes - 16 - len) / kTileRowBytes;
        if (kTileRows > 96) kTileRows = 96;
        if (P->tile_rows && P->tile_rows < kTileRows) kTileRows = P->tile_rows;
        kTileRows &= ~1u;
        int16_t* tile = reinterpret_cast<int16_t*>(smem);                                        // [kTileRows][32]
        Rec* trec = reinterpret_cast<Rec*>(smem + kTileRows * kTileCols * 2);                      // [kTileRows]
        uint8_t* tbs = smem + kTileRows * (kTileCols * 2 + 16);                                    // [kTileRows]
        uint8_t* tseq = tbs + ((kTileRows + 15) & ~15u);
        /* the walk compares the row's character with seq[j-1] every step: kept as window-alphabet code indices, the
         * form the row records hold (a character is in the alphabet exactly once, so codes compare like characters) */
        for (uint32_t c = lane; c < len; c += G) tseq[c] = static_cast<uint8_t>(code_index(seq[c]));
        /* read back relative to the tile base, which the walk keeps in a register anyway */
        const uint8_t* tile_b = reinterpret_cast<const uint8_t*>(tile);
        uint32_t tseq_at = static_cast<uint32_t>(tseq - tile_b);
        RP_KEEP_IN_REGISTER(tseq_at);
        const uint32_t nblk = (len + 16) >> 4;
        const uint32_t margin = P->band_margin;
        const U4 f4 = U4{pack16(kBandFloor, kBandFloor), pack16(kBandFloor, kBandFloor), pack16(kBandFloor, kBandFloor),
                         pack16(kBandFloor, kBandFloor)};
        uint32_t i = best_row, j = len;
        uint32_t t_top = 0, t_rows = 0, t_col0 = 0;  // tile covers ranks (t_top - t_rows, t_top], cols [t_col0, t_col0+32)
        bool have_tile = false, bad = false;
        uint32_t quality = 0;
        /* aln[] is written one position per diagonal / horizontal step, positions falling by one: lane (c mod G) keeps
         * the value of position c and the group stores G finished positions with one coalesced write (put_aln) instead
         * of a lane-0 store — and its address arithmetic — inside every step */
        /* element index (inside a stored row) of columns j and j-1, carried along: one perm() per step to the left */
        uint32_t pj = BAND ? perm_band(j) : perm(j);
        uint32_t pjm = j > 0 ? (BAND ? perm_band(j - 1) : perm(j - 1)) : 0u;
        auto step_left = [&]() {
            --j;
            pj = pjm;
            pjm = j > 0 ? (BAND ? perm_band(j - 1) : perm(j - 1)) : 0u;
        };
        uint32_t pend = kNone;
        auto put_aln = [&](uint32_t c, uint32_t v) {   // c = j - 1, group-uniform
            if ((c & (G - 1)) == static_cast<uint32_t>(lane)) pend = v;
            if ((c & (G - 1)) == 0) {   // group-uniform: positions c .. c+G-1 are complete
                if (c + lane < len) aln[c + lane] = static_cast<uint16_t>(pend);
            }
        };
        while (i != 0) {
            bool need = !have_tile || i + t_rows <= t_top || (j > 0 && j - 1 < t_col0);
            /* when a group that runs in lock step with this one refills, refill too: the groups of a warp then
             * stall for one refill instead of one each (a fresh tile is never wrong) */
            if (G < 32 && any_converged_peer<G>(need)) need = true;
            if (need) {
                syncwarp();
                t_top = i;
                t_rows = i + 1 < kTileRows ? i + 1 : kTileRows;  // down to rank 0 at most
                const uint32_t cbj = j >> 4;
                const uint32_t cba = cbj ? cbj - 1 : 0;
                t_col0 = cba << 4;
                /* the rows' records first (at most three per lane at 32 lanes): their loads are in flight while the
                 * granule loop below waits for its own */
                Rec tr[3];
                if (G == 32) {
#pragma unroll
                    for (uint32_t k = 0; k < 3; ++k) {
                        const uint32_t q = static_cast<uint32_t>(lane) + 32u * k;
                        if (q < t_rows) tr[k] = rec[t_top - q];
                    }
                }
                /* four lanes per tile row, one 16-byte granule each: consecutive lanes write consecutive 16-byte
                 * granules of the tile (no shared-memory bank conflict) and read one 64-byte piece of an H row.
                 * Full matrix: asynchronous copies (cp.async), all of a lane's granules — up to 12 — in flight at once.
                 * Band: through registers, which substitute the out-of-band granules. */
                for (uint32_t e = lane; e < 4 * t_rows; e += G) {
                    const uint32_t q = e >> 2, gq = e & 3u;
                    const uint32_t rk = t_top - q;
                    if (!BAND) {
                        copy16_async(reinterpret_cast<U4*>(tile) + e,
                                     reinterpret_cast<const U4*>(H + static_cast<uint64_t>(rk) * lpa + t_col0) + gq);
                        continue;
                    }
                    U4 v;
                    const uint32_t sr = bs[rk];
                    const uint32_t blk = cba + (gq >> 1);
                    if (rk == 0) {  // virtual root row: H[0][c] = c * g, in the row's register order
                        int16_t t8[8];
#pragma unroll
                        for (uint32_t k = 0; k < 8; ++k) {
                            const uint32_t el = (gq & 1u) * 8 + k;                  // element inside the block
                            const uint32_t col = blk * 16 + unperm_band(el);
                            t8[k] = static_cast<int16_t>(static_cast<int32_t>(col) * g);
                        }
                        v = U4{pack16(t8[0], t8[1]), pack16(t8[2], t8[3]), pack16(t8[4], t8[5]), pack16(t8[6], t8[7])};
                    } else {
                        /* the granule's address does not depend on the row's band start: both loads go out together */
                        v = reinterpret_cast<const U4*>(H + static_cast<uint64_t>(rk) * kBW + ((blk & (NB - 1)) << 4))[gq & 1u];
                        if (blk - sr >= NB) v = f4;
                    }
                    if (gq == 0) tbs[q] = static_cast<uint8_t>(sr);
                    reinterpret_cast<U4*>(tile)[e] = v;
                }
                if (G == 32) {
#pragma unroll
                    for (uint32_t k = 0; k < 3; ++k) {
                        const uint32_t q = static_cast<uint32_t>(lane) + 32u * k;
                        if (q < t_rows) trec[q] = tr[k];
                    }
                } else {
                    for (uint32_t q = lane; q < t_rows; q += G) trec[q] = rec[t_top - q];
                }
                if (!BAND) copy_async_wait();
                have_tile = true;
                syncwarp();
            }
            const uint32_t q = t_top - i;
            const Rec rc = trec[q];
            const uint32_t lo = static_cast<uint32_t>(rc.a);
            const uint32_t cidx = lo & 0xff, np = (lo >> 8) & 0x7f;
            const uint32_t npe = np ? np : 1;
            const uint32_t ej = pj - t_col0;                // element of column j inside a tile row
            const uint32_t ejm = j > 0 ? pjm - t_col0 : 0;  // column j-1
            const int32_t hij = tile[q * kTileCols + ej];
            if (BAND) {
                const uint32_t si = tbs[q];
                const uint32_t dl = j - 16u * si, dr = 16u * (si + NB) - 1u - j;
                if ((si > 0 && dl < margin) || (si + NB < nblk && dr < margin) || hij < worst) {  // group-uniform
                    bad = true;
                    break;
                }
            }
            int32_t mc = 0;
            if (j > 0) mc = cidx == tile_b[tseq_at + j - 1] ? m : x;
            uint32_t found_p = 0;
            int move = 0;  // 1 diag, 2 vert, 3 horiz
            if (np <= 7) {  // group-uniform: every predecessor is in the row's record
                /* 7 of 10 steps of the walk are on rows with several predecessors (the consensus path runs through the
                 * nodes many reads agree on), and on nearly all of them the FIRST in-edge — the oldest, heaviest one — is the
                 * diagonal match.  So the lanes do not spread the candidates over themselves and vote: every lane walks
                 * them in spoa's order (sisd :392-442: any diagonal beats any vertical, lowest in-edge first) and stops at
                 * the first diagonal match — no vote, no lane election, no indexed record field, and the common step costs
                 * what a single-predecessor row costs.  The banded walk looks at every candidate (its acceptance rule
                 * covers all of them, see the general case below). */
                uint64_t pq = rc.a >> 16;     // pred0..2, then rc.b = pred3..6
                uint32_t pd = 0, pv = 0;
                bool okd = false, okv = false, unsure = false;
                for (uint32_t k = 0; k < npe; ++k) {
                    const uint32_t p = np ? static_cast<uint32_t>(pq) & 0xffffu : 0u;
                    pq = k == 2 ? rc.b : pq >> 16;
                    int32_t a, b;
                    uint32_t sp = 0;
                    if (p + t_rows > t_top) {  // predecessor row is inside the tile
                        const int16_t* pr = tile + (t_top - p) * kTileCols;
                        a = pr[ejm];
                        b = pr[ej];
                        if (BAND) sp = tbs[t_top - p];
                    } else if (!BAND) {        // a rare long edge: straight from the HBM copy, with the element
                        const int16_t* hr = H + static_cast<uint64_t>(p) * lpa;   // indices the walk carries anyway
                        a = hr[pjm];
                        b = hr[pj];
                    } else {
                        a = hcell<BAND>(lpa, p, j > 0 ? j - 1 : 0);
                        b = hcell<BAND>(lpa, p, j);
                        sp = bs[p];
                    }
                    if (BAND && p != 0) {  // the candidate cells must be trustworthy too (see the general case)
                        const int32_t dlp = static_cast<int32_t>(j) - 1 - static_cast<int32_t>(16u * sp);
                        const int32_t drp = static_cast<int32_t>(16u * (sp + NB)) - 1 - static_cast<int32_t>(j);
                        unsure |= (sp > 0 && dlp < static_cast<int32_t>(margin)) ||
                                  (sp + NB < nblk && drp < static_cast<int32_t>(margin));
                    }
                    if (!okv && hij == b + g) {
                        okv = true;
                        pv = p;
                    }
                    if (!okd && j > 0 && hij == a + mc) {
                        okd = true;
                        pd = p;
                        if (!BAND) break;
                    }
                }
                if (BAND && unsure) {
                    bad = true;
                    break;
                }
                if (okd) {
                    move = 1;
                    found_p = pd;
                } else if (okv) {
                    move = 2;
                    found_p = pv;
                }
            } else if (npe <= G) {
                /* one predecessor per lane; all diagonal candidates outrank any vertical one (sisd :392-442) */
                uint32_t p = 0;
                bool okd = false, okv = false, unsure = false;
                if (static_cast<uint32_t>(lane) < npe) {
                    if (np) p = static_cast<uint32_t>(lane) < 7 ? rec_pred(rc, lane) : pred_ovf[i * ki + lane];
                    int32_t a = 0, b;
                    uint32_t sp = 0;
                    if (p + t_rows > t_top) {  // predecessor row is inside the tile
                        const int16_t* pr = tile + (t_top - p) * kTileCols;
                        a = pr[ejm];
                        b = pr[ej];
                        if (BAND) sp = tbs[t_top - p];
                    } else {
                        a = hcell<BAND>(lpa, p, j > 0 ? j - 1 : 0);
                        b = hcell<BAND>(lpa, p, j);
                        if (BAND) sp = bs[p];
                    }
                    okd = j > 0 && hij == a + mc;
                    okv = hij == b + g;
                    if (BAND && p != 0) {
                        /* the candidate cells (p, j-1), (p, j) must be trustworthy too: a predecessor whose own band is
                         * cut closer than the margin to these columns (or does not hold them at all) could hide a tie
                         * the full matrix would have resolved the other way */
                        const int32_t dlp = static_cast<int32_t>(j) - 1 - static_cast<int32_t>(16u * sp);
                        const int32_t drp = static_cast<int32_t>(16u * (sp + NB)) - 1 - static_cast<int32_t>(j);
                        unsure = (sp > 0 && dlp < static_cast<int32_t>(margin)) ||
                                 (sp + NB < nblk && drp < static_cast<int32_t>(margin));
                    }
                }
                if (BAND && ballot(unsure)) {  // group-uniform
                    bad = true;
                    break;
                }
                const uint32_t md = ballot(okd);
                const uint32_t mv = ballot(okv);
                const uint32_t sel = md ? md : mv;
                if (sel) {
                    const uint32_t kw = static_cast<uint32_t>(ffs_(sel) - 1);   // winning lane = its predecessor's index
                    found_p = kw < 7 ? (np ? rec_pred(rc, kw) : 0u) : shfl(p, static_cast<int>(kw));
                    move = md ? 1 : 2;
                }
            } else {
                if (BAND && wide_candidates_unsure(bs, rec, pred_ovf, ki, lane, i, j, npe, nblk, margin)) {
                    bad = true;
                    break;
                }
                const uint32_t mp = traceback_step_wide<BAND>(H, bs, rec, pred_ovf, ki, lane, g, i, j, npe, hij, mc, lpa);
                move = static_cast<int>(mp >> 16);
                found_p = mp & 0xffffu;
            }
            if (!move) move = 3;
            if (BAND) {
                /* (iii) the path must look like a real alignment: a long stretch that is mostly mismatches and gaps
                 * means the read's true path probably runs somewhere else — outside the band, where this matrix cannot
                 * see it.  Leaky counter: +2 per mismatch / gap step, -1 per match; a good alignment keeps it near
                 * zero (12 % errors: -0.6 per step), aligned junk drives it up by about +0.5 per step. */
                const bool is_match = move == 1 && mc == m && m != x;
                quality = is_match ? (quality ? quality - 1 : 0u) : quality + 2u;
                if (quality > kBandJunkLimit) {
                    bad = true;
                    break;
                }
            }
            if (move == 1) {
                put_aln(j - 1, i);   // rank for now, node below
                i = found_p;
                step_left();
            } else if (move == 2) {
                i = found_p;
            } else {
                if (j == 0) {  // unreachable for a consistent matrix (column 0 always has a vertical move)
                    if (BAND)
                        bad = true;
                    else
                        fail(kWinInternal);
                    break;
                }
                put_aln(j - 1, kNone);
                step_left();
            }
        }
        /* positions j .. of the block the walk stopped in (nothing pending when j is a multiple of G) */
        if ((j & (G - 1)) != 0) {
            const uint32_t c = (j & ~static_cast<uint32_t>(G - 1)) + lane;
            if (c >= j && c < len) aln[c] = static_cast<uint16_t>(pend);
        }
        syncwarp();
        if (bad) return false;
        /* row 0: remaining columns are horizontal moves (insertions at the start of the read); matched positions
         * hold the DP rank of their row: turn it into the node */
        for (uint32_t c = lane; c < len; c += G) {
            if (c < j) {
                aln[c] = kNone;
            } else {
                const uint32_t r = aln[c];
                if (r != kNone) aln[c] = ord[r];
            }
        }
        syncwarp();
        return true;
    }

    /* add_alignment, Phase D (below): the order update's counters and the remap */
    template <bool kSmem>
    RP_DEV void merge_order(uint32_t n_old, uint32_t n_new) {
        /* (the slot's base is not kept: one more member of this struct costs per-window spills) */
        uint16_t* delta = kSmem ? reinterpret_cast<uint16_t*>(smem)
                                : reinterpret_cast<uint16_t*>(bs + (P->lay.delta - P->lay.bs));
        for (uint32_t q = lane; q < n_old + 2; q += G) delta[q] = 0;
        syncwarp();
        for (uint32_t k = lane; k < n_new; k += G) {
            uint32_t j = newlist[k] >> 16;
            uint32_t key = aln[j];  // aligned new node: end of its cluster block; insertion: K_{j-1}
            uint32_t id = n_old + k;
            uint32_t nr = key + 1 + k;
            order_nxt[nr] = static_cast<uint16_t>(id);
            rank_of[id] = static_cast<uint16_t>(nr);
#if defined(RP_HOST_SIM)
            delta[key + 1] = static_cast<uint16_t>(delta[key + 1] + 1);
#else
            atomicAdd(reinterpret_cast<unsigned int*>(delta + ((key + 1) & ~1u)), (key + 1) & 1u ? 0x10000u : 1u);
#endif
        }
        syncwarp();
        /* inclusive prefix of the counters, then a remap pass whose HBM loads are batched */
        uint32_t carry = 0;
        for (uint32_t q0 = 1; q0 <= n_old; q0 += G) {
            uint32_t q = q0 + lane;
            uint32_t d = q <= n_old ? delta[q] : 0;
            uint32_t inc = warp_incl_sum(d) + carry;
            if (q <= n_old) delta[q] = static_cast<uint16_t>(inc);
            carry = shfl(inc, G - 1);
        }
        syncwarp();
        constexpr int kV = 8;
        for (uint32_t q0 = 1; q0 <= n_old; q0 += G * kV) {
            uint32_t v[kV];
#pragma unroll
            for (int u = 0; u < kV; ++u) {
                uint32_t q = q0 + u * G + lane;
                v[u] = q <= n_old ? order[q] : 0;
            }
#pragma unroll
            for (int u = 0; u < kV; ++u) {
                uint32_t q = q0 + u * G + lane;
                if (q <= n_old) {
                    uint32_t nr = q + delta[q];
                    order_nxt[nr] = static_cast<uint16_t>(v[u]);
                    rank_of[v[u]] = static_cast<uint16_t>(nr);
                }
            }
        }
    }

    /* ---------------------------------------------------------------- graph merge (graph.cpp:155-247) +
     * incremental order update.  aln[j] = aligned node or kNone for every read position j. */
    RP_DEV void add_alignment(const uint8_t* seq, const uint8_t* w, uint32_t len, uint32_t b0) {
        const uint32_t n_old = N;
        /* All phases handle kU positions per lane at a time with the loads of one dependency level issued
         * together (the graph is in HBM: every level costs a full memory latency). */
        constexpr int kU = 4;
        /* Phase A: target node per position (existing node, aligned sibling with the same character, or new) */
        uint32_t n_new = 0;
        for (uint32_t j0 = 0; j0 < len; j0 += G * kU) {
            uint32_t a[kU], c[kU], ca[kU], na[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                uint32_t j = j0 + u * G + lane;
                a[u] = j < len ? aln[j] : kNone;
                c[u] = j < len ? seq[j] : 0;
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                ca[u] = a[u] != kNone ? code[a[u]] : 0;
                na[u] = a[u] != kNone ? al_cnt[a[u]] : 0;
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                uint32_t j = j0 + u * G + lane;
                bool is_new = false;
                uint32_t tgt = kNone, anchor = kNone;
                if (j < len) {
                    if (a[u] == kNone) {
                        is_new = true;
                    } else if (ca[u] == c[u]) {
                        tgt = a[u];
                    } else {
                        for (uint32_t k = 0; k < na[u]; ++k) {
                            uint32_t sb = al[a[u] * ka + k];
                            if (code[sb] == c[u]) {
                                tgt = sb;
                                break;
                            }
                        }
                        if (tgt == kNone) {
                            is_new = true;
                            anchor = a[u];
                        }
                    }
                }
                uint32_t tot;
                uint32_t pos = warp_rank(is_new, &tot);
                if (is_new) {
                    uint32_t id = n_old + n_new + pos;
                    tgt = id;
                    if (id < nmax) {
                        code[id] = static_cast<uint8_t>(c[u]);
                        flags[id] = 0;
                        in_cnt[id] = 0;
                        cov[id] = 0;
                        al_cnt[id] = 0;
                    }
                    newlist[n_new + pos] = (j << 16) | anchor;  // anchor kNone => unaligned insertion
                }
                if (j < len) cur[j] = static_cast<uint16_t>(tgt);
                n_new += tot;
            }
        }
        if (n_old + n_new > nmax) {
            fail(kWinNodeLimit);
            return;
        }
        syncwarp();
        /* Phase B: aligned-cluster membership of new nodes (graph.cpp:221-229) */
        bool lim_a = false;
        for (uint32_t k0 = 0; k0 < n_new; k0 += G) {
            uint32_t k = k0 + lane;
            if (k < n_new) {
                uint32_t e = newlist[k];
                uint32_t anchor = e & 0xffffu;
                uint32_t id = n_old + k;
                if (anchor != kNone) {
                    uint32_t na = al_cnt[anchor];
                    if (na + 1 > ka) {
                        lim_a = true;
                    } else {
                        for (uint32_t q = 0; q < na; ++q) {
                            uint32_t sb = al[anchor * ka + q];
                            al[id * ka + q] = static_cast<uint16_t>(sb);
                            uint32_t ns = al_cnt[sb];
                            al[sb * ka + ns] = static_cast<uint16_t>(id);
                            al_cnt[sb] = static_cast<uint8_t>(ns + 1);
                        }
                        al[id * ka + na] = static_cast<uint16_t>(anchor);
                        al_cnt[id] = static_cast<uint8_t>(na + 1);
                        al[anchor * ka + na] = static_cast<uint16_t>(id);
                        al_cnt[anchor] = static_cast<uint8_t>(na + 1);
                    }
                }
            }
        }
        if (ballot(lim_a)) {
            fail(kWinAlignedLimit);
            return;
        }
        syncwarp();
        /* order keys K_j (non-decreasing along the read): for an old target, or the anchor of an aligned new
         * node, the last rank of its aligned-cluster block; an unaligned insertion inherits K_{j-1} */
        int32_t run = 0;  // K_{-1} = 0: right after the root
        int32_t runb = static_cast<int32_t>(b0);  // backbone coordinate an insertion at the very start inherits
        for (uint32_t j0 = 0; j0 < len; j0 += G * kU) {
            uint32_t bn[kU], rk0[kU], nal[kU], cj[kU], bpv[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                uint32_t j = j0 + u * G + lane;
                bn[u] = j < len ? cur[j] : kNone;
                cj[u] = bn[u];
            }
#pragma unroll
            for (int u = 0; u < kU; ++u)
                if (bn[u] != kNone && bn[u] >= n_old) bn[u] = newlist[bn[u] - n_old] & 0xffffu;  // anchor or kNone
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                rk0[u] = bn[u] != kNone ? rank_of[bn[u]] : 0;
                nal[u] = bn[u] != kNone ? al_cnt[bn[u]] : 0;
                bpv[u] = bn[u] != kNone ? bpos[bn[u]] : 0;
            }
            /* backbone coordinate of every new node (band centre line only, never affects a result): an aligned
             * new node sits where its anchor sits, an insertion where the path was before it */
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                int32_t incb = warp_incl_max(static_cast<int32_t>(bpv[u]));
                if (incb < runb) incb = runb;
                if (cj[u] != kNone && cj[u] >= n_old)
                    bpos[cj[u]] = static_cast<uint16_t>(bn[u] != kNone ? bpv[u] : static_cast<uint32_t>(incb));
                runb = shfl(incb, G - 1);
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                uint32_t j = j0 + u * G + lane;
                uint32_t rmax = rk0[u];
                for (uint32_t q = 0; q < nal[u]; ++q) {
                    uint32_t sb = al[bn[u] * ka + q];
                    if (sb < n_old) {
                        uint32_t rs = rank_of[sb];
                        if (rs > rmax) rmax = rs;
                    }
                }
                int32_t inc = warp_incl_max(static_cast<int32_t>(rmax));
                if (inc < run) inc = run;
                if (j < len) aln[j] = static_cast<uint16_t>(inc);  // aln now holds K_j
                run = shfl(inc, G - 1);
            }
        }
        syncwarp();
        /* Phase C: edges (graph.cpp:81-91,236-243) + per-node sequence counters (Node::Coverage, :32-47) */
        bool lim_e = false;
        for (uint32_t j0 = 0; j0 < len; j0 += G * kU) {
            uint32_t c[kU], pv[kU], ni[kU], cv[kU];
            int32_t wt[kU];
            uint64_t t4[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                uint32_t j = j0 + u * G + lane;
                c[u] = j < len ? cur[j] : kNone;
                pv[u] = (j < len && j > 0) ? cur[j - 1] : kNone;
                wt[u] = (j < len && j > 0) ? static_cast<int32_t>(w[j - 1]) + static_cast<int32_t>(w[j]) : 0;
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                ni[u] = c[u] != kNone ? in_cnt[c[u]] : 0;
                cv[u] = c[u] != kNone ? cov[c[u]] : 0;
                t4[u] = c[u] != kNone ? *reinterpret_cast<const uint64_t*>(in_tail + c[u] * ki) : 0;
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                if (c[u] == kNone) continue;
                if (len >= 2) cov[c[u]] = static_cast<uint16_t>(cv[u] + 1);
                if (pv[u] == kNone) continue;
                uint32_t q = 0;
                for (; q < ni[u]; ++q) {
                    uint32_t t = q < 4 ? (static_cast<uint32_t>(t4[u] >> (16 * q)) & 0xffffu) : in_tail[c[u] * ki + q];
                    if (t == pv[u]) break;
                }
                if (q < ni[u]) {
                    in_w[c[u] * ki + q] += wt[u];
                } else if (ni[u] < ki && ni[u] < 127) {
                    in_tail[c[u] * ki + ni[u]] = static_cast<uint16_t>(pv[u]);
                    in_w[c[u] * ki + ni[u]] = wt[u];
                    in_cnt[c[u]] = static_cast<uint8_t>(ni[u] + 1);
                    flags[pv[u]] |= 1;  // every pv is a distinct node, so lanes never touch the same byte
                } else {
                    lim_e = true;
                }
            }
        }
        if (ballot(lim_e)) {
            fail(kWinEdgeLimit);
            return;
        }
        syncwarp();
        /* Phase D: merge new nodes into the processing order.  New node k (read order) with key K goes to
         * rank K + 1 + k; an old node at rank q moves to q + #{new nodes with key < q}. */
        if (n_new > 0) {
            /* its n_old + 2 counters live in shared memory (the ring is idle now) when they fit, else in the slot's HBM
             * copy, so that nmax is the only node limit whatever the group's share of shared memory; one instantiation
             * per memory space, so that every access compiles to a shared- or a global-memory instruction */
            if ((n_old + 4) * 2 <= smem_bytes)
                merge_order<true>(n_old, n_new);
            else
                merge_order<false>(n_old, n_new);
            if (lane == 0) order_nxt[0] = kNone;
            uint16_t* t = order;
            order = order_nxt;
            order_nxt = t;
            N = n_old + n_new;
        }
        ++n_added;
        syncwarp();
    }

    /* ---------------------------------------------------------------- consensus (graph.cpp:433-516, 377-398)
     * Heaviest bundle.  The pass over the nodes in spoa's rank order is inherently serial (lane 0), but what it
     * reads is not: the warp stages 32 nodes at a time (id, in-degree, first four in-edge tails and weights)
     * into shared memory with coalesced gathers, and scores / best predecessors live in shared memory too
     * when the graph is small enough (int32 scores are exact while the sum of all edge weights < 2^31). */
    struct CStage {
        uint32_t w[4];
        uint16_t t[4];
        uint16_t it;
        uint16_t ni;
        uint32_t pad;
    };

    template <typename ScoreT>
    RP_DEV void better_t(ScoreT* sc, uint16_t* cp, uint32_t it, uint32_t t, int64_t wgt) {
        int64_t si = sc[it];
        if (si < wgt || (si == wgt && cp[it] != kNone && sc[cp[it]] <= sc[t])) {
            sc[it] = static_cast<ScoreT>(wgt);
            cp[it] = static_cast<uint16_t>(t);
        }
    }

    /* one pass over ranks [r_begin, N): graph.cpp:442-456 (skip_dead = false) or :493-513 (true) */
    template <typename ScoreT>
    RP_DEV uint32_t bundle_pass(ScoreT* sc, uint16_t* cp, CStage* stg, uint32_t r_begin, bool skip_dead) {
        uint32_t mx = kNone;
        for (uint32_t r0 = r_begin; r0 < N; r0 += G) {
            const uint32_t r = r0 + lane;
            if (r < N) {
                const uint32_t it = sorder[r];
                CStage e;
                e.it = static_cast<uint16_t>(it);
                e.ni = in_cnt[it];
                const uint64_t t4 = *reinterpret_cast<const uint64_t*>(in_tail + it * ki);
                const U4 w4 = *reinterpret_cast<const U4*>(in_w + it * ki);
                e.t[0] = static_cast<uint16_t>(t4);
                e.t[1] = static_cast<uint16_t>(t4 >> 16);
                e.t[2] = static_cast<uint16_t>(t4 >> 32);
                e.t[3] = static_cast<uint16_t>(t4 >> 48);
                e.w[0] = w4.x; e.w[1] = w4.y; e.w[2] = w4.z; e.w[3] = w4.w;
                e.pad = 0;
                stg[lane] = e;
            }
            syncwarp();
            if (lane == 0) {
                const uint32_t cnt = N - r0 < G ? N - r0 : G;
                for (uint32_t q = 0; q < cnt; ++q) {
                    const CStage& e = stg[q];
                    const uint32_t it = e.it;
                    if (skip_dead) {
                        sc[it] = -1;
                        cp[it] = kNone;
                    }
                    for (uint32_t k = 0; k < e.ni; ++k) {
                        const uint32_t t = k < 4 ? e.t[k] : in_tail[it * ki + k];
                        if (skip_dead && sc[t] == -1) continue;
                        const int64_t wgt = k < 4 ? static_cast<int32_t>(e.w[k]) : in_w[it * ki + k];
                        better_t(sc, cp, it, t, wgt);
                    }
                    if (cp[it] != kNone) sc[it] = static_cast<ScoreT>(sc[it] + sc[cp[it]]);
                    if (mx == kNone || sc[mx] < sc[it]) mx = it;
                }
            }
            syncwarp();
        }
        return shfl(mx, 0);
    }

    template <typename ScoreT>
    RP_DEV uint32_t bundle(ScoreT* sc, uint16_t* cp, CStage* stg) {
        for (uint32_t v = lane; v < N; v += G) {
            sc[v] = -1;
            cp[v] = kNone;
        }
        syncwarp();
        uint32_t mx = bundle_pass(sc, cp, stg, 0, false);
        /* branch completion (graph.cpp:478-516) while the best node still has out-edges */
        while (flags[mx] & 1) {
            /* heads of mx's out-edges = nodes with an in-edge from mx; their other tails are invalidated */
            for (uint32_t v = lane; v < N; v += G) {
                uint32_t ni = in_cnt[v];
                bool hit = false;
                for (uint32_t k = 0; k < ni; ++k) hit |= (in_tail[v * ki + k] == mx);
                if (hit)
                    for (uint32_t k = 0; k < ni; ++k) {
                        uint32_t t = in_tail[v * ki + k];
                        if (t != mx) sc[t] = -1;
                    }
            }
            syncwarp();
            uint32_t nm = bundle_pass(sc, cp, stg, static_cast<uint32_t>(srank[mx]) + 1, true);
            if (nm == kNone) break;  // cannot happen: a node with out-edges has successors of higher rank
            mx = nm;
        }
        /* hand the predecessor chain over in the HBM array the emitter reads */
        if (cp != cpred)
            for (uint32_t v = lane; v < N; v += G) cpred[v] = cp[v];
        syncwarp();
        return mx;
    }

    RP_DEV uint32_t consensus(uint8_t* out, uint16_t* out_cov, uint32_t out_cap, bool trim, uint32_t n_seq) {
        spoa_sort(false);
        if (status != kWinOk) return 0;
        /* int32 scores in shared memory are exact iff the total edge weight fits */
        uint64_t wsum = 0;
        for (uint32_t v = lane; v < N; v += G) {
            uint32_t ni = in_cnt[v];
            for (uint32_t k = 0; k < ni; ++k) wsum += static_cast<uint32_t>(in_w[v * ki + k]);
        }
        for (int d = G / 2; d > 0; d >>= 1) wsum += shfl_down(wsum, d);
        wsum = shfl(wsum, 0);
        const uint32_t npad = (N + 7) & ~7u;
        uint32_t mx;
        if (wsum < 0x7fffffffull && npad * 6 + sizeof(CStage) * G <= smem_bytes && !(P->debug_flags & 1)) {
            int32_t* sc = reinterpret_cast<int32_t*>(smem);
            uint16_t* cp = reinterpret_cast<uint16_t*>(smem + npad * 4);
            CStage* stg = reinterpret_cast<CStage*>(smem + npad * 6);
            mx = bundle(sc, cp, stg);
        } else {
            mx = bundle(score, cpred, reinterpret_cast<CStage*>(smem));
        }
        /* walk predecessors back; the path is stored reversed in `stack`, then emitted forward */
        uint32_t clen = 0;
        if (lane == 0) {
            uint32_t v = mx;
            while (v != kNone && clen < P->lim.stack_cap) {
                stack[clen++] = static_cast<uint16_t>(v);
                v = cpred[v];
            }
        }
        clen = shfl(clen, 0);
        syncwarp();
        /* coverage (graph.cpp:388-394): node + its aligned nodes, counted as sequences through the node */
        uint32_t thr = (n_seq - 1) / 2;
        uint32_t first = 0xffffffffu, last = 0;
        for (uint32_t k = lane; k < clen; k += G) {
            uint32_t v = stack[clen - 1 - k];
            uint32_t c = cov[v];
            uint32_t na = al_cnt[v];
            for (uint32_t q = 0; q < na; ++q) c += cov[al[v * ka + q]];
            if (c > 0xffffu) c = 0xffffu;
            dp_rank[k] = static_cast<uint16_t>(c);  // dp_rank is idle here: per-base coverage scratch
            if (c >= thr) {
                if (k < first) first = k;
                if (k + 1 > last) last = k + 1;
            }
        }
        return finish_consensus(out, out_cov, out_cap, trim, clen, first, last);
    }

    RP_DEV uint32_t finish_consensus(uint8_t* out, uint16_t* out_cov, uint32_t out_cap, bool trim, uint32_t clen,
                                      uint32_t first, uint32_t last) {
        for (int d = G / 2; d > 0; d >>= 1) {
            uint32_t of = shfl_down(first, d), ol = shfl_down(last, d);
            if (of < first) first = of;
            if (ol > last) last = ol;
        }
        first = shfl(first, 0);
        last = shfl(last, 0);
        uint32_t b = 0, e = clen;  // [b, e)
        if (trim) {
            /* window.cpp:125-146: begin = first index with coverage >= thr, end = last such index;
             * keep [begin, end] only when begin < end */
            if (first != 0xffffffffu && last >= 1 && first < last - 1) {
                b = first;
                e = last;
            }
        }
        uint32_t n = e - b;
        if (n > out_cap) {
            fail(kWinInternal);
            return 0;
        }
        for (uint32_t k = b + lane; k < e; k += G) {
            uint32_t v = stack[clen - 1 - k];
            out[k - b] = code[v];
            out_cov[k - b] = cur_cov(k);
        }
        syncwarp();
        return n;
    }

    RP_DEV uint16_t cur_cov(uint32_t k) const { return dp_rank[k]; }
};

/* spoa's worst-case alignment score (alignment_engine.cpp:101-110); int16 is safe iff it stays above
 * INT16_MIN + 1024 (simd impl :699-745) */
RP_DEV int64_t worst_case_score(int32_t m, int32_t g, int64_t len, int64_t nodes) {
    int64_t i = len + 8, j = nodes;
    int64_t mn = i < j ? i : j;
    int64_t df = i > j ? i - j : j - i;
    int64_t a = -1 * (m * mn + g * df);
    int64_t b = g * i + g * j;
    return a < b ? a : b;
}
RP_DEV bool fits_int16(int32_t m, int32_t g, int64_t len, int64_t nodes) {
    if (g < -kMaxGapInt16) return false;
    return worst_case_score(m, g, len, nodes) >= static_cast<int64_t>(-32768 + 1024);
}

/* Processes one window end to end. `slot`: this group's HBM scratch, `smem`: this group's shared memory. */
template <int G, int KB = 16>
RP_DEV void poa_window(const PoaParams& P, uint32_t w, uint8_t* slot, uint8_t* smem) {
    using PW = PoaWarp<G, KB>;
    constexpr uint32_t kCC = PW::kCC;
    constexpr uint32_t kBW = PW::kBW;
    constexpr uint32_t NB = PW::NB;
    PW W;
    W.bind(&P, slot, smem, P.smem_per_group);
    W.status = kWinOk;
    const uint32_t s0 = P.win_first[w], s1 = P.win_first[w + 1];
    W.alpha = P.win_alpha[w];
    uint32_t nc = 0;
    while (nc < 8 && ((W.alpha >> (8 * nc)) & 0xff) != 0) ++nc;
    W.ncodes = nc;
    const uint32_t lane = W.lane;
    uint8_t* out = P.cons + P.out_off[w];
    uint16_t* out_cov = P.cons_cov + P.out_off[w];

    uint32_t boff = P.seq_off[s0];
    uint32_t blen = P.seq_off[s0 + 1] - boff;
    if (blen > P.lim.nmax) {
        if (lane == 0) {
            P.status[w] = kWinNodeLimit;
            P.cons_len[w] = 0;
        }
        return;
    }
    W.init_backbone(P.bases + boff, P.weights + boff, blen);

    for (uint32_t s = s0 + 1; s < s1 && W.status == kWinOk; ++s) {
        uint32_t off = P.seq_off[s];
        uint32_t len = P.seq_off[s + 1] - off;
        const uint8_t* seq = P.bases + off;
        const uint8_t* wts = P.weights + off;
        if (len > P.lim.lmax) {
            W.fail(kWinSeqTooLong);
            break;
        }
        bool sub = !(P.seq_flags[s] & 1);
        uint32_t nrows = W.N;
        uint32_t b0 = 0, span = blen;   // backbone interval the layer covers (band centre line)
        if (sub) {
            b0 = P.seq_begin[s];
            const uint32_t e0 = P.seq_end[s];
            span = e0 >= b0 ? e0 - b0 + 1 : 1;
            W.mark_subgraph(b0, e0);
            if (W.status != kWinOk) break;
            nrows = W.build_dp_order_subgraph();
        }
        /* spoa picks its int32 engine from a worst-case bound over ALL nodes of the graph (fits_int16).  That bound
         * is far from what a real matrix holds (column 0 only falls by |g| per level of graph DEPTH), and exact
         * arithmetic gives the same answer in either width, so a window that fails the bound is still computed in
         * int16 and the finished matrix is checked for having stayed in range (matrix_in_range).  The bound says
         * nothing about the top of the range: a long copy of the read scores up to max(match, mismatch) per column even
         * where the bound holds (a deep graph), and spoa's int16 engine wraps there, so such a window is refused. */
        const int64_t worst = worst_case_score(P.match, P.gap, len, nrows);
        const bool fits = P.gap >= -kMaxGapInt16 && worst >= static_cast<int64_t>(-32768 + 1024);
        const int64_t short_side = static_cast<int64_t>(len) + 8 < nrows ? static_cast<int64_t>(len) + 8 : nrows;
        const int64_t top_step = P.match > P.mismatch ? (P.match > 0 ? P.match : 0) : (P.mismatch > 0 ? P.mismatch : 0);
        if (P.gap < -kMaxGapInt16 || top_step * short_side > 32767 - 1024) {
            W.fail(kWinNeedsInt32);
            break;
        }
        const bool verify_range = !fits;
        const uint32_t lpa = (len + 1 + kCC - 1) / kCC * kCC;
        /* shared memory (chunk-local): profile chunk | ring of the last R DP rows; the traceback re-uses it */
        const uint32_t prof_bytes = W.ncodes * kCC * 2;
        const uint32_t tb_bytes = 8 * PW::kTileRowBytes + 32 + len;  // at least 8 tile rows + the read
        if (prof_bytes + 2 * kCC * 2 > P.smem_per_group || tb_bytes > P.smem_per_group) {
            W.fail(kWinSeqTooLong);
            break;
        }
        uint32_t ring_rows = (P.smem_per_group - prof_bytes) / (kCC * 2);
        if (ring_rows > 32) ring_rows = 32;
        W.prof = reinterpret_cast<int16_t*>(smem);
        W.ring = reinterpret_cast<int16_t*>(smem + prof_bytes);
        /* racon -b: the alignment is first tried inside a band of 16*G columns.  Preconditions: the row is longer
         * than the band, band starts fit a byte, the band rows fit the matrix scratch, and real scores are
         * separated from anything derived from an excluded cell (worst > kBandFloor + match * len). */
        const uint32_t nblk = (len + 16) >> 4;
        const bool band = P.banded && nblk > NB && nblk - NB <= 255u && fits &&
                          worst > static_cast<int64_t>(kBandFloor) + static_cast<int64_t>(P.match > 0 ? P.match : 0) * (len + 8) &&
                          static_cast<uint64_t>(nrows + 1) * kBW <= P.lim.hcap;
        uint32_t pred_rows = W.build_program(nrows, sub, band, len, b0, span);
        uint32_t best_row, n_best;
        int32_t best;
        bool done = false;
        if (band) {
            /* the band's profile and ring rows are narrower than a full chunk's: more ring rows fit */
            const uint32_t bprof = W.ncodes * kBW * 2;
            uint32_t bring = (P.smem_per_group - bprof) / (kBW * 2);
            if (bring > 32) bring = 32;
            W.ring = reinterpret_cast<int16_t*>(smem + bprof);
            W.dp_band(seq, nrows, len, bring, &best_row, &best, &n_best);
            W.ring = reinterpret_cast<int16_t*>(smem + prof_bytes);
            done = best_row != 0;
            if (done && n_best > 1) {
                best_row = W.template resolve_sink_tie<true>(nrows, len, lpa, best, sub);
                if (W.status != kWinOk) break;
            }
            if (done) done = W.template traceback<true>(best_row, len, lpa, seq, sub, static_cast<int32_t>(worst));
            if (P.band_stats && lane == 0) {
                count_add(P.band_stats, 1);
                if (!done) count_add(P.band_stats + 1, 1);
            }
            if (W.status != kWinOk) break;
        }
        /* tests only (debug_flags bit 1): every accepted band result is recomputed with the full matrix and compared */
        const bool audit = done && (P.debug_flags & 2u) && static_cast<uint64_t>(nrows + 1) * lpa <= P.lim.hcap;
        if (audit) {
            for (uint32_t c = lane; c < len; c += G) W.cur[c] = W.aln[c];
            W.syncwarp();
            done = false;
        }
        if (!done) {
            if (static_cast<uint64_t>(nrows + 1) * lpa > P.lim.hcap) {
                W.fail(kWinMatrixLimit);
                break;
            }
            W.dp(seq, nrows, len, lpa, ring_rows, &best_row, &best, &n_best);
            if (verify_range && !W.matrix_in_range(nrows, len, lpa)) {
                W.fail(kWinNeedsInt32);
                break;
            }
            if (n_best > 1) {
                best_row = W.template resolve_sink_tie<false>(nrows, len, lpa, best, sub);
                if (W.status != kWinOk) break;
            }
            W.template traceback<false>(best_row, len, lpa, seq, sub, 0);
            if (audit) {
                bool diff = false;
                for (uint32_t c = lane; c < len; c += G) diff |= W.cur[c] != W.aln[c];
                if (W.ballot(diff) && lane == 0 && P.band_stats) count_add(P.band_stats + 2, 1);
            }
        }
        W.add_alignment(seq, wts, len, b0);
        if (P.stats) pred_rows = W.warp_incl_sum(pred_rows);
        if (P.stats) pred_rows = W.shfl(pred_rows, G - 1);
        if (P.stats && lane == 0) {
            const unsigned long long cols = (band && done) ? kBW : len + 1;   // columns the accepted DP computed per row
            count_add(P.stats + 3, pred_rows * cols);
            count_add(P.stats, 1);
            count_add(P.stats + 1, (nrows + 1) * cols);
            if (n_best > 1) count_add(P.stats + 2, 1);
        }
    }
    uint32_t clen = 0;
    if (W.status == kWinOk) clen = W.consensus(out, out_cov, P.out_cap[w], (P.win_flags[w] & 1) != 0, s1 - s0);
    if (lane == 0) {
        P.status[w] = W.status;
        P.cons_len[w] = W.status == kWinOk ? clen : 0;
    }
    W.syncwarp();
}

}  // namespace rp
