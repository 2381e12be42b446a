/*
 * myers_core.cuh — batched global pairwise alignment with edlib-identical CIGARs (device code).
 *
 * Replaces, per overlap, what racon asks of edlib in Overlap::align_overlaps
 * (/root/reference/src/overlap.cpp:205-224): edlibAlign(query, target, NW, k=-1, TASK_PATH) + standard CIGAR.
 * The alignment edlib returns is a function of EXACT edit distances only (see oracle/myers_oracle.cpp, pinned
 * against the unmodified edlib): priority traceback up > left > diagonal below 1 MiB of alignment data,
 * Hirschberg with the smallest-split-row rule above (vendor/edlib/edlib/src/edlib.cpp:987-1097, 1128-1180,
 * 1198-1363).  Any exact banded method therefore reproduces it; this one is built for a warp:
 *
 *   * one warp per overlap, lanes = 64-bit words of the Myers/Hyyro bit-vector column (word w of the band lives
 *     in lane w % 32, slot (w / 32) % kAlnSlots), Ukkonen band of the diagonals that a path of cost <= k can touch
 *     (k + 1 rows, sliding one row per column); a column is processed in rounds of 32 words;
 *   * the horizontal carry between the words of a round: a word's carry-out depends on its carry-in only through
 *     "carry-in < 0", monotonically, so every word evaluates both cases and the chain is a generate/propagate
 *     carry chain, resolved for all words at once with two ballots and one integer add;
 *   * distance by k doubling, starting at the widest band that still fits one round (any k that succeeds gives
 *     the exact distance); Hirschberg columns with k = the known score of the sub-problem, the forward and the
 *     reverse pass of a node side by side in the two half-warps when the band fits 16 words; base cases store the
 *     vertical-(+1) and horizontal-(+1) bit-vectors of every band word (two sibling leaves side by side, by the same
 *     pass) and are walked back with edlib's move priority, the stored words of 32 columns at a time held in the lanes;
 *   * operations are written backwards into one buffer (right sub-problem first), run-length encoded, and — when
 *     a window length is set — turned into racon's breaking points (src/overlap.cpp:226-292) by the same warp.
 */
#pragma once
#include "rp_warp.cuh"

namespace rp {

#if defined(RP_HOST_SIM)
static unsigned long g_sim_leaf_pairs = 0;   // test-only: how often two leaves shared a warp
#endif

constexpr int kAlnSlots = 8;                  // band words per lane -> band of up to 256 words = 16384 rows
constexpr uint32_t kAlnMaxSyms = 16;             // distinct characters per pair (match-mask rows)
constexpr int32_t kAlnInf = 1 << 28;

enum : uint32_t {
    kAlnOk = 0,
    kAlnBandLimit = 1,
    kAlnAlphabetLimit = 2,
    kAlnStoreLimit = 3,
    kAlnInternal = 4,
    kAlnRunLimit = 5,
    kAlnTooLong = 6
};

struct AlnLimits {
    uint32_t max_len;        // longest query / target
    uint32_t store_words;    // capacity (in 64-bit words) of each of the two base-case bit-vector stores
};

struct AlnLayout {
    uint64_t peq_f, peq_r, col_l, col_r, store_pv, store_ph, store_first, store2_pv, store2_ph, store2_first, ops, stack,
        lut, bytes;
};

RP_HD AlnLayout make_aln_layout(const AlnLimits& L) {
    AlnLayout a;
    uint64_t o = 0;
    auto take = [&](uint64_t bytes) {
        uint64_t r = o;
        o = (o + bytes + 255) / 256 * 256;
        return r;
    };
    const uint64_t nw = (L.max_len + 63) / 64 + 2;
    a.peq_f = take(kAlnMaxSyms * nw * 8);
    a.peq_r = take(kAlnMaxSyms * nw * 8);
    a.col_l = take((static_cast<uint64_t>(L.max_len) + 2) * 4);
    a.col_r = take((static_cast<uint64_t>(L.max_len) + 2) * 4);
    a.store_pv = take(static_cast<uint64_t>(L.store_words) * 8);
    a.store_ph = take(static_cast<uint64_t>(L.store_words) * 8);
    a.store_first = take((static_cast<uint64_t>(L.max_len) + 2) * 4);
    a.store2_pv = take(static_cast<uint64_t>(L.store_words) * 8);   // second store set: two leaves per warp
    a.store2_ph = take(static_cast<uint64_t>(L.store_words) * 8);
    a.store2_first = take((static_cast<uint64_t>(L.max_len) + 2) * 4);
    a.ops = take(2ull * L.max_len + 64);
    a.stack = take(128 * 5 * 4);
    a.lut = take(256);
    a.bytes = (o + 4095) / 4096 * 4096;
    return a;
}

struct AlnParams {
    uint32_t n_pairs;
    const uint8_t* bases;       // all queries and targets, concatenated
    const uint32_t* q_off;
    const uint32_t* q_len;
    const uint32_t* t_off;
    const uint32_t* t_len;
    const uint32_t* queue;
    uint32_t* queue_head;
    /* outputs: run-length encoded operations ('M','I','D'), pair p at runs + run_off[p], capacity run_cap[p] */
    uint32_t* runs;             // (count << 8) | op
    const uint32_t* run_off;
    const uint32_t* run_cap;
    uint32_t* n_runs;
    int32_t* dist;
    uint32_t* status;
    /* breaking points (Overlap::find_breaking_points_from_cigar, src/overlap.cpp:226-292), when window_length != 0:
     * pair p writes n_bp[p] (t, q) points (two per window that saw a match) at bp + 2 * bp_off[p] */
    uint32_t window_length;
    const uint32_t* t_begin;    // target coordinate of the first target base of the pair
    const uint32_t* q_start;    // query coordinate (in alignment orientation) of the first query base
    uint32_t* bp;
    const uint32_t* bp_off;     // in points
    const uint32_t* bp_cap;     // in points
    uint32_t* n_bp;
    uint8_t* scratch;
    AlnLimits lim;
    AlnLayout lay;
};

struct AlnWarp {
    const AlnParams* P;
    int lane;
    uint64_t *peq_f, *peq_r, *store_pv, *store_ph, *store2_pv, *store2_ph;
    uint32_t* store2_first;
    int32_t *col_l, *col_r;
    uint32_t* store_first;
    uint8_t* ops;
    uint32_t* stack;
    uint8_t* lut;       // byte -> index among the pair's symbols (kAlnMaxSyms = not present)
    uint32_t status;
    uint32_t nsyms;     // distinct characters of the pair (<= kAlnMaxSyms); lut maps a byte to its index

    RP_DEV void bind(const AlnParams* p, uint8_t* slot) {
        P = p;
        lane = lane_id();
        const AlnLayout& y = p->lay;
        peq_f = reinterpret_cast<uint64_t*>(slot + y.peq_f);
        peq_r = reinterpret_cast<uint64_t*>(slot + y.peq_r);
        col_l = reinterpret_cast<int32_t*>(slot + y.col_l);
        col_r = reinterpret_cast<int32_t*>(slot + y.col_r);
        store_pv = reinterpret_cast<uint64_t*>(slot + y.store_pv);
        store_ph = reinterpret_cast<uint64_t*>(slot + y.store_ph);
        store_first = reinterpret_cast<uint32_t*>(slot + y.store_first);
        store2_pv = reinterpret_cast<uint64_t*>(slot + y.store2_pv);
        store2_ph = reinterpret_cast<uint64_t*>(slot + y.store2_ph);
        store2_first = reinterpret_cast<uint32_t*>(slot + y.store2_first);
        ops = slot + y.ops;
        stack = reinterpret_cast<uint32_t*>(slot + y.stack);
        lut = slot + y.lut;
        status = kAlnOk;
    }

    /* match masks of the (possibly reversed) query sub-range: peq[s * nw + w] bit b = (q[64w+b] == symbol s) */
    RP_DEV void build_peq(uint64_t* peq, const uint8_t* q, uint32_t n, bool rev) {
        /* 32 bases per step: one coalesced byte load, one ballot per symbol; lane s keeps symbol s's 32 bits */
        const uint32_t nw = (n + 63) / 64;
        uint32_t* peq32 = reinterpret_cast<uint32_t*>(peq);
        for (uint32_t g = 0; g < nw * 2; ++g) {
            const uint32_t i = g * 32 + static_cast<uint32_t>(lane);
            const bool valid = i < n;
            const uint32_t code = valid ? lut[rev ? q[n - 1 - i] : q[i]] : 0xffu;
            uint32_t mine = 0;
            for (uint32_t sidx = 0; sidx < nsyms; ++sidx) {
                const uint32_t bits = ballot(code == sidx);
                if (static_cast<uint32_t>(lane) == sidx) mine = bits;
            }
            if (lane < static_cast<int>(nsyms)) peq32[(static_cast<uint64_t>(lane) * nw + (g >> 1)) * 2 + (g & 1)] = mine;
        }
        syncwarp();
    }

    /* One problem of a banded pass: the (n x m) matrix of the query whose match masks are peq against t (read
     * backwards when rev_t), threshold k, columns 0..stop_col.  col receives the stop column (mode 1); spv, sph and
     * sfirst are the store set a mode-2 pass fills. */
    struct BandProblem {
        const uint64_t* peq;
        const uint8_t* t;
        bool rev_t;
        uint32_t n, m;
        int32_t k;
        uint32_t stop_col;
        int32_t* col;
        uint64_t *spv, *sph;
        uint32_t* sfirst;
    };

    /* One banded pass over columns 0..stop_col of the (n x m) problem with threshold k.
     * mode 0: returns H[n-1][stop_col] (the distance when stop_col == m-1), kAlnInf if the band misses it;
     * mode 1: additionally writes col[r+1] = H[r][stop_col] for every row r (kAlnInf outside the band),
     *         col[0] = stop_col + 1 (the boundary row above the matrix);
     * mode 2: additionally stores the vertical-(+1) and horizontal-(+1) words of every column (base case). */
    RP_DEV int32_t band_pass(const uint64_t* peq, uint32_t n, const uint8_t* t, uint32_t m, bool rev_t, int32_t k,
                             uint32_t stop_col, int mode, int32_t* col) {
        const BandProblem pr{peq, t, rev_t, n, m, k, stop_col, col, store_pv, store_ph, store_first};
        const int32_t span = band_span(n, m, k);
        if (span <= 32) return band_pass_t<1, 32>(pr, pr, mode);
        if (span <= 32 * kAlnSlots) return band_pass_t<kAlnSlots, 32>(pr, pr, mode);
        fail(kAlnBandLimit);
        return kAlnInf;
    }

    /* widest the band can get, in words: its k+1 rows straddle at most ceil(rows / 64) + 1 words */
    RP_DEV static int32_t band_span(uint32_t n, uint32_t m, int32_t k) {
        const int32_t delta = static_cast<int32_t>(n) - static_cast<int32_t>(m);
        const int32_t rows = (k + delta) / 2 + (k - delta) / 2 + 1;
        int32_t span = (rows + 63) / 64 + 1;
        const int32_t nw = static_cast<int32_t>((n + 63) / 64);
        return span > nw ? nw : span;
    }

    /* The two passes of one Hirschberg node — forward over the left half of the target into col_a, reverse over the
     * right half into col_b (edlib.cpp:1237-1262) — have the same n, m, k and therefore the same band geometry.
     * When that band fits 16 words they run side by side, one per half-warp; otherwise one after the other. */
    RP_DEV void band_pass_pair(const uint64_t* peq_a, const uint64_t* peq_b, uint32_t n, const uint8_t* t, uint32_t m,
                               int32_t k, uint32_t stop_a, uint32_t stop_b, int32_t* col_a, int32_t* col_b) {
        if (band_span(n, m, k) <= 16) {
            band_pass_t<1, 16>({peq_a, t, false, n, m, k, stop_a, col_a}, {peq_b, t, true, n, m, k, stop_b, col_b}, 1);
        } else {
            band_pass(peq_a, n, t, m, false, k, stop_a, 1, col_a);
            if (status != kAlnOk) return;
            band_pass(peq_b, n, t, m, true, k, stop_b, 1, col_b);
        }
    }

    RP_DEV static uint32_t rotr_w(uint32_t x, int r, int width) {  // rotate right inside the low `width` bits
        const uint32_t mask = width == 32 ? 0xffffffffu : ((1u << width) - 1u);
        x &= mask;
        return r ? ((x >> r) | (x << (width - r))) & mask : x;
    }

    /* SLOTS = band words a lane may hold at once.  With a band of <= W words (SLOTS = 1) the word that enters at
     * the bottom always lands in the lane whose previous word has just left at the top.
     * W = lanes per problem: 32 (one problem, a; b is not read) or 16 (problem a in lanes 0-15, b in lanes 16-31,
     * each with its own n, m, k, target and store set; SLOTS = 1, so every band fits one round of 16 words).
     * Every lane returns its own problem's result. */
    template <int SLOTS, int W>
    RP_DEV int32_t band_pass_t(const BandProblem& a, const BandProblem& b, int mode) {
        static_assert(W == 32 || (W == 16 && SLOTS == 1), "two problems per warp need single-slot bands");
        const bool second = W == 16 && lane >= 16;   // field by field: a selected reference would keep both in memory
        const uint64_t* peq = second ? b.peq : a.peq;
        const uint8_t* t = second ? b.t : a.t;
        const bool rev_t = second ? b.rev_t : a.rev_t;
        const uint32_t n = second ? b.n : a.n, m = second ? b.m : a.m, stop_col = second ? b.stop_col : a.stop_col;
        const int32_t k = second ? b.k : a.k;
        int32_t* col = second ? b.col : a.col;
        uint64_t* spv = second ? b.spv : a.spv;
        uint64_t* sph = second ? b.sph : a.sph;
        uint32_t* sfirst = second ? b.sfirst : a.sfirst;
        const int sl = lane & (W - 1);        // my lane inside the problem's lane group
        const int gbase = lane & ~(W - 1);    // first lane of the group
        const uint32_t last_col = W == 16 && b.stop_col > a.stop_col ? b.stop_col : a.stop_col;

        const int32_t delta = static_cast<int32_t>(n) - static_cast<int32_t>(m);
        const int32_t dlo = -((k - delta) / 2), dhi = (k + delta) / 2;  // diagonals i - j a cost-<=k path can touch
        const uint32_t nw = (n + 63) / 64;
        if (ballot(dhi < 0 || dlo > 0)) {  // k < |delta|: a band misses its corner cell (callers never ask for this)
            fail(kAlnInternal);
            return kAlnInf;
        }
        uint64_t pv[SLOTS], mv[SLOTS];
#pragma unroll
        for (int s = 0; s < SLOTS; ++s) {
            pv[s] = ~0ull;
            mv[s] = 0;
        }
        int32_t whi_prev = -1;   // last active word of the previous column
        int32_t sb = 0;          // H at the bottom row of word whi_prev (after the previous column)
        uint64_t store_pos = 0;
        const int32_t n1 = static_cast<int32_t>(n) - 1;
        uint32_t sidx_next = lut[rev_t ? t[m - 1] : t[0]];
        uint32_t tc_next = stop_col >= 1 ? (rev_t ? t[m - 2] : t[1]) : 0;
        for (uint32_t j = 0; j <= last_col; ++j) {
            const bool live = j <= stop_col;   // the other half-warp's problem may run longer
            int32_t rlo = static_cast<int32_t>(j) + dlo, rhi = static_cast<int32_t>(j) + dhi;
            if (rlo < 0) rlo = 0;
            if (rhi > n1) rhi = n1;
            const int32_t wlo = rlo >> 6, whi = rhi >> 6;
            /* the band slides one row per column, so at most one word enters at the bottom (vertical +1 everywhere);
             * the words of column 0 are still in their initial state */
            if (live) {
                if (j == 0) {
                    sb = 64 * (whi + 1);  // boundary column: H[r][-1] = r + 1
                } else if (whi != whi_prev) {
                    sb += 64;
                    if ((whi & (W - 1)) == sl) {
#pragma unroll
                        for (int q = 0; q < SLOTS; ++q)
                            if (SLOTS == 1 || q == ((whi >> 5) % SLOTS)) {
                                pv[q] = ~0ull;
                                mv[q] = 0;
                            }
                    }
                }
            }
            /* symbol index of this column's target character; the character two columns ahead and the index one
             * column ahead are already in flight */
            const uint32_t sidx = sidx_next;
            sidx_next = lut[tc_next];
            if (j + 1 < stop_col) tc_next = rev_t ? t[m - 3 - j] : t[j + 2];
            const uint64_t* peq_row = peq + static_cast<uint64_t>(sidx < nsyms ? sidx : 0) * nw;
            const bool known = sidx < nsyms;
            int32_t carry = 1;  // horizontal delta entering the top word of the band (edlib.cpp:766: hout = 1)
            int32_t last_hout = 0;
            if (mode == 2 && live && sl == 0)
                sfirst[j] = (static_cast<uint32_t>(wlo) << 16) | static_cast<uint32_t>(whi - wlo + 1);
            /* rounds of W consecutive words; with two problems per warp exactly one in both halves, also in a half
             * whose problem has ended (its band may then be empty) */
            const int32_t wend = W == 16 ? wlo : whi;
            for (int32_t w0 = wlo; w0 <= wend; w0 += W) {
                const int rot = w0 & (W - 1);
                const int pos = (sl - rot) & (W - 1);    // my word's position inside the round
                const int32_t w = w0 + pos;              // the word of this round that lives in my lane
                const bool act = live && w <= whi;
                uint64_t Pv = pv[0], Mv = mv[0];
                if (SLOTS > 1) {
                    const int s = (w >> 5) % SLOTS;
#pragma unroll
                    for (int q = 1; q < SLOTS; ++q)
                        if (q == s) {
                            Pv = pv[q];
                            Mv = mv[q];
                        }
                }
                const uint64_t Eq = (act && known) ? peq_row[w] : 0ull;
                /* The carry into a word matters to its carry-out only through "hin < 0" (it ORs bit 0 into Eq), and
                 * a negative carry-in can only lower the carry-out.  So every word evaluates both cases, and the
                 * chain "negative out = generate | (propagate & negative in)" is resolved for all words at once
                 * with two ballots and one integer add. */
                const uint64_t Eq1 = Eq | 1ull;
                const uint64_t Xh0 = (((Eq & Pv) + Pv) ^ Pv) | Eq;
                const uint64_t Xh1 = (((Eq1 & Pv) + Pv) ^ Pv) | Eq1;
                const bool neg0 = act && ((Pv & Xh0) >> 63) != 0;
                const bool neg1 = act && ((Pv & Xh1) >> 63) != 0;
                const uint32_t gen = rotr_w(ballot(neg0) >> gbase, rot, W);
                const uint32_t prop = rotr_w(ballot(neg1 && !neg0) >> gbase, rot, W);
                const uint32_t cin = carry < 0 ? 1u : 0u;
                const uint32_t negin = ((gen | prop) + gen + cin) ^ prop;  // bit p: negative carry into position p
                const bool hneg = ((negin >> pos) & 1u) != 0;
                const uint64_t Xh = hneg ? Xh1 : Xh0;
                const uint64_t Xv = Eq | Mv;
                const uint64_t Ph = Mv | ~(Xh | Pv);
                const uint64_t Mh = Pv & Xh;
                const int32_t hout = act ? static_cast<int32_t>(Ph >> 63) - static_cast<int32_t>(Mh >> 63) : 0;
                int32_t hin = shfl(hout, gbase | ((sl + W - 1) & (W - 1)));
                if (pos == 0) hin = carry;
                const uint64_t Phs = (Ph << 1) | (hin > 0 ? 1ull : 0ull);
                const uint64_t Mhs = (Mh << 1) | (hneg ? 1ull : 0ull);
                const uint64_t Pvn = Mhs | ~(Xv | Phs);
                const uint64_t Mvn = Phs & Xv;
                if (act) {
                    if (SLOTS == 1) {
                        pv[0] = Pvn;
                        mv[0] = Mvn;
                    } else {
                        const int s = (w >> 5) % SLOTS;
#pragma unroll
                        for (int q = 0; q < SLOTS; ++q)
                            if (q == s) {
                                pv[q] = Pvn;
                                mv[q] = Mvn;
                            }
                    }
                    if (mode == 2) {
                        const uint64_t spos = store_pos + static_cast<uint64_t>(w - wlo);
                        if (spos < P->lim.store_words) {
                            spv[spos] = Pvn;
                            sph[spos] = Ph;
                        } else {
                            status = kAlnStoreLimit;
                        }
                    }
                }
                /* carry into the next round = hout of the last word of this round */
                const int32_t last_w = (w0 + W - 1 <= whi) ? w0 + W - 1 : whi;
                last_hout = shfl(hout, gbase | (last_w & (W - 1)));
                carry = last_hout;
            }
            if (mode == 2 && ballot(status != kAlnOk)) {  // some lane ran out of store space
                fail(kAlnStoreLimit);
                return kAlnInf;
            }
            if (live) {
                if (mode == 2) store_pos += static_cast<uint64_t>(whi - wlo + 1);
                sb += last_hout;
                whi_prev = whi;
            }
        }
        /* H at row r of the stop column: bottom score minus the vertical deltas below r */
        const int32_t j = static_cast<int32_t>(stop_col);
        int32_t rlo = j + dlo, rhi = j + dhi;
        if (rlo < 0) rlo = 0;
        if (rhi > n1) rhi = n1;
        const int32_t wlo = rlo >> 6, whi = rhi >> 6;
        int32_t result = kAlnInf;
        if (mode == 1)
            for (uint32_t r = sl; r <= n; r += W) col[r] = (r == 0) ? j + 1 : kAlnInf;
        syncwarp();
        /* walk the words from the bottom of the band up; words of one round are handled together.  With two problems
         * per warp each band is a single round, so every lane runs the loop below once. */
        int32_t below = 0;  // sum of vertical deltas of all words below the current round
        const int32_t rounds = W == 16 ? 1 : (whi - wlo) / W + 1;
        for (int32_t rd = 0; rd < rounds; ++rd) {
            /* this round covers words (wbot-W+1 .. wbot) clipped to wlo */
            const int32_t wbot = whi - rd * W;
            const int32_t w = wbot - ((wbot - sl) & (W - 1));  // the word <= wbot congruent to my lane
            const bool act = w >= wlo && w > wbot - W;
            uint64_t Pv = 0, Mv = 0;
            if (SLOTS == 1) {
                if (act) {
                    Pv = pv[0];
                    Mv = mv[0];
                }
            } else {
                const int s = (w >> 5) % SLOTS;
#pragma unroll
                for (int q = 0; q < SLOTS; ++q)
                    if (q == s && act) {
                        Pv = pv[q];
                        Mv = mv[q];
                    }
            }
            const int32_t mine = act ? popc64(Pv) - popc64(Mv) : 0;
            /* suffix sum over the words of this round that lie below mine (larger w); round_sum over all of them */
            int32_t suffix = 0, round_sum = 0;
            for (int d = 0; d < W; ++d) {
                const int32_t ww = wbot - d;
                const int32_t v = shfl(mine, gbase | (ww & (W - 1)));
                if (ww > w) suffix += v;
                round_sum += v;
            }
            if (act) {
                const int32_t hbot = sb - below - suffix;  // H at row 64w + 63
                /* rows of my word */
                if (mode == 1) {
                    for (int b = 63; b >= 0; --b) {
                        const int32_t r = w * 64 + b;
                        if (r <= n1 && r >= rlo && r <= rhi) col[r + 1] = h_in_word(hbot, Pv, Mv, b);
                    }
                }
                if ((n1 >> 6) == w && n1 >= rlo && n1 <= rhi) result = h_in_word(hbot, Pv, Mv, n1 & 63);
            }
            below += round_sum;
        }
        /* the lane that owns row n-1 holds the result: the minimum over each group ends in its first lane */
        for (int d = W / 2; d > 0; d >>= 1) {
            int32_t o = shfl_down(result, d);
            result = o < result ? o : result;
        }
        result = shfl(result, gbase);
        syncwarp();
        return result;
    }

    /* H at row b of a band word whose bottom row (b = 63) holds hbot: hbot minus the vertical deltas of the rows
     * below b (the Pv / Mv bits above bit b) */
    RP_DEV static int32_t h_in_word(int32_t hbot, uint64_t Pv, uint64_t Mv, int b) {
        const uint64_t above = b == 63 ? 0ull : (~0ull << (b + 1));
        return hbot - (popc64(Pv & above) - popc64(Mv & above));
    }

    RP_DEV void fail(uint32_t st) {
        if (status == kAlnOk) status = st;
    }

    RP_DEV static int popc64(uint64_t x) {
        return popc(static_cast<uint32_t>(x)) + popc(static_cast<uint32_t>(x >> 32));
    }

    /* base case: store the band, then walk back with edlib's priority up > left > diagonal (edlib.cpp:987-1097).
     * Operations are written backwards: ops[--wpos]. */
    RP_DEV void base_case(const uint8_t* q, uint32_t n, const uint8_t* t, uint32_t m, int32_t best, uint32_t* wpos,
                          bool stored) {
        if (!stored) {  // (a whole pair below the 1 MiB rule arrives with the band of its distance pass stored)
            build_peq(peq_f, q, n, false);
            int32_t d = band_pass(peq_f, n, t, m, false, best, m - 1, 2, nullptr);
            if (status != kAlnOk) return;
            if (d != best) {
                fail(kAlnInternal);
                return;
            }
        }
        walk_stored(n, m, store_pv, store_ph, store_first, col_l, wpos);
    }

    /* Walks a stored band back from its bottom-right cell with edlib's priority up > left > diagonal
     * (edlib.cpp:987-1097).  spv/sph/sfirst: the store set filled by a mode-2 pass; coloff: an idle int32 array that
     * receives the start of every column in the store. */
    RP_DEV void walk_stored(uint32_t n, uint32_t m, const uint64_t* spv, const uint64_t* sph, const uint32_t* sfirst,
                            int32_t* coloff, uint32_t* wpos) {
        /* column offsets of the store: exclusive prefix of the per-column word counts */
        uint32_t run = 0;
        for (uint32_t j0 = 0; j0 < m; j0 += 32) {
            uint32_t j = j0 + lane;
            uint32_t cnt = j < m ? (sfirst[j] & 0xffffu) : 0;
            uint32_t inc = warp_incl_sum(cnt);
            if (j < m) coloff[j] = static_cast<int32_t>(run + inc - cnt);  // start of column j in the store
            run += shfl(inc, 31);
        }
        syncwarp();
        /* The walk is serial, its loads need not be: the lanes hold the stored words of 32 consecutive columns
         * (lane l: column jhi - l, band words wa and wa - 1), refilled with one round of parallel loads whenever the
         * walk leaves that block; every step then takes its column's words from the owning lane by shuffle.  All
         * lanes execute the (uniform) walk; lane 0 writes the operations. */
        int32_t i = static_cast<int32_t>(n) - 1, j = static_cast<int32_t>(m) - 1;
        uint32_t pos = *wpos;
        int32_t jhi = -1, jlo = 0, wa = 0;
        uint64_t pva = 0, pha = 0, pvb = 0, phb = 0;
        uint32_t have = 0;  // bit 0: word wa stored for my column, bit 1: word wa - 1
        while (i >= 0 && j >= 0) {
            const int32_t w = i >> 6;
            if (j > jhi || j < jlo || w > wa || w < wa - 1) {
                jhi = j;
                jlo = j >= 31 ? j - 31 : 0;
                wa = w;
                const int32_t c = j - lane;
                pva = pha = pvb = phb = 0;
                have = 0;
                if (c >= 0) {
                    const uint32_t sf = sfirst[c];
                    const int32_t wl = static_cast<int32_t>(sf >> 16), cnt = static_cast<int32_t>(sf & 0xffffu);
                    const uint64_t base = static_cast<uint64_t>(coloff[c]);
                    if (wa >= wl && wa < wl + cnt) {
                        pva = spv[base + static_cast<uint64_t>(wa - wl)];
                        pha = sph[base + static_cast<uint64_t>(wa - wl)];
                        have |= 1u;
                    }
                    if (wa - 1 >= wl && wa - 1 < wl + cnt) {
                        pvb = spv[base + static_cast<uint64_t>(wa - 1 - wl)];
                        phb = sph[base + static_cast<uint64_t>(wa - 1 - wl)];
                        have |= 2u;
                    }
                }
            }
            const int src = jhi - j;
            const bool first_word = w == wa;
            const uint64_t pv = shfl(first_word ? pva : pvb, src);
            const uint64_t ph = shfl(first_word ? pha : phb, src);
            const uint32_t hv = shfl(have, src);
            if (!(hv & (first_word ? 1u : 2u))) {  // cannot happen: optimal paths stay inside the band
                status = kAlnInternal;
                break;
            }
            const uint64_t bit = 1ull << (i & 63);
            uint8_t op;
            if (pv & bit) {
                op = 'I';
                --i;
            } else if (ph & bit) {
                op = 'D';
                --j;
            } else {
                op = 'M';
                --i;
                --j;
            }
            --pos;
            if (lane == 0) ops[pos] = op;
        }
        if (status == kAlnOk) {
            /* the rest of the query / target is all insertions / deletions */
            const uint32_t ri = static_cast<uint32_t>(i + 1), rj = static_cast<uint32_t>(j + 1);
            for (uint32_t x = lane; x < ri; x += 32) ops[pos - 1 - x] = 'I';
            pos -= ri;
            for (uint32_t x = lane; x < rj; x += 32) ops[pos - 1 - x] = 'D';
            pos -= rj;
        }
        *wpos = shfl(pos, 0);
        status = shfl(status, 0);
        syncwarp();
    }


    /* Two sibling leaves of the Hirschberg tree whose bands fit 16 words, filled side by side by one two-problem
     * pass: leaf A (left child: peq_f, store set 1) in lanes 0-15, leaf B (right child: peq_r, store set 2) in lanes
     * 16-31.  Then both are walked, the right leaf first: operations are written backwards. */
    RP_DEV void leaf_pair(const uint8_t* qa, uint32_t na, const uint8_t* ta, uint32_t ma, int32_t ka, const uint8_t* qb,
                          uint32_t nb, const uint8_t* tb, uint32_t mb, int32_t kb, uint32_t* wpos) {
#if defined(RP_HOST_SIM)
        if (lane == 0) ++g_sim_leaf_pairs;
#endif
        build_peq(peq_f, qa, na, false);
        build_peq(peq_r, qb, nb, false);
        const int32_t d =
            band_pass_t<1, 16>({peq_f, ta, false, na, ma, ka, ma - 1, nullptr, store_pv, store_ph, store_first},
                               {peq_r, tb, false, nb, mb, kb, mb - 1, nullptr, store2_pv, store2_ph, store2_first}, 2);
        if (status != kAlnOk) return;
        if (ballot(d != (lane < 16 ? ka : kb))) {  // each leaf must reproduce its known score
            fail(kAlnInternal);
            return;
        }
        walk_stored(nb, mb, store2_pv, store2_ph, store2_first, col_r, wpos);
        if (status != kAlnOk) return;
        walk_stored(na, ma, store_pv, store_ph, store_first, col_l, wpos);
    }

    RP_DEV void emit_run(uint8_t op, uint32_t count, uint32_t* wpos) {
        uint32_t pos = *wpos;
        for (uint32_t x = lane; x < count; x += 32) ops[pos - 1 - x] = op;
        *wpos = pos - count;
        syncwarp();
    }

    /* Walks the pair's run-length encoded operations once (one lane: a few thousand runs) and emits, per target
     * window that saw at least one match, the first matching (t, q) and the position one past the last match
     * (src/overlap.cpp:226-292).  Window ends are i-1 for every multiple i of window_length with
     * t_begin < i < t_end, then t_end-1 (:229-235).  Returns the number of points, 0xffffffff on overflow. */
    RP_DEV uint32_t breaking_points(uint32_t p, uint32_t m, uint32_t n_runs) {
        const uint32_t w = P->window_length;
        const int64_t t_begin = P->t_begin[p], t_end = t_begin + m;
        const uint32_t* runs = P->runs + P->run_off[p];
        uint32_t* out = P->bp + 2ull * P->bp_off[p];
        const uint32_t cap = P->bp_cap[p];
        int64_t t = t_begin - 1, q = static_cast<int64_t>(P->q_start[p]) - 1;
        const int64_t i0 = (t_begin / w + 1) * static_cast<int64_t>(w);
        const int64_t none = static_cast<int64_t>(1) << 40;
        int64_t wend = i0 < t_end ? i0 - 1 : t_end - 1;
        bool found = false;
        uint32_t ft = 0, fq = 0, lt = 0, lq = 0, nb = 0;
        bool overflow = false;
        auto boundary = [&]() {
            if (found) {
                if (nb + 2 <= cap) {
                    out[2 * nb] = ft;
                    out[2 * nb + 1] = fq;
                    out[2 * nb + 2] = lt;
                    out[2 * nb + 3] = lq;
                } else {
                    overflow = true;
                }
                nb += 2;
            }
            found = false;
            if (wend == t_end - 1)
                wend = none;
            else
                wend = (wend + 1 + w < t_end) ? wend + w : t_end - 1;
        };
        for (uint32_t r = 0; r < n_runs; ++r) {
            const uint32_t run = runs[r];
            int64_t c = run >> 8;
            const uint32_t op = run & 0xffu;
            if (op == 'M') {
                while (c > 0) {
                    if (!found) {
                        found = true;
                        ft = static_cast<uint32_t>(t + 1);
                        fq = static_cast<uint32_t>(q + 1);
                    }
                    const int64_t room = wend - t;
                    const int64_t step = c < room ? c : room;
                    t += step;
                    q += step;
                    c -= step;
                    lt = static_cast<uint32_t>(t + 1);
                    lq = static_cast<uint32_t>(q + 1);
                    if (t == wend) boundary();
                }
            } else if (op == 'I') {
                q += c;
            } else {
                while (c > 0) {
                    const int64_t room = wend - t;
                    const int64_t step = c < room ? c : room;
                    t += step;
                    c -= step;
                    if (t == wend) boundary();
                }
            }
        }
        return overflow ? 0xffffffffu : nb;
    }

    /* edlib's 1 MiB rule (edlib.cpp:1155-1157): an (n x m) problem whose bit-vectors take less than 1 MiB is a base
     * case, traced back from its stored band; a larger one is split */
    RP_DEV static bool below_1mib_rule(uint32_t n, uint32_t m) {
        return 20ull * ((n + 63) / 64) * m + 8ull * m < 1024ull * 1024ull;
    }

    /* whole pair: distance, Hirschberg recursion (explicit stack), run-length encoding */
    RP_DEV void align_pair(uint32_t p) {
        const uint8_t* q = P->bases + P->q_off[p];
        const uint8_t* t = P->bases + P->t_off[p];
        const uint32_t n = P->q_len[p], m = P->t_len[p];
        status = kAlnOk;
        /* alphabet of the pair */
        nsyms = 0;
        {
            /* 256-bit "seen" bitmap per lane over a strided share of the bytes, OR-reduced across the warp */
            uint32_t seen[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (uint32_t x = lane; x < n + m; x += 32) {
                const uint32_t c = x < n ? q[x] : t[x - n];
                const uint32_t bit = 1u << (c & 31);
#pragma unroll
                for (int k = 0; k < 8; ++k) seen[k] |= (c >> 5) == static_cast<uint32_t>(k) ? bit : 0u;
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
#pragma unroll
                for (int d = 16; d >= 1; d >>= 1) seen[k] |= shfl(seen[k], lane ^ d);
            }
            uint32_t ns = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) ns += static_cast<uint32_t>(popc(seen[k]));
            nsyms = ns > kAlnMaxSyms ? 0xffffffffu : ns;
            /* byte -> symbol index table (256 B, stays in L1) for the per-column lookup of the target character:
             * lane l fills bytes 8l .. 8l+7, which all live in bitmap word l / 4 */
            {
                uint32_t myword = 0, before = 0;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    if (k == (lane >> 2)) myword = seen[k];
                    if (k < (lane >> 2)) before += static_cast<uint32_t>(popc(seen[k]));
                }
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const uint32_t c = static_cast<uint32_t>(lane) * 8 + e;
                    const uint32_t hit = (myword >> (c & 31)) & 1u;
                    const uint32_t idx = before + static_cast<uint32_t>(popc(myword & ((1u << (c & 31)) - 1u)));
                    lut[c] = static_cast<uint8_t>((hit && idx < kAlnMaxSyms) ? idx : kAlnMaxSyms);
                }
            }
            syncwarp();
            if (nsyms == 0xffffffffu) {
                nsyms = 0;
                fail(kAlnAlphabetLimit);
            }
        }
        int32_t best = -1;
        uint32_t n_out = 0;
        bool direct = false;
        if (status == kAlnOk) {
            if (n == 0 || m == 0) {
                best = static_cast<int32_t>(n + m);
            } else {
                build_peq(peq_f, q, n, false);
                /* a column costs one round per 32 band words whatever the fill, so start with the widest band that
                 * still fits one round (band = k + 1 rows); the distance found does not depend on the schedule */
                int32_t k = 64 * 29;
                const int32_t kmax = static_cast<int32_t>(n > m ? n : m);
                /* a pair below edlib's 1 MiB rule is traced back from stored bit-vectors: store them right here
                 * (any band that contains the optimal paths serves), so the pair needs no second pass */
                direct = below_1mib_rule(n, m);
                for (;;) {
                    int32_t diff = static_cast<int32_t>(n) - static_cast<int32_t>(m);
                    if (diff < 0) diff = -diff;
                    if (k >= diff) {
                        int32_t kk = k < kmax ? k : kmax;
                        int32_t d = band_pass(peq_f, n, t, m, false, kk, m - 1, direct ? 2 : 0, nullptr);
                        if (status != kAlnOk) break;
                        if (d <= kk) {
                            best = d;
                            break;
                        }
                        if (kk == kmax) {
                            fail(kAlnInternal);
                            break;
                        }
                    }
                    k *= 2;
                }
            }
        }
        uint32_t wpos = n + m;
        if (status == kAlnOk) {
            uint32_t sp = 0;
            auto push = [&](uint32_t qo, uint32_t ql, uint32_t to, uint32_t tl, int32_t b) {
                if (lane == 0) {
                    stack[sp * 5 + 0] = qo;
                    stack[sp * 5 + 1] = ql;
                    stack[sp * 5 + 2] = to;
                    stack[sp * 5 + 3] = tl;
                    stack[sp * 5 + 4] = static_cast<uint32_t>(b);
                }
                ++sp;
            };
            push(0, n, 0, m, best);
            syncwarp();
            while (sp > 0 && status == kAlnOk) {
                --sp;
                const uint32_t qo = stack[sp * 5 + 0], ql = stack[sp * 5 + 1], to = stack[sp * 5 + 2],
                               tl = stack[sp * 5 + 3];
                const int32_t b = static_cast<int32_t>(stack[sp * 5 + 4]);
                syncwarp();
                if (ql == 0 || tl == 0) {  // edlib.cpp:1136-1143
                    emit_run(ql == 0 ? 'D' : 'I', ql + tl, &wpos);
                    continue;
                }
                if (below_1mib_rule(ql, tl)) {
                    base_case(q + qo, ql, t + to, tl, b, &wpos, direct && ql == n && tl == m);
                    continue;
                }
                const uint32_t lw = tl / 2, rw = tl - lw;
                build_peq(peq_f, q + qo, ql, false);
                build_peq(peq_r, q + qo, ql, true);
                /* col_l[r+1] = L[r] (forward, left half); col_r[x+1]: reversed rows (reverse, right half) */
                band_pass_pair(peq_f, peq_r, ql, t + to, tl, b, lw - 1, rw - 1, col_l, col_r);
                if (status != kAlnOk) break;
                syncwarp();
                /* R[r] = dist(q[r..], t[lw..]) = reversed-problem cell row (ql-1-r): col_r[ql - r]; R[ql] = rw */
                uint32_t bestr = 0xffffffffu;
                for (uint32_t r = lane; r + 2 <= ql; r += 32) {
                    int32_t l = col_l[r + 1], rr = col_r[ql - (r + 1)];
                    if (l + rr == b && r < bestr) bestr = r;
                }
                for (int d = 16; d > 0; d >>= 1) {
                    uint32_t o = shfl_down(bestr, d);
                    bestr = o < bestr ? o : bestr;
                }
                bestr = shfl(bestr, 0);
                int32_t split, ls, rs;
                if (bestr != 0xffffffffu) {
                    split = static_cast<int32_t>(bestr);
                    ls = col_l[bestr + 1];
                    rs = col_r[ql - (bestr + 1)];
                } else if (static_cast<int32_t>(lw) + col_r[ql] == b) {  // boundary row -1: R[0] = col_r[ql]
                    split = -1;
                    ls = static_cast<int32_t>(lw);
                    rs = col_r[ql];
                } else if (col_l[ql] + static_cast<int32_t>(rw) == b) {   // boundary row ql-1: L[ql-1] = col_l[ql]
                    split = static_cast<int32_t>(ql) - 1;
                    ls = col_l[ql];
                    rs = static_cast<int32_t>(rw);
                } else {
                    fail(kAlnInternal);
                    break;
                }
                const uint32_t ul = static_cast<uint32_t>(split + 1);
                if (sp + 2 > 120) {
                    fail(kAlnInternal);
                    break;
                }
                const uint32_t qa_n = ul, qb_n = ql - ul;
                if (qa_n > 0 && qb_n > 0 && lw > 0 && rw > 0 && below_1mib_rule(qa_n, lw) &&
                    below_1mib_rule(qb_n, rw) && band_span(qa_n, lw, ls) <= 16 && band_span(qb_n, rw, rs) <= 16) {
                    /* both children are base cases with narrow bands: fill them side by side, then walk right, left */
                    leaf_pair(q + qo, qa_n, t + to, lw, ls, q + qo + ul, qb_n, t + to + lw, rw, rs, &wpos);
                    continue;
                }
                push(qo, ul, to, lw, ls);
                push(qo + ul, ql - ul, to + lw, rw, rs);  // popped first: operations are written backwards
                syncwarp();
            }
        }
        /* run-length encode ops[wpos .. n+m) */
        if (status == kAlnOk) {
            const uint32_t total = n + m - wpos;
            const uint8_t* o = ops + wpos;
            uint32_t* out = P->runs + P->run_off[p];
            const uint32_t cap = P->run_cap[p];
            uint32_t base = 0;
            for (uint32_t x0 = 0; x0 < total; x0 += 32) {
                uint32_t x = x0 + lane;
                bool start = x < total && (x == 0 || o[x] != o[x - 1]);
                uint32_t tot;
                uint32_t pos = warp_rank(start, &tot);
                if (start) {
                    /* run length: scan forward (runs are short on real data; long runs cost one lane) */
                    uint32_t e = x + 1;
                    while (e < total && o[e] == o[x]) ++e;
                    if (base + pos < cap) out[base + pos] = ((e - x) << 8) | o[x];
                }
                base += tot;
            }
            n_out = base;
            if (n_out > cap) fail(kAlnRunLimit);
        }
        syncwarp();
        if (P->window_length != 0) {
            uint32_t nb = 0;
            if (status == kAlnOk && lane == 0) nb = breaking_points(p, m, n_out);
            nb = shfl(nb, 0);
            if (nb == 0xffffffffu) {
                fail(kAlnInternal);
                nb = 0;
            }
            if (lane == 0) P->n_bp[p] = nb;
        }
        if (lane == 0) {
            P->status[p] = status;
            P->dist[p] = status == kAlnOk ? best : -1;
            P->n_runs[p] = status == kAlnOk ? n_out : 0;
        }
        syncwarp();
    }
};

RP_DEV void aln_pair(const AlnParams& P, uint32_t p, uint8_t* slot) {
    AlnWarp W;
    W.bind(&P, slot);
    W.align_pair(p);
}

}  // namespace rp
