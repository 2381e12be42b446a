/*
 * sim_main.cu — TEST-ONLY host simulation of the device code (built by racon_b200/build.py:build_sim
 * with g++ -x c++ -DRP_HOST_SIM=1 into racon_b200/lib/libracon_sim.so).
 *
 * It runs the very same poa_core.cuh / myers_core.cuh device functions with each simulated warp as
 * 32 cooperative fibres (rp_warp.cuh), and the very same host packing (poa_pack.hpp), so that the
 * CPU-only test suite can exercise graph merge, order maintenance, traceback, consensus etc. under
 * gdb/ASan.  It is not part of libracon_b200.so and nothing in the product path links or loads it.
 */
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "myers_core.cuh"
#include "poa_core.cuh"
#include "poa_pack.hpp"

namespace {

void* sim_alloc(size_t n) { return std::malloc(n ? n : 1); }
void sim_free(void* p) { std::free(p); }
const rp::HostAllocator kSimAlloc{sim_alloc, sim_free};

struct Job {
    const rp::PoaParams* P;
    uint32_t w;
    uint8_t* slot;
    uint8_t* smem;
};

struct AlnJob {
    const rp::AlnParams* P;
    uint32_t p;
    uint8_t* slot;
};

void aln_entry(void* arg) {
    AlnJob* j = static_cast<AlnJob*>(arg);
    rp::aln_pair(*j->P, j->p, j->slot);
}

template <int G, int KB>
void group_entry(void* arg) {
    Job* j = static_cast<Job*>(arg);
    rp::poa_window<G, KB>(*j->P, j->w, j->slot, j->smem);
}

}  // namespace

extern "C" {

/* Pairwise alignment through the simulated device code.  runs: n_pairs x run_stride uint32 ((count << 8) | op).  A pair
 * with a sequence longer than max_len gets status kAlnTooLong, no runs and distance -1.  With window_length != 0 also
 * breaking points: bp = n_pairs x bp_stride (t, q) points, n_bp = points per pair; with 0, t_begin, q_start, bp and
 * n_bp may be null. */
int rp_sim_aln_bp(uint32_t n_pairs, const uint8_t* bases, const uint32_t* q_off, const uint32_t* q_len,
                  const uint32_t* t_off, const uint32_t* t_len, uint32_t max_len, uint32_t store_words, uint32_t* runs,
                  uint32_t run_stride, uint32_t* n_runs, int32_t* dist, uint32_t* status, uint32_t window_length,
                  const uint32_t* t_begin, const uint32_t* q_start, uint32_t* bp, uint32_t bp_stride, uint32_t* n_bp) {
    rp::AlnParams P;
    std::memset(&P, 0, sizeof(P));
    P.n_pairs = n_pairs;
    P.bases = bases;
    P.q_off = q_off;
    P.q_len = q_len;
    P.t_off = t_off;
    P.t_len = t_len;
    std::vector<uint32_t> roff(n_pairs), rcap(n_pairs, run_stride), boff(n_pairs), bcap(n_pairs, bp_stride);
    for (uint32_t p = 0; p < n_pairs; ++p) {
        roff[p] = p * run_stride;
        boff[p] = p * bp_stride;
    }
    P.runs = runs;
    P.run_off = roff.data();
    P.run_cap = rcap.data();
    P.n_runs = n_runs;
    P.dist = dist;
    P.status = status;
    P.window_length = window_length;
    P.t_begin = t_begin;
    P.q_start = q_start;
    P.bp = bp;
    P.bp_off = boff.data();
    P.bp_cap = bcap.data();
    P.n_bp = n_bp;
    P.lim.max_len = max_len;
    P.lim.store_words = store_words;
    P.lay = rp::make_aln_layout(P.lim);
    std::vector<uint8_t> slot(P.lay.bytes + 64);
    uint8_t* slot_al = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(slot.data()) + 15) & ~uintptr_t(15));
    for (uint32_t p = 0; p < n_pairs; ++p) {
        if (q_len[p] > max_len || t_len[p] > max_len) {
            status[p] = rp::kAlnTooLong;
            n_runs[p] = 0;
            dist[p] = -1;
            continue;
        }
        AlnJob job{&P, p, slot_al};
        rp::sim::run_warp(aln_entry, &job);
    }
    return 0;
}

/* The same without breaking points. */
int rp_sim_aln(uint32_t n_pairs, const uint8_t* bases, const uint32_t* q_off, const uint32_t* q_len,
               const uint32_t* t_off, const uint32_t* t_len, uint32_t max_len, uint32_t store_words, uint32_t* runs,
               uint32_t run_stride, uint32_t* n_runs, int32_t* dist, uint32_t* status) {
    return rp_sim_aln_bp(n_pairs, bases, q_off, q_len, t_off, t_len, max_len, store_words, runs, run_stride, n_runs, dist,
                         status, 0, nullptr, nullptr, nullptr, 0, nullptr);
}

unsigned long rp_sim_leaf_pairs() { return rp::g_sim_leaf_pairs; }
/* Flat window set in, consensus out.  limits: {nmax, lmax, ki, ka, smem_per_group, tile_rows, debug_flags,
 * lanes per group (8/16/32), banded, band margin, matrix scratch cells (0 = nmax x padded lmax), columns per lane
 * of a banded row (16/8/4; 8 and 4 only with 32 lanes)}.  With banded,
 * stats[4] = alignments tried in the band, stats[5] = redone with the full matrix.  Returns 0 or <0. */
int rp_sim_poa(uint32_t n_windows, const char* bases, const char* quals, const uint64_t* seq_off,
               const uint8_t* seq_has_qual, const uint32_t* seq_begin, const uint32_t* seq_end,
               const uint32_t* win_first, const uint8_t* win_type, int8_t match, int8_t mismatch, int8_t gap,
               int trim, const uint32_t* limits, char* out, uint32_t stride, uint32_t* out_len, uint8_t* polished,
               uint32_t* status, uint16_t* cov_out, uint64_t* stats) {
    rp::PackedBatch pb(&kSimAlloc);
    for (uint32_t w = 0; w < n_windows; ++w) {
        uint32_t s0 = win_first[w], s1 = win_first[w + 1];
        std::vector<const char*> sp, qp;
        std::vector<uint32_t> ln, bg, en;
        for (uint32_t s = s0; s < s1; ++s) {
            sp.push_back(bases + seq_off[s]);
            bool q = quals && seq_has_qual && seq_has_qual[s];
            qp.push_back(q ? quals + seq_off[s] : nullptr);
            ln.push_back(static_cast<uint32_t>(seq_off[s + 1] - seq_off[s]));
            bg.push_back(seq_begin[s]);
            en.push_back(seq_end[s]);
        }
        int r = pb.add(s1 - s0, sp.data(), ln.data(), qp.data(), bg.data(), en.data(), win_type[w], trim);
        if (r != rp::kPackOk) return -100 + r;
    }
    pb.build_queue();

    rp::PoaParams P;
    std::memset(&P, 0, sizeof(P));
    rp::set_scores(P, match, mismatch, gap);
    P.n_windows = pb.n_gpu();
    P.bases = pb.bases.data;
    P.weights = pb.weights.data;
    P.seq_off = pb.seq_off.data;
    P.seq_begin = pb.seq_begin.data;
    P.seq_end = pb.seq_end.data;
    P.seq_flags = pb.seq_flags.data;
    P.win_first = pb.win_first.data;
    P.win_flags = pb.win_flags.data;
    P.win_alpha = pb.win_alpha.data;
    P.queue = pb.queue.data;
    uint32_t head = 0;
    P.queue_head = &head;
    std::vector<uint8_t> cons(pb.out_total + 16);
    std::vector<uint16_t> cov(pb.out_total + 16);
    std::vector<uint32_t> clen(pb.n_gpu() + 1), st(pb.n_gpu() + 1);
    P.cons = cons.data();
    P.cons_cov = cov.data();
    P.out_off = pb.out_off.data;
    P.out_cap = pb.out_cap.data;
    P.cons_len = clen.data();
    P.status = st.data();
    P.stats = stats;
    P.lim.nmax = limits[0];
    P.lim.lmax = limits[1];
    P.lim.lp = (limits[1] + 1 + rp::kChunkCols - 1) / rp::kChunkCols * rp::kChunkCols;
    P.lim.ki = limits[2];
    P.lim.ka = limits[3];
    P.lim.stack_cap = limits[0] * 4 + 64;
    P.lim.hcap = limits[10] ? limits[10] : (limits[0] + 1) * P.lim.lp;
    P.lay = rp::make_layout(P.lim);
    P.smem_per_group = limits[4];
    P.tile_rows = limits[5];
    P.debug_flags = limits[6];
    const uint32_t lanes = limits[7] ? limits[7] : 32;
    P.banded = limits[8];
    P.band_margin = limits[9];
    P.band_stats = (stats && P.banded) ? reinterpret_cast<unsigned long long*>(stats + 4) : nullptr;
    std::vector<uint8_t> slot(P.lay.bytes + 64);
    std::vector<uint8_t> smem(P.smem_per_group + 64);
    uint8_t* slot_al = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(slot.data()) + 15) & ~uintptr_t(15));
    uint8_t* smem_al = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem.data()) + 15) & ~uintptr_t(15));
    P.scratch = slot_al;

    for (uint32_t q = 0; q < pb.n_gpu(); ++q) {
        Job job{&P, pb.queue.data[q], slot_al, smem_al};
        const uint32_t kb = limits[11] ? limits[11] : 16;   // columns per lane of a banded row
        if (lanes == 8)
            rp::sim::run_warp(group_entry<8, 16>, &job, 256 * 1024, 8);
        else if (lanes == 16)
            rp::sim::run_warp(group_entry<16, 16>, &job, 256 * 1024, 16);
        else if (kb == 4)
            rp::sim::run_warp(group_entry<32, 4>, &job, 256 * 1024, 32);
        else if (kb == 8)
            rp::sim::run_warp(group_entry<32, 8>, &job, 256 * 1024, 32);
        else
            rp::sim::run_warp(group_entry<32, 16>, &job, 256 * 1024, 32);
    }

    for (uint32_t w = 0; w < n_windows; ++w) {
        int32_t gi = pb.gpu_index[w];
        char* o = out + static_cast<uint64_t>(w) * stride;
        if (gi == -1) {
            const std::string& c = pb.trivial[w];
            if (c.size() > stride) return -2;
            std::memcpy(o, c.data(), c.size());
            out_len[w] = static_cast<uint32_t>(c.size());
            polished[w] = 0;
            status[w] = 0;
        } else if (gi == -2) {
            out_len[w] = 0;
            polished[w] = 0;
            status[w] = rp::kWinAlphabetLimit;
        } else {
            uint32_t n = clen[gi];
            if (n > stride) return -2;
            std::memcpy(o, cons.data() + pb.out_off.data[gi], n);
            if (cov_out) std::memcpy(cov_out + static_cast<uint64_t>(w) * stride, cov.data() + pb.out_off.data[gi], n * 2);
            out_len[w] = n;
            status[w] = st[gi];
            polished[w] = st[gi] == rp::kWinOk ? 1 : 0;
        }
    }
    return 0;
}

}  // extern "C"
