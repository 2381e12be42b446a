/*
 * myers_oracle.cpp — CPU ORACLE for the pre-alignment row (SURVEY.md §8 a10 / f1).  TEST INFRASTRUCTURE ONLY.
 *
 * What racon asks of edlib (Overlap::align_overlaps, /root/reference/src/overlap.cpp:205-224):
 *   edlibAlign(query, target, NW, k = -1, TASK_PATH)  ->  edlibAlignmentToCigar(..., EDLIB_CIGAR_STANDARD)
 * edlib (vendor/edlib/edlib/src/edlib.cpp) is a banded block bit-vector implementation; this file restates
 * WHAT it computes, not how, as plain dynamic programming on exact edit distances:
 *
 *   distance      : global (NW) edit distance, unit costs (edlib.cpp:141-191; k doubling only finds it faster).
 *   alignment     : obtainAlignment (edlib.cpp:1128-1180):
 *       - empty query/target: all 'D' / all 'I' (:1136-1143);
 *       - if (2*8+4) * ceil(qlen/64) * tlen + 8 * tlen < 1 MiB: traceback from the bottom-right cell with the
 *         priority  up ('I': query base unmatched)  >  left ('D')  >  diagonal ('M')   (:987-1097).
 *         edlib can only step onto cells inside its Ukkonen band, but every cell it would step to lies on an
 *         optimal path and therefore inside any valid band, so the band never changes the outcome;
 *       - else Hirschberg (:1198-1363): split the target after leftHalfWidth = tlen / 2 columns; with
 *         L[r] = dist(query[0..r], target[0..lw-1]) and R[r] = dist(query[r..], target[lw..]) take the SMALLEST
 *         r in [0, qlen-2] with L[r] + R[r+1] == best (:1294-1302), else r = -1 if lw + R[0] == best (:1304-1311),
 *         else r = qlen-1 if L[qlen-1] + (tlen-lw) == best (:1312-1320); recurse on both parts with their scores.
 *   CIGAR         : standard format, '=' and 'X' both written as 'M', run-length encoded (:262-317).
 *
 * PINNING: tests/test_myers_oracle.py compares this file with the UNMODIFIED edlib (oracle/_ref, ref_edlib_cigar)
 * on random pairs across lengths (1 .. 6000, i.e. both the traceback and the Hirschberg regime), error rates and
 * length imbalances, and on tie-rich pairs (homopolymer-length errors, tandem repeats, low-complexity runs) in both
 * regimes, byte for byte.
 */
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace {

/* last column of the exact DP between a[0..n) and b[0..m): out[i] = dist(a[0..i), b[0..m)), i = 0..n */
void last_column(const char* a, int n, const char* b, int m, std::vector<int>& out) {
    out.resize(n + 1);
    for (int i = 0; i <= n; ++i) out[i] = i;
    for (int j = 1; j <= m; ++j) {
        int diag = out[0];
        out[0] = j;
        const char c = b[j - 1];
        for (int i = 1; i <= n; ++i) {
            int up = out[i - 1] + 1, left = out[i] + 1, d = diag + (a[i - 1] == c ? 0 : 1);
            diag = out[i];
            out[i] = std::min(d, std::min(up, left));
        }
    }
}

void traceback(const char* q, int n, const char* t, int m, std::string& ops) {
    /* full matrix (only used below edlib's 1 MiB threshold: n*m < ~3.4 M cells) */
    std::vector<int32_t> H(static_cast<size_t>(n + 1) * (m + 1));
    auto at = [&](int i, int j) -> int32_t& { return H[static_cast<size_t>(j) * (n + 1) + i]; };
    for (int i = 0; i <= n; ++i) at(i, 0) = i;
    for (int j = 1; j <= m; ++j) {
        at(0, j) = j;
        for (int i = 1; i <= n; ++i)
            at(i, j) = std::min(at(i - 1, j - 1) + (q[i - 1] == t[j - 1] ? 0 : 1), std::min(at(i - 1, j), at(i, j - 1)) + 1);
    }
    std::string rev;
    int i = n, j = m;
    while (i > 0 || j > 0) {
        if (i > 0 && j > 0) {
            if (at(i - 1, j) + 1 == at(i, j)) {  // up first
                rev.push_back('I');
                --i;
            } else if (at(i, j - 1) + 1 == at(i, j)) {  // then left
                rev.push_back('D');
                --j;
            } else {
                rev.push_back('M');
                --i;
                --j;
            }
        } else if (i > 0) {
            rev.push_back('I');
            --i;
        } else {
            rev.push_back('D');
            --j;
        }
    }
    ops.append(rev.rbegin(), rev.rend());
}

/* rule: the alignment-data size (bytes) from which on edlib switches from the traceback to Hirschberg; edlib's is
 * 1 MiB, tests move it to show that a pair's alignment depends on which side of the rule a node falls.
 * tree (optional): receives (query length, target length, score, leaf) of every node with a non-empty query and
 * target, in pre-order (a node, then its left part, then its right part). */
void obtain_alignment(const char* q, int n, const char* t, int m, int best, long long rule, std::string& ops,
                      std::vector<int32_t>* tree) {
    if (n == 0 || m == 0) {  // edlib.cpp:1136-1143
        ops.append(static_cast<size_t>(n + m), n == 0 ? 'D' : 'I');
        return;
    }
    const long long blocks = (n + 63) / 64;
    const long long data = (2 * 8 + 4) * blocks * m + 2LL * 4 * m;  // edlib.cpp:1155-1157
    const bool leaf = data < rule;
    if (tree) tree->insert(tree->end(), {n, m, best, leaf ? 1 : 0});
    if (leaf) {
        traceback(q, n, t, m, ops);
        return;
    }
    const int lw = m / 2, rw = m - lw;
    std::vector<int> L, Rr;
    last_column(q, n, t, lw, L);  // L[i] = dist(q[0..i), t[0..lw))  -> row index r = i - 1
    std::string rq(q, q + n), rt(t + lw, t + m);
    std::reverse(rq.begin(), rq.end());
    std::reverse(rt.begin(), rt.end());
    last_column(rq.data(), n, rt.data(), rw, Rr);  // Rr[k] = dist(q[n-k..n), t[lw..m))
    auto Rfrom = [&](int r) { return Rr[n - r]; };  // R[r] = dist(q[r..n), t[lw..m)), r = 0..n
    int split = -2, ls = 0, rs = 0;
    for (int r = 0; r <= n - 2; ++r) {
        if (L[r + 1] + Rfrom(r + 1) == best) {  // left cell row r, its lower-right neighbour row r+1
            split = r;
            ls = L[r + 1];
            rs = Rfrom(r + 1);
            break;
        }
    }
    if (split == -2 && lw + Rfrom(0) == best) {  // boundary row -1
        split = -1;
        ls = lw;
        rs = Rfrom(0);
    }
    if (split == -2 && L[n] + rw == best) {  // boundary row n-1
        split = n - 1;
        ls = L[n];
        rs = rw;
    }
    if (split == -2) {  // cannot happen for a correct `best`
        ops.append("?");
        return;
    }
    const int ul = split + 1;
    obtain_alignment(q, ul, t, lw, ls, rule, ops, tree);
    obtain_alignment(q + ul, n - ul, t + lw, rw, rs, rule, ops, tree);
}

int edit_distance_of(const char* q, uint32_t ql, const char* t, uint32_t tl) {
    std::vector<int> col;
    last_column(q, static_cast<int>(ql), t, static_cast<int>(tl), col);
    return col[ql];
}

}  // namespace

extern "C" {

/* CIGAR (standard format) of the alignment edlib would return for (query, target) if its 1 MiB rule were `rule`
 * bytes (edlib: 1048576); returns its length, -2 if `cap` is too small.  *edit_distance receives the NW edit
 * distance. */
int64_t oracle_myers_cigar(const char* q, uint32_t ql, const char* t, uint32_t tl, char* out, uint64_t cap,
                           int32_t* edit_distance, uint64_t rule) {
    const int best = edit_distance_of(q, ql, t, tl);
    if (edit_distance) *edit_distance = best;
    std::string ops;
    obtain_alignment(q, static_cast<int>(ql), t, static_cast<int>(tl), best, static_cast<long long>(rule), ops, nullptr);
    std::string cigar;
    for (size_t i = 0; i < ops.size();) {
        size_t j = i;
        while (j < ops.size() && ops[j] == ops[i]) ++j;
        cigar += std::to_string(j - i);
        cigar.push_back(ops[i]);
        i = j;
    }
    if (cigar.size() + 1 > cap) return -2;
    std::memcpy(out, cigar.c_str(), cigar.size() + 1);
    return static_cast<int64_t>(cigar.size());
}

/* The node tree of the same alignment: 4 int32 per node (query length, target length, score, 1 for a traceback leaf /
 * 0 for a Hirschberg split), pre-order, nodes with an empty side left out.  Returns the node count, -2 if more than
 * `cap` nodes. */
int64_t oracle_myers_tree(const char* q, uint32_t ql, const char* t, uint32_t tl, uint64_t rule, int32_t* out,
                          uint64_t cap) {
    const int best = edit_distance_of(q, ql, t, tl);
    std::string ops;
    std::vector<int32_t> tree;
    obtain_alignment(q, static_cast<int>(ql), t, static_cast<int>(tl), best, static_cast<long long>(rule), ops, &tree);
    const uint64_t nodes = tree.size() / 4;
    if (nodes > cap) return -2;
    if (!tree.empty()) std::memcpy(out, tree.data(), tree.size() * sizeof(int32_t));
    return static_cast<int64_t>(nodes);
}

}  // extern "C"
