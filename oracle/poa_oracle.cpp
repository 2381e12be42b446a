/*
 * poa_oracle.cpp — CPU ORACLE.  TEST INFRASTRUCTURE ONLY: never linked into, called by, or shipped
 * with the product library.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg use it.
 *
 * A from-scratch restatement (index-based arrays, scalar int32 arithmetic) of the reference's
 * per-window POA consensus path.  Each function cites the reference lines it restates:
 *   Window::generate_consensus            /root/reference/src/window.cpp:65-149
 *   Graph::AddAlignment/AddSequence/...   /root/reference/vendor/spoa/src/graph.cpp:76-110,155-247
 *   Graph::TopologicalSort                /root/reference/vendor/spoa/src/graph.cpp:249-303
 *   Graph::TraverseHeaviestBundle etc.    /root/reference/vendor/spoa/src/graph.cpp:377-516
 *   Graph::Subgraph/ExtractSubgraph       /root/reference/vendor/spoa/src/graph.cpp:518-605
 *   NW-linear DP + traceback              /root/reference/vendor/spoa/src/sisd_alignment_engine.cpp:118-254,292-460
 *   (the AVX2 engine, simd_alignment_engine_implementation.hpp:506-1109, computes the same values)
 *
 * PINNING: tests/test_oracle.py checks this file against (a) the SURVEY.md §8(d) known-answer
 * checksums produced by the reference, (b) oracle/_ref (the unmodified reference compiled here)
 * window by window on synthetic full-span, partial-span, quality-weighted and NGS windows, and
 * (c) golden fixtures under tests/golden/ generated from oracle/_ref.
 *
 * The only non-"plain C" piece is std::sort for the layer order: the reference sorts layer indices
 * with std::sort (unstable; window.cpp:85-86), so bit-identical layer order for equal keys needs the
 * same libstdc++ algorithm.
 */
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

namespace {

struct Stats {
    std::atomic<uint64_t> alignments{0}, cells{0}, pred_cells{0}, sink_ties{0}, multi_sink{0},
        subgraph_alignments{0}, branch_completions{0}, max_nodes{0}, max_indeg{0}, max_aligned{0},
        far_pred_rows{0}, pred_rows{0};
};
Stats g_stats;

/* oracle_poa_trace_begin/_end: while on, every alignment appends (read length, graph rows, lowest column-0 value, lowest
 * and highest cell) of its finished int32 matrix.  Single-threaded runs only (n_threads == 1). */
bool g_trace_on = false;
std::vector<int64_t> g_trace;

/* oracle_poa_set_tie_rules: TESTS ONLY.  Each set bit replaces one of spoa's tie rules with its opposite, so that a test
 * can show that its windows reach the rule (the consensus changes); 0, the default, is spoa. */
enum : uint32_t {
    kTieLastInEdgeDiag = 1u << 0,    // traceback, diagonal step: the last explaining in-edge instead of the first
    kTieHorizFirst = 1u << 1,        // traceback: horizontal step before vertical
    kTieLastSink = 1u << 2,          // last tied sink in rank order instead of the first
    kTieBundleStrict = 1u << 3,      // heaviest bundle, equal weights: scores[pred] < scores[tail] instead of <=
    kTieLastBestNode = 1u << 4,      // heaviest bundle: the last best node in rank order instead of the first
};
std::atomic<uint32_t> g_tie_rules{0};

bool tie_rule(uint32_t bit) { return (g_tie_rules.load(std::memory_order_relaxed) & bit) != 0; }

/* the heaviest-bundle choice of graph.cpp:448-449 / 500-501 between the current predecessor and tail t */
bool heavier_edge(int64_t weight, int64_t score, int64_t pred_score, int64_t tail_score) {
    if (score != weight) return score < weight;
    return tie_rule(kTieBundleStrict) ? pred_score < tail_score : pred_score <= tail_score;
}

/* graph.cpp:454-456 / 506-508: is `s` a new best node score over `best`? */
bool new_best(int64_t best, int64_t s) { return tie_rule(kTieLastBestNode) ? best <= s : best < s; }

struct Edge {
    uint32_t tail, head;
    int64_t weight;
    std::vector<uint32_t> labels;
};

struct Graph {
    // node arrays
    std::vector<uint8_t> code;  // the character itself (spoa's dense coder_ only renames characters)
    std::vector<std::vector<uint32_t>> inedges, outedges;  // edge indices, creation order
    std::vector<std::vector<uint32_t>> aligned;
    std::vector<Edge> edges;
    std::vector<uint32_t> rank_to_node;
    uint32_t n_sequences = 0;

    uint32_t size() const { return static_cast<uint32_t>(code.size()); }

    uint32_t add_node(uint8_t c) {  // graph.cpp:76-79
        code.push_back(c);
        inedges.emplace_back();
        outedges.emplace_back();
        aligned.emplace_back();
        return size() - 1;
    }

    void add_edge(uint32_t tail, uint32_t head, uint32_t w) {  // graph.cpp:81-91
        for (uint32_t e : outedges[tail]) {
            if (edges[e].head == head) {
                edges[e].labels.push_back(n_sequences);
                edges[e].weight += w;
                return;
            }
        }
        edges.push_back(Edge{tail, head, static_cast<int64_t>(w), {n_sequences}});
        uint32_t e = static_cast<uint32_t>(edges.size() - 1);
        outedges[tail].push_back(e);
        inedges[head].push_back(e);
    }

    // graph.cpp:93-110; returns first node id or -1
    int64_t add_sequence(const char* seq, const std::vector<uint32_t>& w, uint32_t begin, uint32_t end) {
        if (begin == end) return -1;
        int64_t prev = -1;
        for (uint32_t i = begin; i < end; ++i) {
            uint32_t curr = add_node(static_cast<uint8_t>(seq[i]));
            if (prev >= 0) add_edge(static_cast<uint32_t>(prev), curr, w[i - 1] + w[i]);
            prev = curr;
        }
        return static_cast<int64_t>(size()) - (end - begin);
    }

    // graph.cpp:155-247.  alignment = (node id or -1, sequence position or -1)
    void add_alignment(const std::vector<std::pair<int32_t, int32_t>>& alignment, const char* seq,
                       uint32_t len, const std::vector<uint32_t>& w) {
        if (len == 0) return;
        if (alignment.empty()) {
            add_sequence(seq, w, 0, len);
            ++n_sequences;
            topological_sort();
            return;
        }
        std::vector<uint32_t> valid;
        for (const auto& it : alignment)
            if (it.second != -1) valid.push_back(static_cast<uint32_t>(it.second));
        // unaligned prefix / suffix chains (always empty for NW, kept for fidelity)
        int64_t begin = add_sequence(seq, w, 0, valid.front());
        int64_t prev = begin >= 0 ? static_cast<int64_t>(size()) - 1 : -1;
        int64_t last = add_sequence(seq, w, valid.back() + 1, len);
        for (const auto& it : alignment) {
            if (it.second == -1) continue;
            uint8_t c = static_cast<uint8_t>(seq[it.second]);
            int64_t curr = -1;
            if (it.first == -1) {
                curr = add_node(c);
            } else {
                uint32_t jt = static_cast<uint32_t>(it.first);
                if (code[jt] == c) {
                    curr = jt;
                } else {
                    for (uint32_t kt : aligned[jt])
                        if (code[kt] == c) {
                            curr = kt;
                            break;
                        }
                    if (curr < 0) {
                        curr = add_node(c);
                        uint32_t cu = static_cast<uint32_t>(curr);
                        for (uint32_t kt : aligned[jt]) {
                            aligned[kt].push_back(cu);
                            aligned[cu].push_back(kt);
                        }
                        aligned[jt].push_back(cu);
                        aligned[cu].push_back(jt);
                    }
                }
            }
            if (begin < 0) begin = curr;
            if (prev >= 0)
                add_edge(static_cast<uint32_t>(prev), static_cast<uint32_t>(curr), w[it.second - 1] + w[it.second]);
            prev = curr;
        }
        if (last >= 0)
            add_edge(static_cast<uint32_t>(prev), static_cast<uint32_t>(last), w[valid.back()] + w[valid.back() + 1]);
        ++n_sequences;
        topological_sort();
    }

    // graph.cpp:249-303
    void topological_sort() {
        rank_to_node.clear();
        uint32_t n = size();
        std::vector<uint8_t> marks(n, 0), ignored(n, 0);
        std::vector<uint32_t> stack;
        for (uint32_t root = 0; root < n; ++root) {
            if (marks[root] != 0) continue;
            stack.push_back(root);
            while (!stack.empty()) {
                uint32_t curr = stack.back();
                bool valid = true;
                if (marks[curr] != 2) {
                    for (uint32_t e : inedges[curr]) {
                        uint32_t t = edges[e].tail;
                        if (marks[t] != 2) {
                            stack.push_back(t);
                            valid = false;
                        }
                    }
                    if (!ignored[curr]) {
                        for (uint32_t a : aligned[curr]) {
                            if (marks[a] != 2) {
                                stack.push_back(a);
                                ignored[a] = 1;
                                valid = false;
                            }
                        }
                    }
                    if (valid) {
                        marks[curr] = 2;
                        if (!ignored[curr]) {
                            rank_to_node.push_back(curr);
                            for (uint32_t a : aligned[curr]) rank_to_node.push_back(a);
                        }
                    } else {
                        marks[curr] = 1;
                    }
                }
                if (valid) stack.pop_back();
            }
        }
    }

    // Node::Coverage, graph.cpp:32-47: distinct labels over in- and out-edges
    uint32_t coverage(uint32_t v) const {
        std::vector<uint32_t> l;
        for (uint32_t e : inedges[v]) l.insert(l.end(), edges[e].labels.begin(), edges[e].labels.end());
        for (uint32_t e : outedges[v]) l.insert(l.end(), edges[e].labels.begin(), edges[e].labels.end());
        std::sort(l.begin(), l.end());
        return static_cast<uint32_t>(std::unique(l.begin(), l.end()) - l.begin());
    }

    // graph.cpp:478-516
    int64_t branch_completion(uint32_t rank, std::vector<int64_t>& scores, std::vector<int64_t>& pred) {
        uint32_t start = rank_to_node[rank];
        for (uint32_t e : outedges[start])
            for (uint32_t f : inedges[edges[e].head])
                if (edges[f].tail != start) scores[edges[f].tail] = -1;
        int64_t max = -1;
        for (uint32_t i = rank + 1; i < rank_to_node.size(); ++i) {
            uint32_t it = rank_to_node[i];
            scores[it] = -1;
            pred[it] = -1;
            for (uint32_t e : inedges[it]) {
                uint32_t t = edges[e].tail;
                if (scores[t] == -1) continue;
                if (heavier_edge(edges[e].weight, scores[it], pred[it] >= 0 ? scores[pred[it]] : 0, scores[t])) {
                    scores[it] = edges[e].weight;
                    pred[it] = t;
                }
            }
            if (pred[it] >= 0) scores[it] += scores[pred[it]];
            if (max < 0 || new_best(scores[max], scores[it])) max = it;
        }
        return max;
    }

    // graph.cpp:433-476 + 377-398 (non-verbose summary)
    std::string generate_consensus(std::vector<uint32_t>* summary) {
        std::vector<uint32_t> cons;
        if (!rank_to_node.empty()) {
            uint32_t n = size();
            std::vector<int64_t> pred(n, -1), scores(n, -1);
            int64_t max = -1;
            for (uint32_t it : rank_to_node) {
                for (uint32_t e : inedges[it]) {
                    uint32_t t = edges[e].tail;
                    if (heavier_edge(edges[e].weight, scores[it], pred[it] >= 0 ? scores[pred[it]] : 0, scores[t])) {
                        scores[it] = edges[e].weight;
                        pred[it] = t;
                    }
                }
                if (pred[it] >= 0) scores[it] += scores[pred[it]];
                if (max < 0 || new_best(scores[max], scores[it])) max = it;
            }
            if (!outedges[max].empty()) {
                std::vector<uint32_t> node_to_rank(n, 0);
                for (uint32_t i = 0; i < rank_to_node.size(); ++i) node_to_rank[rank_to_node[i]] = i;
                while (!outedges[max].empty()) {
                    g_stats.branch_completions++;
                    max = branch_completion(node_to_rank[max], scores, pred);
                }
            }
            while (pred[max] >= 0) {
                cons.push_back(static_cast<uint32_t>(max));
                max = pred[max];
            }
            cons.push_back(static_cast<uint32_t>(max));
            std::reverse(cons.begin(), cons.end());
        }
        std::string dst;
        for (uint32_t v : cons) dst += static_cast<char>(code[v]);
        if (summary) {
            summary->clear();
            for (uint32_t v : cons) {
                uint32_t c = coverage(v);
                for (uint32_t a : aligned[v]) c += coverage(a);
                summary->push_back(c);
            }
        }
        return dst;
    }

    // graph.cpp:518-539 (called as ExtractSubgraph(nodes_[end], nodes_[begin]))
    std::vector<uint8_t> extract_subgraph(uint32_t from, uint32_t min_id) const {
        std::vector<uint8_t> dst(size(), 0);
        std::vector<uint32_t> stack{from};
        while (!stack.empty()) {
            uint32_t curr = stack.back();
            stack.pop_back();
            if (!dst[curr] && curr >= min_id) {
                for (uint32_t e : inedges[curr]) stack.push_back(edges[e].tail);
                for (uint32_t a : aligned[curr]) stack.push_back(a);
                dst[curr] = 1;
            }
        }
        return dst;
    }

    // graph.cpp:541-595
    Graph subgraph(uint32_t begin, uint32_t end, std::vector<uint32_t>* sub_to_graph) const {
        auto in_sub = extract_subgraph(end, begin);
        Graph sub;
        sub_to_graph->clear();
        std::vector<int64_t> g2s(size(), -1);
        for (uint32_t v = 0; v < size(); ++v) {
            if (!in_sub[v]) continue;
            g2s[v] = sub.add_node(code[v]);
            sub_to_graph->push_back(v);
        }
        for (uint32_t v = 0; v < size(); ++v) {
            if (!in_sub[v]) continue;
            uint32_t jt = static_cast<uint32_t>(g2s[v]);
            for (uint32_t e : inedges[v])
                if (g2s[edges[e].tail] >= 0)
                    sub.add_edge(static_cast<uint32_t>(g2s[edges[e].tail]), jt, static_cast<uint32_t>(edges[e].weight));
            for (uint32_t a : aligned[v])
                if (g2s[a] >= 0) sub.aligned[jt].push_back(static_cast<uint32_t>(g2s[a]));
        }
        sub.topological_sort();
        return sub;
    }
};

struct Engine {
    int32_t m, x, g;
    std::vector<int32_t> H;
    std::vector<uint32_t> node_to_rank;

    // sisd_alignment_engine.cpp:118-254 (Initialize, kNW+kLinear) and :292-460 (Linear)
    std::vector<std::pair<int32_t, int32_t>> align(const char* seq, uint32_t len, const Graph& graph) {
        std::vector<std::pair<int32_t, int32_t>> alignment;
        uint32_t n = graph.size();
        if (n == 0 || len == 0) return alignment;
        const uint64_t W = len + 1;
        if (H.size() < W * (n + 1)) H.resize(W * (n + 1));
        node_to_rank.resize(n);
        const auto& r2n = graph.rank_to_node;
        for (uint32_t i = 0; i < n; ++i) node_to_rank[r2n[i]] = i;

        H[0] = 0;
        for (uint64_t j = 1; j < W; ++j) H[j] = static_cast<int32_t>(j) * g;
        const int32_t kNegInf = INT32_MIN + 1024;
        for (uint32_t i = 1; i <= n; ++i) {
            const auto& in = graph.inedges[r2n[i - 1]];
            int32_t penalty = in.empty() ? 0 : kNegInf;
            for (uint32_t e : in) penalty = std::max(penalty, H[(node_to_rank[graph.edges[e].tail] + 1) * W]);
            H[i * W] = penalty + g;
        }

        int32_t max_score = kNegInf;
        uint32_t max_i = 0, max_j = 0;
        uint32_t n_sinks = 0, n_tied = 0;
        uint64_t pred_cells = 0, far = 0, prow = 0;
        std::vector<int32_t> prof(W);
        for (uint32_t i = 1; i <= n; ++i) {
            uint32_t v = r2n[i - 1];
            const auto& in = graph.inedges[v];
            uint8_t c = graph.code[v];
            prof[0] = 0;
            for (uint32_t j = 0; j < len; ++j) prof[j + 1] = (c == static_cast<uint8_t>(seq[j])) ? m : x;
            uint32_t pred_i = in.empty() ? 0 : node_to_rank[graph.edges[in[0]].tail] + 1;
            int32_t* Hr = &H[i * W];
            const int32_t* Hp = &H[pred_i * W];
            for (uint64_t j = 1; j < W; ++j) Hr[j] = std::max(Hp[j - 1] + prof[j], Hp[j] + g);
            prow++;
            if (i - pred_i > 8) far++;
            for (size_t p = 1; p < in.size(); ++p) {
                pred_i = node_to_rank[graph.edges[in[p]].tail] + 1;
                Hp = &H[pred_i * W];
                for (uint64_t j = 1; j < W; ++j) Hr[j] = std::max(Hp[j - 1] + prof[j], std::max(Hr[j], Hp[j] + g));
                prow++;
                if (i - pred_i > 8) far++;
            }
            pred_cells += W * std::max<size_t>(1, in.size());
            for (uint64_t j = 1; j < W; ++j) Hr[j] = std::max(Hr[j - 1] + g, Hr[j]);
            if (graph.outedges[v].empty()) {
                ++n_sinks;
                if (max_score < Hr[W - 1]) {
                    max_score = Hr[W - 1];
                    max_i = i;
                    max_j = static_cast<uint32_t>(W - 1);
                    n_tied = 1;
                } else if (max_score == Hr[W - 1]) {
                    ++n_tied;
                    if (tie_rule(kTieLastSink)) max_i = i;
                }
            }
        }
        g_stats.alignments++;
        g_stats.cells += W * (n + 1);
        g_stats.pred_cells += pred_cells;
        g_stats.far_pred_rows += far;
        g_stats.pred_rows += prow;
        if (n_sinks > 1) g_stats.multi_sink++;
        if (n_tied > 1) g_stats.sink_ties++;
        if (g_trace_on) {
            int64_t col0 = 0, lo = H[0], hi = H[0];
            for (uint64_t c = 0; c < W * (n + 1); ++c) {
                lo = std::min<int64_t>(lo, H[c]);
                hi = std::max<int64_t>(hi, H[c]);
                if (c % W == 0) col0 = std::min<int64_t>(col0, H[c]);
            }
            g_trace.insert(g_trace.end(), {static_cast<int64_t>(len), static_cast<int64_t>(n), col0, lo, hi});
        }
        if (max_i == 0 && max_j == 0) return alignment;

        uint32_t i = max_i, j = max_j, prev_i = 0, prev_j = 0;
        while (!(i == 0 && j == 0)) {
            int32_t Hij = H[i * W + j];
            bool found = false;
            if (i != 0 && j != 0) {
                uint32_t v = r2n[i - 1];
                const auto& in = graph.inedges[v];
                int32_t mc = (graph.code[v] == static_cast<uint8_t>(seq[j - 1])) ? m : x;
                size_t np = std::max<size_t>(1, in.size());
                const bool last_first = tie_rule(kTieLastInEdgeDiag);
                for (size_t k = 0; k < np && !found; ++k) {
                    size_t p = last_first ? np - 1 - k : k;
                    uint32_t pi = in.empty() ? 0 : node_to_rank[graph.edges[in[p]].tail] + 1;
                    if (Hij == H[pi * W + (j - 1)] + mc) {
                        prev_i = pi;
                        prev_j = j - 1;
                        found = true;
                    }
                }
            }
            const bool horiz_first = tie_rule(kTieHorizFirst);
            if (!found && horiz_first && j != 0 && Hij == H[i * W + j - 1] + g) {
                prev_i = i;
                prev_j = j - 1;
                found = true;
            }
            if (!found && i != 0) {
                const auto& in = graph.inedges[r2n[i - 1]];
                size_t np = std::max<size_t>(1, in.size());
                for (size_t p = 0; p < np && !found; ++p) {
                    uint32_t pi = in.empty() ? 0 : node_to_rank[graph.edges[in[p]].tail] + 1;
                    if (Hij == H[pi * W + j] + g) {
                        prev_i = pi;
                        prev_j = j;
                        found = true;
                    }
                }
            }
            if (!found && !horiz_first && Hij == H[i * W + j - 1] + g) {
                prev_i = i;
                prev_j = j - 1;
                found = true;
            }
            alignment.emplace_back(i == prev_i ? -1 : static_cast<int32_t>(r2n[i - 1]),
                                   j == prev_j ? -1 : static_cast<int32_t>(j - 1));
            i = prev_i;
            j = prev_j;
        }
        std::reverse(alignment.begin(), alignment.end());
        return alignment;
    }
};

struct Seq {
    const char* data;
    uint32_t len;
    const char* qual;  // nullptr => weight 1
    uint32_t begin, end;
};

std::vector<uint32_t> weights_of(const Seq& s) {  // graph.cpp:121-146
    std::vector<uint32_t> w(s.len, 1);
    if (s.qual)
        for (uint32_t i = 0; i < s.len; ++i) w[i] = static_cast<uint32_t>(static_cast<int>(s.qual[i]) - 33);
    return w;
}

/* The graph's shape, for oracle_graph_shape: node count after the backbone and after each layer (in the order the
 * layers are aligned), and the largest in-degree and aligned-set size of the final graph. */
struct Shape {
    std::vector<uint32_t> nodes;
    uint32_t max_indeg = 0, max_aligned = 0;
};

// Window::generate_consensus, window.cpp:65-149.  seqs[0] = backbone.
bool window_consensus(const std::vector<Seq>& seqs, int type_tgs, bool trim, Engine& engine, std::string* consensus,
                      std::vector<uint32_t>* coverage, Shape* shape = nullptr) {
    coverage->clear();
    if (shape) *shape = Shape{};
    if (seqs.size() < 3) {
        consensus->assign(seqs[0].data, seqs[0].len);
        return false;
    }
    Graph graph;
    graph.add_alignment({}, seqs[0].data, seqs[0].len, weights_of(seqs[0]));
    if (shape) shape->nodes.push_back(graph.size());

    std::vector<uint32_t> rank(seqs.size());
    for (uint32_t i = 0; i < seqs.size(); ++i) rank[i] = i;
    std::sort(rank.begin() + 1, rank.end(), [&](uint32_t l, uint32_t r) { return seqs[l].begin < seqs[r].begin; });

    uint32_t blen = seqs[0].len;
    uint32_t offset = static_cast<uint32_t>(0.01 * blen);
    for (uint32_t j = 1; j < seqs.size(); ++j) {
        const Seq& s = seqs[rank[j]];
        std::vector<std::pair<int32_t, int32_t>> alignment;
        if (s.begin < offset && s.end > blen - offset) {
            alignment = engine.align(s.data, s.len, graph);
        } else {
            std::vector<uint32_t> map;
            Graph sub = graph.subgraph(s.begin, s.end, &map);
            g_stats.subgraph_alignments++;
            alignment = engine.align(s.data, s.len, sub);
            for (auto& it : alignment)
                if (it.first != -1) it.first = static_cast<int32_t>(map[it.first]);  // graph.cpp:597-605
        }
        graph.add_alignment(alignment, s.data, s.len, weights_of(s));
        if (shape) shape->nodes.push_back(graph.size());
    }
    {
        uint64_t n = graph.size(), mi = 0, ma = 0;
        for (uint32_t v = 0; v < n; ++v) {
            mi = std::max<uint64_t>(mi, graph.inedges[v].size());
            ma = std::max<uint64_t>(ma, graph.aligned[v].size());
        }
        uint64_t cur = g_stats.max_nodes.load();
        while (cur < n && !g_stats.max_nodes.compare_exchange_weak(cur, n)) {}
        cur = g_stats.max_indeg.load();
        while (cur < mi && !g_stats.max_indeg.compare_exchange_weak(cur, mi)) {}
        cur = g_stats.max_aligned.load();
        while (cur < ma && !g_stats.max_aligned.compare_exchange_weak(cur, ma)) {}
        if (shape) {
            shape->max_indeg = static_cast<uint32_t>(mi);
            shape->max_aligned = static_cast<uint32_t>(ma);
        }
    }

    std::vector<uint32_t> cov;
    *consensus = graph.generate_consensus(&cov);
    if (type_tgs && trim) {
        uint32_t avg = static_cast<uint32_t>((seqs.size() - 1) / 2);
        int32_t b = 0, e = static_cast<int32_t>(consensus->size()) - 1;
        for (; b < static_cast<int32_t>(consensus->size()); ++b)
            if (cov[b] >= avg) break;
        for (; e >= 0; --e)
            if (cov[e] >= avg) break;
        if (b < e) {
            *consensus = consensus->substr(b, e - b + 1);
            cov = std::vector<uint32_t>(cov.begin() + b, cov.begin() + e + 1);
        }  // else: reference prints a "chimeric" warning and keeps the untrimmed consensus
    }
    *coverage = cov;
    return true;
}

/* oracle_poa_consensus, and with `shape_out` also each window's Shape (see oracle_graph_shape) */
double run_windows(uint32_t n_windows, const char* bases, const char* quals, const uint64_t* seq_off,
                   const uint8_t* seq_has_qual, const uint32_t* seq_begin, const uint32_t* seq_end,
                   const uint32_t* win_first, const uint8_t* win_type, int8_t match, int8_t mismatch, int8_t gap,
                   int trim, uint32_t n_threads, char* out, uint32_t out_stride, uint32_t* out_len, uint8_t* polished,
                   uint32_t* cov_out, std::vector<Shape>* shape_out) {
    if (n_threads == 0) n_threads = 1;
    std::atomic<uint32_t> next(0);
    std::atomic<int> failed(0);
    uint32_t max_bl = 1;
    for (uint32_t w = 0; w < n_windows; ++w) {
        uint32_t s0 = win_first[w];
        max_bl = std::max(max_bl, static_cast<uint32_t>(seq_off[s0 + 1] - seq_off[s0]));
    }
    const std::string dummy(max_bl, '!');
    auto t0 = std::chrono::steady_clock::now();
    auto work = [&]() {
        Engine engine{match, mismatch, gap, {}, {}};
        for (;;) {
            uint32_t w = next.fetch_add(1);
            if (w >= n_windows) break;
            std::vector<Seq> seqs;
            for (uint32_t s = win_first[w]; s < win_first[w + 1]; ++s) {
                uint64_t o = seq_off[s];
                uint32_t len = static_cast<uint32_t>(seq_off[s + 1] - o);
                bool q = quals && seq_has_qual && seq_has_qual[s];
                Seq e{bases + o, len, q ? quals + o : nullptr, seq_begin[s], seq_end[s]};
                if (s == win_first[w]) {
                    if (!q) e.qual = dummy.data();  // polisher.cpp:174,396-399: dummy '!' => weight 0
                    seqs.push_back(e);
                } else {
                    if (len == 0 || e.begin == e.end) continue;  // window.cpp:45-47
                    seqs.push_back(e);
                }
            }
            std::string cons;
            std::vector<uint32_t> cov;
            bool ok = window_consensus(seqs, win_type[w], trim != 0, engine, &cons, &cov,
                                       shape_out ? &(*shape_out)[w] : nullptr);
            if (cons.size() > out_stride) {
                failed = 1;
                continue;
            }
            std::memcpy(out + static_cast<uint64_t>(w) * out_stride, cons.data(), cons.size());
            out_len[w] = static_cast<uint32_t>(cons.size());
            polished[w] = ok ? 1 : 0;
            if (cov_out)
                for (size_t k = 0; k < cov.size(); ++k) cov_out[static_cast<uint64_t>(w) * out_stride + k] = cov[k];
        }
    };
    if (n_threads == 1) {
        work();
    } else {
        std::vector<std::thread> pool;
        for (uint32_t t = 0; t < n_threads; ++t) pool.emplace_back(work);
        for (auto& th : pool) th.join();
    }
    auto t1 = std::chrono::steady_clock::now();
    if (failed) return -1.0;
    return std::chrono::duration<double>(t1 - t0).count();
}

}  // namespace

extern "C" {

/* Same contract as ref_poa_consensus (oracle/ref_harness.cpp) plus an optional per-base coverage
 * matrix `cov_out` (n_windows x out_stride uint32, coverage of the returned consensus). */
double oracle_poa_consensus(uint32_t n_windows, const char* bases, const char* quals, const uint64_t* seq_off,
                            const uint8_t* seq_has_qual, const uint32_t* seq_begin, const uint32_t* seq_end,
                            const uint32_t* win_first, const uint8_t* win_type, int8_t match, int8_t mismatch,
                            int8_t gap, uint32_t window_length, int trim, uint32_t n_threads, char* out,
                            uint32_t out_stride, uint32_t* out_len, uint8_t* polished, uint32_t* cov_out) {
    (void)window_length;
    return run_windows(n_windows, bases, quals, seq_off, seq_has_qual, seq_begin, seq_end, win_first, win_type, match,
                       mismatch, gap, trim, n_threads, out, out_stride, out_len, polished, cov_out, nullptr);
}

/* The consensus pass of oracle_poa_consensus, reporting each window's graph shape instead of its consensus:
 * nodes = n_windows x nodes_stride uint32, the node count after the backbone and after each aligned layer, in the
 * order the layers are aligned (sorted by begin; layers skipped as empty are not counted), n_nodes = entries per
 * window (0 for windows of fewer than 3 sequences, which build no graph), max_indeg / max_aligned = the largest
 * in-degree and aligned-set size of the final graph.  Returns 0, or -1 when an output does not fit. */
int oracle_graph_shape(uint32_t n_windows, const char* bases, const char* quals, const uint64_t* seq_off,
                       const uint8_t* seq_has_qual, const uint32_t* seq_begin, const uint32_t* seq_end,
                       const uint32_t* win_first, const uint8_t* win_type, int8_t match, int8_t mismatch, int8_t gap,
                       uint32_t window_length, uint32_t n_threads, char* out, uint32_t out_stride, uint32_t* nodes,
                       uint32_t nodes_stride, uint32_t* n_nodes, uint32_t* max_indeg, uint32_t* max_aligned) {
    (void)window_length;
    std::vector<uint32_t> out_len(n_windows);
    std::vector<uint8_t> polished(n_windows);
    std::vector<Shape> shapes(n_windows);
    if (run_windows(n_windows, bases, quals, seq_off, seq_has_qual, seq_begin, seq_end, win_first, win_type, match,
                    mismatch, gap, 1, n_threads, out, out_stride, out_len.data(), polished.data(), nullptr,
                    &shapes) < 0)
        return -1;
    for (uint32_t w = 0; w < n_windows; ++w) {
        const Shape& s = shapes[w];
        if (s.nodes.size() > nodes_stride) return -1;
        std::copy(s.nodes.begin(), s.nodes.end(), nodes + static_cast<uint64_t>(w) * nodes_stride);
        n_nodes[w] = static_cast<uint32_t>(s.nodes.size());
        max_indeg[w] = s.max_indeg;
        max_aligned[w] = s.max_aligned;
    }
    return 0;
}

/* out[12]: alignments, cells, pred_cells, sink_ties, multi_sink, subgraph_alignments, branch_completions,
 * max_nodes, max_indeg, max_aligned, far_pred_rows(>8 ranks away), pred_rows.  Resets the counters. */
void oracle_poa_stats(uint64_t* out) {
    out[0] = g_stats.alignments.exchange(0);
    out[1] = g_stats.cells.exchange(0);
    out[2] = g_stats.pred_cells.exchange(0);
    out[3] = g_stats.sink_ties.exchange(0);
    out[4] = g_stats.multi_sink.exchange(0);
    out[5] = g_stats.subgraph_alignments.exchange(0);
    out[6] = g_stats.branch_completions.exchange(0);
    out[7] = g_stats.max_nodes.exchange(0);
    out[8] = g_stats.max_indeg.exchange(0);
    out[9] = g_stats.max_aligned.exchange(0);
    out[10] = g_stats.far_pred_rows.exchange(0);
    out[11] = g_stats.pred_rows.exchange(0);
}

/* TESTS ONLY: replace spoa's tie rules by the ones set in `mask` (kTie* above) for every later call; 0 restores spoa. */
void oracle_poa_set_tie_rules(uint32_t mask) { g_tie_rules = mask; }

void oracle_poa_trace_begin(void) {
    g_trace.clear();
    g_trace_on = true;
}

/* Stops the trace; copies up to `cap` records of 5 int64 (see g_trace) to `out` and returns how many were taken. */
uint64_t oracle_poa_trace_end(int64_t* out, uint64_t cap) {
    g_trace_on = false;
    const uint64_t n = g_trace.size() / 5;
    std::memcpy(out, g_trace.data(), std::min(n, cap) * 5 * sizeof(int64_t));
    return n;
}

}  // extern "C"
