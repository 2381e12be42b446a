/*
 * host_mirror.cpp — see host_mirror.hpp.  Thin: all work happens behind the C ABI on the GPU.
 */
#include "host_mirror.hpp"

#include <algorithm>
#include <array>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <iterator>
#include <numeric>
#include <stdexcept>

#include "racon_b200.h"
#include "reads_io.hpp"

namespace racon_b200 {
namespace {

/* A hard error (negative rp_status) ends the process with a message, as the reference's batch objects do.  A device stage
 * of the polisher owns several batch objects and read stores: while it runs (run_stage) the error is thrown instead, the
 * stage's objects are destroyed on the way out, and the read stores are released before the same message is printed. */
thread_local int hard_error_scopes = 0;

struct HardError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

[[noreturn]] void hard_error(const std::string& message) {
    if (hard_error_scopes > 0) throw HardError(message);
    fprintf(stderr, "%s\n", message.c_str());
    exit(1);
}

std::string status_text(rp_status s) { return std::string(rp_strerror(s)) + " (" + rp_last_error() + ")"; }

}  // namespace

std::shared_ptr<Window> createWindow(uint64_t id, uint32_t rank, WindowType type, const char* backbone,
                                     uint32_t backbone_length, const char* quality, uint32_t quality_length) {
    if (backbone_length == 0 || backbone_length != quality_length) {  // window.cpp:19-23
        fprintf(stderr, "[racon_b200::createWindow] error: empty backbone sequence/unequal quality length!\n");
        exit(1);
    }
    return std::shared_ptr<Window>(new Window(id, rank, type, backbone, backbone_length, quality, quality_length));
}

Window::Window(uint64_t id, uint32_t rank, WindowType type, const char* backbone, uint32_t backbone_length,
               const char* quality, uint32_t quality_length)
    : id_(id), rank_(rank), type_(type), consensus_(), sequences_(), qualities_(), positions_() {
    sequences_.emplace_back(backbone, backbone_length);
    qualities_.emplace_back(quality, quality_length);
    positions_.emplace_back(0, 0);
}

Window::~Window() {}

void Window::add_layer(const char* sequence, uint32_t sequence_length, const char* quality, uint32_t quality_length,
                       uint32_t begin, uint32_t end) {
    if (sequence_length == 0 || begin == end) return;  // window.cpp:45-47
    if (quality != nullptr && sequence_length != quality_length) {
        fprintf(stderr, "[racon_b200::Window::add_layer] error: unequal quality size!\n");
        exit(1);
    }
    if (begin >= end || begin > sequences_.front().second || end > sequences_.front().second) {
        fprintf(stderr, "[racon_b200::Window::add_layer] error: layer begin and end positions are invalid!\n");
        exit(1);
    }
    sequences_.emplace_back(sequence, sequence_length);
    qualities_.emplace_back(quality, quality_length);
    positions_.emplace_back(begin, end);
}

void Window::add_layer(const char* sequence, uint32_t sequence_length, const char* quality, uint32_t quality_length,
                       uint32_t begin, uint32_t end, const Origin& origin) {
    const size_t before = sequences_.size();
    add_layer(sequence, sequence_length, quality, quality_length, begin, end);
    if (sequences_.size() > before && origins_.size() == before) origins_.push_back(origin);
}

std::atomic<uint32_t> BatchProcessor::batches{0};

std::unique_ptr<BatchProcessor> createBatch(uint32_t max_window_depth, uint32_t device, size_t avail_mem, int8_t gap,
                                            int8_t mismatch, int8_t match, bool cuda_banded_alignment,
                                            uint32_t window_length, bool trim) {
    return std::unique_ptr<BatchProcessor>(new BatchProcessor(max_window_depth, device, avail_mem, gap, mismatch,
                                                              match, cuda_banded_alignment, window_length, trim));
}

BatchProcessor::BatchProcessor(uint32_t max_window_depth, uint32_t device, size_t avail_mem, int8_t gap,
                               int8_t mismatch, int8_t match, bool cuda_banded_alignment, uint32_t window_length,
                               bool trim)
    : trim_(trim) {
    bid_ = BatchProcessor::batches++;
    rp_status s = rp_poa_create(&poa_, static_cast<int>(device), avail_mem, match, mismatch, gap,
                                cuda_banded_alignment ? 1 : 0, window_length, max_window_depth);
    if (s != RP_OK) {  // hard failure, like GW_CU_CHECK_ERR / std::runtime_error in the reference
        hard_error("[racon_b200::BatchProcessor] error: " + status_text(s));
    }
}

BatchProcessor::~BatchProcessor() { rp_poa_destroy(poa_); }

bool BatchProcessor::addWindow(std::shared_ptr<Window> window) {
    const size_t n = window->sequences_.size();
    std::vector<const char*> seq(n), qual(n);
    std::vector<uint32_t> len(n), begin(n), end(n);
    for (size_t i = 0; i < n; ++i) {
        seq[i] = window->sequences_[i].first;
        len[i] = window->sequences_[i].second;
        qual[i] = window->qualities_[i].first;
        begin[i] = window->positions_[i].first;
        end[i] = window->positions_[i].second;
    }
    rp_status s;
    if (reads_ != nullptr && window->origins_.size() == n) {
        std::vector<uint32_t> id(n), offset(n);
        std::vector<uint8_t> reverse(n);
        for (size_t i = 0; i < n; ++i) {
            id[i] = window->origins_[i].seq_id;
            offset[i] = window->origins_[i].offset;
            reverse[i] = window->origins_[i].reverse ? 1 : 0;
        }
        s = rp_poa_add_window_refs(poa_, reads_, static_cast<uint32_t>(n), id.data(), offset.data(), len.data(),
                                   reverse.data(), begin.data(), end.data(),
                                   window->type_ == WindowType::kTGS ? RP_WINDOW_TGS : RP_WINDOW_NGS, trim_ ? 1 : 0);
    } else {
        s = rp_poa_add_window(poa_, static_cast<uint32_t>(n), seq.data(), len.data(), qual.data(), begin.data(),
                              end.data(), window->type_ == WindowType::kTGS ? RP_WINDOW_TGS : RP_WINDOW_NGS,
                              trim_ ? 1 : 0);
    }
    if (s == RP_BATCH_FULL) return false;
    if (s != RP_OK) {
        hard_error("[racon_b200::BatchProcessor::addWindow] error: " + status_text(s));
    }
    windows_.push_back(window);
    return true;
}

bool BatchProcessor::hasWindows() const { return rp_poa_size(poa_) > 0; }

const std::vector<bool>& BatchProcessor::generateConsensus() {
    launch();
    return collect();
}

void BatchProcessor::launch() {
    const rp_status s = rp_poa_run(poa_);
    if (s != RP_OK) {
        hard_error("[racon_b200::BatchProcessor::launch] error: " + status_text(s));
    }
}

const std::vector<bool>& BatchProcessor::collect() {
    const rp_status s = rp_poa_sync(poa_);
    if (s != RP_OK) {
        hard_error("[racon_b200::BatchProcessor::collect] error: " + status_text(s));
    }
    window_consensus_status_.clear();
    failed_.clear();
    for (uint32_t i = 0; i < windows_.size(); ++i) {
        const char* c = nullptr;
        uint32_t l = 0;
        int polished = 0;
        uint32_t st = 0;
        rp_poa_fetch(poa_, i, &c, &l, nullptr, &polished);
        rp_poa_window_status(poa_, i, &st);
        if (st != RP_WIN_OK) {
            /* a window that exceeded a device limit keeps its backbone (never silently re-run on the CPU) */
            fprintf(stderr, "[racon_b200::BatchProcessor] warning: window %lu exceeded device limit %u\n",
                    static_cast<unsigned long>(windows_[i]->id_), st);
            windows_[i]->consensus_ = std::string(windows_[i]->sequences_.front().first,
                                                  windows_[i]->sequences_.front().second);
            window_consensus_status_.push_back(false);
            failed_.push_back(i);
            continue;
        }
        windows_[i]->consensus_.assign(c, l);
        window_consensus_status_.push_back(polished != 0);
    }
    return window_consensus_status_;
}

bool BatchProcessor::ready() {
    const rp_status s = rp_poa_query(poa_);
    if (s == RP_NOT_READY) return false;
    if (s != RP_OK) {
        hard_error("[racon_b200::BatchProcessor::ready] error: " + status_text(s));
    }
    return true;
}

void BatchProcessor::reset() {
    windows_.clear();
    window_consensus_status_.clear();
    rp_poa_reset(poa_);
}

/* ---- BatchAligner ---- */
std::atomic<uint32_t> BatchAligner::batches{0};

std::unique_ptr<BatchAligner> createBatchAligner(uint32_t max_query_size, uint32_t max_target_size,
                                                 uint32_t max_alignments, uint32_t device_id) {
    return std::unique_ptr<BatchAligner>(new BatchAligner(max_query_size, max_target_size, max_alignments, device_id));
}

BatchAligner::BatchAligner(uint32_t max_query_size, uint32_t max_target_size, uint32_t max_alignments,
                           uint32_t device_id)
    : max_alignments_(max_alignments) {
    bid_ = batches++;
    rp_status s = rp_aln_create(&aln_, static_cast<int>(device_id), 0,
                                max_query_size > max_target_size ? max_query_size : max_target_size);
    if (s != RP_OK) {
        hard_error("[racon_b200::BatchAligner] error: " + status_text(s));
    }
}

BatchAligner::~BatchAligner() { rp_aln_destroy(aln_); }

bool BatchAligner::addOverlap(const char* q, uint32_t q_len, const char* t, uint32_t t_len, std::string* cigar) {
    if (max_alignments_ && cigars_.size() >= max_alignments_) return false;
    rp_status s = rp_aln_add(aln_, q, q_len, t, t_len);
    if (s == RP_BATCH_FULL) return false;
    if (s != RP_OK) {
        hard_error("[racon_b200::BatchAligner::addOverlap] error: " + status_text(s));
    }
    cigars_.push_back(cigar);
    return true;
}

void BatchAligner::alignAll() {
    rp_status s = rp_aln_run(aln_);
    if (s != RP_OK) {
        hard_error("[racon_b200::BatchAligner::alignAll] error: " + status_text(s));
    }
}

void BatchAligner::generate_cigar_strings() {
    rp_status s = rp_aln_sync(aln_);
    if (s != RP_OK) {
        hard_error("[racon_b200::BatchAligner::generate_cigar_strings] error: " + status_text(s));
    }
    for (uint32_t i = 0; i < cigars_.size(); ++i) {
        const char* c = nullptr;
        uint32_t l = 0, st = 0;
        rp_aln_fetch_cigar(aln_, i, &c, &l, nullptr, &st);
        if (cigars_[i]) cigars_[i]->assign(st == RP_ALN_OK ? c : "", st == RP_ALN_OK ? l : 0);
    }
}

void BatchAligner::reset() {
    cigars_.clear();
    rp_aln_reset(aln_);
}

std::string format_fasta(const std::string& target_name, const PolishedSequence& s) {
    std::string out;
    out.reserve(target_name.size() + s.tags.size() + s.data.size() + 3);
    out += '>';
    out += target_name;
    out += s.tags;
    out += '\n';
    out += s.data;
    out += '\n';
    return out;
}

/* ---- Polisher ---- */
namespace {

/* The scheduler of both device stages.  Lane l is idle or busy; fill(l) hands an idle lane the next piece of work and
 * launches it (false: nothing left), ready(l) tests a busy lane without blocking, drain(l) collects a finished one.  Every
 * idle lane is refilled before the next collect; the lane collected is one that has finished, else the oldest in flight
 * (waiting on it instead of polling in a loop). */
template <typename Fill, typename Ready, typename Drain>
void run_lanes(size_t n_lanes, Fill&& fill, Ready&& ready, Drain&& drain) {
    std::vector<uint8_t> busy(n_lanes, 0);
    std::deque<size_t> in_flight;   // busy lanes, oldest launch first
    while (true) {
        for (size_t l = 0; l < n_lanes; ++l) {
            if (!busy[l] && fill(l)) {
                busy[l] = 1;
                in_flight.push_back(l);
            }
        }
        if (in_flight.empty()) return;
        auto it = std::find_if(in_flight.begin(), in_flight.end(), [&](size_t l) { return ready(l); });
        if (it == in_flight.end()) it = in_flight.begin();
        const size_t l = *it;
        in_flight.erase(it);
        busy[l] = 0;
        drain(l);
    }
}

std::vector<uint64_t> every_index(size_t n) {
    std::vector<uint64_t> ids(n);
    std::iota(ids.begin(), ids.end(), 0);
    return ids;
}

/* Runs one device stage of the polisher: on a hard error anywhere inside, the stage's batch objects (its locals) are
 * destroyed while the error leaves it, then release() frees the read stores, then the process ends with the message. */
template <typename Stage, typename Release>
void run_stage(Stage&& stage, Release&& release) {
    ++hard_error_scopes;
    try {
        stage();
    } catch (const HardError& e) {
        --hard_error_scopes;
        release();
        fprintf(stderr, "%s\n", e.what());
        exit(1);
    }
    --hard_error_scopes;
}

}  // namespace

Polisher::Polisher(std::vector<SequenceView> sequences, uint64_t targets_size, WindowType window_type,
                   bool fragment_correction, uint32_t window_length, double quality_threshold, bool trim, int8_t match,
                   int8_t mismatch, int8_t gap, std::vector<uint32_t> devices)
    : sequences_(std::move(sequences)), targets_size_(targets_size), window_type_(window_type),
      fragment_correction_(fragment_correction), window_length_(window_length), quality_threshold_(quality_threshold),
      trim_(trim), match_(match), mismatch_(mismatch), gap_(gap), devices_(std::move(devices)),
      dummy_quality_(window_length, '!'),  // polisher.cpp:174
      reverse_complement_(sequences_.size()), reverse_quality_(sequences_.size()), targets_coverages_(targets_size, 0) {
    if (window_length == 0) {  // polisher.cpp:71-75
        fprintf(stderr, "[racon_b200::Polisher] error: invalid window length!\n");
        exit(1);
    }
    if (devices_.empty()) {
        fprintf(stderr, "[racon_b200::Polisher] error: empty device list!\n");
        exit(1);
    }
    /* without any device no index can be checked: the first device call then fails with "no CUDA device", as for one
     * index (SAM input builds its windows without a device) */
    const int count = rp_device_count();
    for (uint32_t d : devices_) {
        if (count > 0 && d >= static_cast<uint32_t>(count)) {
            fprintf(stderr, "[racon_b200::Polisher] error: device %u out of range (%d CUDA devices)!\n", d, count);
            exit(1);
        }
    }
}

Polisher::~Polisher() { release_read_stores(); }

void Polisher::release_read_stores() {
    for (auto& s : stores_) rp_reads_destroy(s.second);
    stores_.clear();
}

/* rp_reads is read-only once rp_reads_create has returned, so every batch object on `device` shares its one store */
const rp_reads* Polisher::read_store(uint32_t device, const std::vector<uint8_t>& members) {
    for (const auto& s : stores_)
        if (s.first == device) return s.second;
    std::vector<const char*> data(sequences_.size()), quality(sequences_.size());
    std::vector<uint32_t> length(sequences_.size());
    for (size_t i = 0; i < sequences_.size(); ++i) {
        if (!members.empty() && !members[i]) continue;   // absent: length 0, no bytes on the device
        data[i] = sequences_[i].data;
        quality[i] = sequences_[i].quality;
        length[i] = sequences_[i].length;
    }
    rp_reads* store = nullptr;
    const rp_status s = rp_reads_create(&store, static_cast<int>(device), static_cast<uint32_t>(data.size()),
                                        data.data(), quality.data(), length.data());
    if (s != RP_OK) hard_error("[racon_b200::Polisher] error: read store: " + status_text(s));
    stores_.emplace_back(device, store);
    return store;
}

const char* Polisher::reverse_complement(uint32_t id) {  // Sequence::create_reverse_complement, sequence.cpp:58-93
    std::string& r = reverse_complement_[id];
    if (r.empty() && sequences_[id].length) {
        const SequenceView& s = sequences_[id];
        r.resize(s.length);
        for (uint32_t i = 0; i < s.length; ++i) {
            char c = s.data[s.length - 1 - i];
            switch (c) {
                case 'A': c = 'T'; break;
                case 'C': c = 'G'; break;
                case 'G': c = 'C'; break;
                case 'T': c = 'A'; break;
                default: break;
            }
            r[i] = c;
        }
    }
    return r.data();
}

const char* Polisher::reverse_quality(uint32_t id) {
    std::string& r = reverse_quality_[id];
    const SequenceView& s = sequences_[id];
    if (r.empty() && s.quality && s.length) r.assign(std::reverse_iterator<const char*>(s.quality + s.length),
                                                     std::reverse_iterator<const char*>(s.quality));
    return s.quality ? r.data() : nullptr;
}

size_t Polisher::find_overlap_breaking_points(std::vector<Overlap>& overlaps) {
    return find_overlap_breaking_points(overlaps, every_index(overlaps.size()));
}

size_t Polisher::find_overlap_breaking_points(std::vector<Overlap>& overlaps, const std::vector<uint64_t>& ids) {
    /* an overlap that came with an alignment (SAM input) keeps it, as in Overlap::find_breaking_points
     * (overlap.cpp:186-203); only the others are aligned, in batches, on the device */
    std::vector<uint64_t> todo;
    todo.reserve(ids.size());
    uint32_t longest = 1;
    for (uint64_t k : ids) {
        Overlap& o = overlaps[k];
        if (!o.breaking_points_.empty()) continue;
        if (!o.cigar.empty()) {
            breaking_points_from_cigar(o, window_length_);
            std::string().swap(o.cigar);
        } else {
            todo.push_back(k);
            longest = std::max(longest, std::max(o.q_end - o.q_begin, o.t_end - o.t_begin));
        }
    }
    if (todo.empty()) return 0;
    run_stage([&] { align(overlaps, todo, longest); }, [&] { release_read_stores(); });
    std::sort(failed_overlaps_.begin(), failed_overlaps_.end());   // lanes finish in any order
    return todo.size();
}

void Polisher::align(std::vector<Overlap>& overlaps, const std::vector<uint64_t>& todo, uint32_t longest) {
    struct Lane {
        std::unique_ptr<rp_aln, void (*)(rp_aln*)> aln{nullptr, rp_aln_destroy};
        uint32_t device = 0;
        size_t first = 0, end = 0;   // the lane's batch: todo[first, end)
    };
    std::vector<Lane> lanes(devices_.size());
    /* a hard error on any lane ends the run like a single-device one (run_stage) */
    auto fail = [](const std::string& what) {
        hard_error("[racon_b200::Polisher::find_overlap_breaking_points] error: " + what);
    };
    for (size_t l = 0; l < lanes.size(); ++l) {
        lanes[l].device = devices_[l];
        rp_aln* aln = nullptr;
        rp_status s = rp_aln_create(&aln, static_cast<int>(devices_[l]), 0, longest);
        lanes[l].aln.reset(aln);
        if (s == RP_OK) s = rp_aln_set_window_length(aln, window_length_);
        if (s != RP_OK) fail(status_text(s));
    }
    size_t next = 0;   // the shared cursor over todo
    auto fill = [&](size_t l) {
        Lane& lane = lanes[l];
        if (next == todo.size()) return false;
        rp_aln* aln = lane.aln.get();
        lane.first = next;
        for (; next < todo.size(); ++next) {
            const Overlap& o = overlaps[todo[next]];
            /* the spans racon hands to the aligner (overlap.cpp:193-197) */
            const uint32_t q_start = o.strand ? o.q_length - o.q_end : o.q_begin;
            rp_status s;
            if (resident_reads_) {
                s = rp_aln_add_overlap_ref(aln, read_store(lane.device), o.q_id, q_start, o.q_end - o.q_begin,
                                           o.strand != 0, o.t_id, o.t_begin, o.t_end - o.t_begin);
            } else {
                const char* q = (o.strand ? reverse_complement(o.q_id) : sequences_[o.q_id].data) + q_start;
                const char* t = sequences_[o.t_id].data + o.t_begin;
                s = rp_aln_add_overlap(aln, q, o.q_end - o.q_begin, t, o.t_end - o.t_begin, o.t_begin, q_start);
            }
            if (s == RP_BATCH_FULL) break;
            if (s != RP_OK) fail(status_text(s));
        }
        if (next == lane.first) fail("overlap does not fit an empty batch");
        lane.end = next;
        const rp_status s = rp_aln_run(aln);   // asynchronous: the host goes on filling the other lanes
        if (s != RP_OK) fail(status_text(s));
        return true;
    };
    auto ready = [&](size_t l) {
        const rp_status s = rp_aln_query(lanes[l].aln.get());
        if (s != RP_OK && s != RP_NOT_READY) fail(status_text(s));
        return s == RP_OK;
    };
    auto drain = [&](size_t l) {
        Lane& lane = lanes[l];
        rp_aln* aln = lane.aln.get();
        rp_status s = rp_aln_sync(aln);
        if (s != RP_OK) fail(status_text(s));
        for (size_t j = lane.first; j < lane.end; ++j) {
            const size_t k = todo[j];
            const uint32_t* pts = nullptr;
            uint32_t n = 0, st = 0;
            rp_aln_fetch_cigar(aln, static_cast<uint32_t>(j - lane.first), nullptr, nullptr, nullptr, &st);
            if (st != RP_ALN_OK) {
                /* the reference re-aligns such overlaps with its CPU edlib (cudapolisher.cpp:213); this path has no CPU
                 * aligner, so the overlap contributes no layers and the caller is told */
                fprintf(stderr, "[racon_b200::Polisher] warning: overlap %zu exceeded device limit %u\n", k, st);
                failed_overlaps_.push_back(k);
                continue;
            }
            rp_aln_fetch_breaking_points(aln, static_cast<uint32_t>(j - lane.first), &pts, &n);
            overlaps[k].breaking_points_.clear();
            for (uint32_t b = 0; b < n; ++b) overlaps[k].breaking_points_.emplace_back(pts[2 * b], pts[2 * b + 1]);
        }
        s = rp_aln_reset(aln);
        if (s != RP_OK) fail(status_text(s));
    };
    run_lanes(lanes.size(), fill, ready, drain);
}

void Polisher::initialize(std::vector<Overlap>& overlaps) {
    find_overlap_breaking_points(overlaps);
    count_coverages(overlaps);
    build_windows(overlaps);
}

void Polisher::count_coverages(const std::vector<Overlap>& overlaps) {
    targets_coverages_.assign(targets_size_, 0);
    for (const Overlap& o : overlaps) ++targets_coverages_[o.t_id];
}

void Polisher::build_windows(const std::vector<Overlap>& overlaps) {
    build_windows(overlaps, every_index(overlaps.size()), 0, targets_size_, 0, ReadGroups::kAllWindows);
}

void Polisher::build_windows(const std::vector<Overlap>& overlaps, const std::vector<uint64_t>& ids,
                             uint64_t first_target, uint64_t end_target, uint32_t first_window, uint32_t end_window) {
    /* one window per window_length_ bases of every target (polisher.cpp:383-401) */
    std::vector<uint64_t> first_window_id(end_target - first_target);
    for (uint64_t i = first_target; i < end_target; ++i) {
        const SequenceView& tgt = sequences_[i];
        first_window_id[i - first_target] = windows_.size();
        for (uint64_t k = first_window; k < end_window && k * window_length_ < tgt.length; ++k) {
            const uint32_t j = static_cast<uint32_t>(k * window_length_);
            const uint32_t length = std::min(j + window_length_, tgt.length) - j;
            windows_.emplace_back(createWindow(i, static_cast<uint32_t>(k), window_type_, tgt.data + j, length,
                                               tgt.quality ? tgt.quality + j : dummy_quality_.data(), length));
            windows_.back()->set_backbone_origin(static_cast<uint32_t>(i), j);
        }
    }
    /* one layer per pair of breaking points (polisher.cpp:405-458) */
    for (uint64_t k : ids)
        add_layers(overlaps[k], first_window_id[overlaps[k].t_id - first_target], first_window, end_window);
}

void Polisher::add_layers(const Overlap& o, uint64_t first_window_id, uint32_t first_window, uint32_t end_window) {
    const SequenceView& sequence = sequences_[o.q_id];
    const auto& breaking_points = o.breaking_points();
    for (uint32_t j = 0; j + 1 < breaking_points.size(); j += 2) {
        const uint32_t window = breaking_points[j].first / window_length_;
        if (window < first_window || window >= end_window) continue;   // another part's window
        if (breaking_points[j + 1].second - breaking_points[j].second < 0.02 * window_length_) continue;

        const char* quality = o.strand ? reverse_quality(o.q_id) : sequence.quality;
        if (quality != nullptr) {
            double average_quality = 0;
            for (uint32_t k = breaking_points[j].second; k < breaking_points[j + 1].second; ++k) {
                average_quality += static_cast<uint32_t>(quality[k]) - 33;
            }
            average_quality /= breaking_points[j + 1].second - breaking_points[j].second;
            if (average_quality < quality_threshold_) continue;
        }

        const uint64_t window_id = first_window_id + (window - first_window);
        const uint32_t window_start = window * window_length_;
        const char* data = (o.strand ? reverse_complement(o.q_id) : sequence.data) + breaking_points[j].second;
        const uint32_t data_length = breaking_points[j + 1].second - breaking_points[j].second;
        const char* layer_quality = quality == nullptr ? nullptr : quality + breaking_points[j].second;
        const uint32_t quality_length = quality == nullptr ? 0 : data_length;

        windows_[window_id]->add_layer(data, data_length, layer_quality, quality_length,
                                       breaking_points[j].first - window_start,
                                       breaking_points[j + 1].first - window_start - 1,
                                       Window::Origin{o.q_id, breaking_points[j].second, o.strand != 0});
    }
}

void Polisher::polish(std::vector<PolishedSequence>& dst, bool drop_unpolished_sequences) {
    /* the windows are kept: their consensus stays readable (Polisher::windows) */
    Stitch stitch;
    consensus([&](const PolishedSequence& p) { dst.push_back(p); }, stitch, drop_unpolished_sequences, 0, false,
              resident_reads_, false);
}

void Polisher::polish_streaming(const std::function<void(const PolishedSequence&)>& sink,
                                bool drop_unpolished_sequences, size_t memory, bool banded, bool resident_reads) {
    Stitch stitch;
    consensus(sink, stitch, drop_unpolished_sequences, memory, banded, resident_reads || resident_reads_, true);
}

void Polisher::consensus(const std::function<void(const PolishedSequence&)>& sink, Stitch& stitch,
                         bool drop_unpolished_sequences, size_t memory, bool banded, bool resident_reads, bool release) {
    run_stage([&] { consensus_lanes(sink, stitch, drop_unpolished_sequences, memory, banded, resident_reads, release); },
              [&] { release_read_stores(); });
    std::sort(failed_windows_.begin(), failed_windows_.end());   // batches finish in any order
}

void Polisher::consensus_lanes(const std::function<void(const PolishedSequence&)>& sink, Stitch& stitch,
                               bool drop_unpolished_sequences, size_t memory, bool banded, bool resident_reads,
                               bool release) {
    constexpr size_t kObjectsPerLane = 2;   // one runs on the device while the host fills / collects the other
    struct Slot {
        std::unique_ptr<BatchProcessor> batch;
        size_t first = 0, count = 0;   // the object's batch: windows [first, first + count)
    };
    /* slot s runs on devices_[s % lanes]: the first round of batches goes to every lane before any gets a second */
    std::vector<Slot> slots(kObjectsPerLane * devices_.size());
    for (size_t i = 0; i < slots.size(); ++i) {
        const uint32_t device = devices_[i % devices_.size()];
        slots[i].batch = createBatch(0, device, memory, gap_, mismatch_, match_, banded, window_length_, trim_);
        /* resident reads: every sequence goes to the device once; the windows (whose pieces know their origin,
         * build_windows) are then added by reference and their layers extracted on the device */
        slots[i].batch->useReadStore(resident_reads ? read_store(device) : nullptr);
    }
    std::vector<uint8_t> polished(windows_.size(), 0);   // Window::generate_consensus' flag, until stitched
    std::string& polished_data = stitch.data;             // carried over when windows_ ends inside a target
    uint32_t& num_polished_windows = stitch.polished_windows;
    auto emit = [&](size_t w) {  // polisher.cpp:504-530, one window at a time, in window order
        num_polished_windows += polished[w];
        polished_data += windows_[w]->consensus();
        const uint64_t target_length = sequences_[windows_[w]->id()].length;
        /* the target's last window (racon: the last window of all, or one followed by a rank-0 window) */
        if ((static_cast<uint64_t>(windows_[w]->rank()) + 1) * window_length_ >= target_length) {
            const double polished_ratio = num_polished_windows / static_cast<double>(windows_[w]->rank() + 1);
            if (!drop_unpolished_sequences || polished_ratio > 0) {
                std::string tags = fragment_correction_ ? "r" : "";
                tags += " LN:i:" + std::to_string(polished_data.size());
                tags += " RC:i:" + std::to_string(targets_coverages_[windows_[w]->id()]);
                tags += " XC:f:" + std::to_string(polished_ratio);
                sink(PolishedSequence{windows_[w]->id(), tags, polished_data});
            }
            num_polished_windows = 0;
            polished_data.clear();
        }
        if (release) windows_[w].reset();  // polisher.cpp:531: the window is not needed any more
    };
    InOrderStitcher stitcher(windows_.size());
    size_t next = 0;   // the shared cursor over windows_
    auto fill = [&](size_t i) {
        Slot& slot = slots[i];
        if (next == windows_.size()) return false;
        slot.first = next;
        while (next < windows_.size() && slot.batch->addWindow(windows_[next])) ++next;
        slot.count = next - slot.first;
        if (slot.count == 0) {
            hard_error(std::string("[racon_b200::Polisher::") + (release ? "polish_streaming" : "polish") +
                       "] error: window does not fit an empty batch");
        }
        slot.batch->launch();  // asynchronous: the host goes on filling the other objects / stitching
        return true;
    };
    auto ready = [&](size_t i) { return slots[i].batch->ready(); };
    auto drain = [&](size_t i) {
        Slot& slot = slots[i];
        const std::vector<bool>& flags = slot.batch->collect();
        for (uint32_t k : slot.batch->failedWindows()) failed_windows_.push_back(slot.first + k);
        for (size_t k = 0; k < slot.count; ++k) polished[slot.first + k] = flags[k] ? 1 : 0;
        slot.batch->reset();   // drops the batch's references to its windows
        stitcher.finish(slot.first, slot.count, emit);
    };
    run_lanes(slots.size(), fill, ready, drain);
}

/* ---- target groups ---- */
uint64_t read_store_bytes(uint64_t sum_of_lengths, bool any_quality) {
    return (sum_of_lengths + 16) * (any_quality ? 2 : 1);
}

namespace {
std::string over_budget(const std::string& target_name, uint64_t bytes, uint64_t budget) {
    return "[racon_b200::Polisher] error: target " + target_name + " needs a read store of " + std::to_string(bytes) +
           " bytes, over the budget of " + std::to_string(budget) + " bytes per device!";
}
std::string window_over_budget(const std::string& target_name, uint32_t window, uint64_t bytes, uint64_t budget) {
    return "[racon_b200::Polisher] error: window " + std::to_string(window) + " of target " + target_name +
           " needs a read store of " + std::to_string(bytes) + " bytes, over the budget of " + std::to_string(budget) +
           " bytes per device!";
}
}  // namespace

TargetOverBudget::TargetOverBudget(uint64_t target, uint64_t bytes, uint64_t budget)
    : std::runtime_error(over_budget("#" + std::to_string(target), bytes, budget)), target(target), bytes(bytes),
      budget(budget) {}

std::string TargetOverBudget::message(const std::string& target_name) const {
    return over_budget(target_name, bytes, budget);
}

WindowOverBudget::WindowOverBudget(uint64_t target, uint32_t window, uint64_t bytes, uint64_t budget)
    : TargetOverBudget(window_over_budget("#" + std::to_string(target), window, bytes, budget), target, bytes, budget),
      window(window) {}

std::string WindowOverBudget::message(const std::string& target_name) const {
    return window_over_budget(target_name, window, bytes, budget);
}

namespace {
/* The store of the group being planned: the sequences in it (stamp_of_[i] == stamp_), their summed length and whether
 * any has a quality string. */
class OpenStore {
public:
    explicit OpenStore(const std::vector<SequenceView>& sequences)
        : sequences_(sequences), stamp_of_(sequences.size(), 0) {}
    void open() {   // a new, empty store
        ++stamp_;
        joining_.clear();
        sum_ = 0;
        quality_ = false;
    }
    /* the store's bytes if sequences `ids` joined it (a sequence in it already, or named twice, counts once) */
    uint64_t bytes_with(const std::vector<uint32_t>& ids) {
        for (uint32_t id : joining_) stamp_of_[id] = 0;   // offered last time and not committed
        joining_.clear();
        joined_sum_ = sum_;
        joined_quality_ = quality_;
        for (uint32_t id : ids) {
            if (stamp_of_[id] == stamp_) continue;
            stamp_of_[id] = stamp_;
            joining_.push_back(id);
            joined_sum_ += sequences_[id].length;
            joined_quality_ = joined_quality_ || (sequences_[id].quality != nullptr && sequences_[id].length > 0);
        }
        return read_store_bytes(joined_sum_, joined_quality_);
    }
    void commit() {   // the sequences of the last bytes_with join the store
        joining_.clear();
        sum_ = joined_sum_;
        quality_ = joined_quality_;
    }

private:
    const std::vector<SequenceView>& sequences_;
    std::vector<uint64_t> stamp_of_;
    std::vector<uint32_t> joining_;
    uint64_t stamp_ = 0, sum_ = 0, joined_sum_ = 0;
    bool quality_ = false, joined_quality_ = false;
};
}  // namespace

ReadGroups plan_read_groups(uint64_t targets_size, const std::vector<SequenceView>& sequences,
                            const std::vector<Overlap>& overlaps, uint64_t budget, uint32_t window_length) {
    /* the overlaps of every target, in their original order (stable counting sort by t_id) */
    std::vector<uint64_t> by_target_first(targets_size + 1, 0), by_target(overlaps.size());
    for (const Overlap& o : overlaps) ++by_target_first[o.t_id + 1];
    for (uint64_t t = 0; t < targets_size; ++t) by_target_first[t + 1] += by_target_first[t];
    {
        std::vector<uint64_t> at(by_target_first.begin(), by_target_first.end() - 1);
        for (uint64_t k = 0; k < overlaps.size(); ++k) by_target[at[overlaps[k].t_id]++] = k;
    }
    auto n_windows = [&](uint64_t t) {
        return (static_cast<uint64_t>(sequences[t].length) + window_length - 1) / window_length;
    };
    /* the windows [first, last] of its target that overlap o touches (all at 0 without a window length) */
    auto touched = [&](const Overlap& o) -> std::pair<uint64_t, uint64_t> {
        if (window_length == 0) return {0, 0};
        const uint64_t last_window = std::max<uint64_t>(n_windows(o.t_id), 1) - 1;
        const uint64_t first = std::min<uint64_t>(o.t_begin / window_length, last_window);
        const uint64_t last = o.t_end > o.t_begin ? std::min<uint64_t>((o.t_end - 1) / window_length, last_window) : 0;
        return {first, std::max(first, last)};
    };

    ReadGroups plan;
    std::vector<ReadGroups::Group>& groups = plan.groups;
    OpenStore store(sequences);
    std::vector<uint32_t> ids;   // the sequences a target, or a window, would add to the store
    bool open = false;           // the last group takes further targets
    for (uint64_t t = 0; t < targets_size; ++t) {
        ids.assign(1, static_cast<uint32_t>(t));
        for (uint64_t k = by_target_first[t]; k < by_target_first[t + 1]; ++k) ids.push_back(overlaps[by_target[k]].q_id);
        if (open) {
            const uint64_t bytes = store.bytes_with(ids);
            if (bytes <= budget) {
                store.commit();
                groups.back().end_target = t + 1;
                groups.back().bytes = bytes;
                continue;
            }
        }
        store.open();   // t starts a group of its own
        const uint64_t bytes = store.bytes_with(ids);
        open = bytes <= budget;
        if (open) {
            store.commit();
            groups.push_back({t, t + 1, 0, ReadGroups::kAllWindows, bytes});
            continue;
        }
        const uint64_t n = window_length > 0 ? n_windows(t) : 0;
        if (n == 0) throw TargetOverBudget(t, bytes, budget);

        /* t alone is over the budget: its windows are cut greedily into maximal parts [a, b), each a group of its own */
        std::vector<std::array<uint64_t, 3>> spans;   // (first window, last window, overlap) of t's overlaps
        for (uint64_t k = by_target_first[t]; k < by_target_first[t + 1]; ++k) {
            const auto w = touched(overlaps[by_target[k]]);
            spans.push_back({w.first, w.second, by_target[k]});
        }
        std::sort(spans.begin(), spans.end());
        std::vector<size_t> carry;   // the spans of the last part that reach past it
        size_t s = 0;                // spans[s..]: those that start in a window no part has yet
        for (uint64_t a = 0, b; a < n; a = b) {
            store.open();
            ids.assign(1, static_cast<uint32_t>(t));
            for (size_t i : carry) ids.push_back(overlaps[spans[i][2]].q_id);
            const size_t part_first = s;
            uint64_t part_bytes = 0;
            for (b = a; b < n; ++b) {   // window b joins while the store fits
                size_t e = s;
                for (; e < spans.size() && spans[e][0] == b; ++e) ids.push_back(overlaps[spans[e][2]].q_id);
                const uint64_t joined = store.bytes_with(ids);
                if (joined > budget) {
                    if (b == a) throw WindowOverBudget(t, static_cast<uint32_t>(a), joined, budget);
                    break;
                }
                store.commit();
                part_bytes = joined;
                s = e;
                ids.clear();
            }
            groups.push_back({t, t + 1, static_cast<uint32_t>(a), static_cast<uint32_t>(b), part_bytes});
            carry.erase(std::remove_if(carry.begin(), carry.end(), [&](size_t i) { return spans[i][1] < b; }),
                        carry.end());
            for (size_t i = part_first; i < s; ++i)
                if (spans[i][1] >= b) carry.push_back(i);
        }
    }

    /* The groups that hold overlap o, [first, end): those of its target whose windows it touches.  Groups come in
     * (target, window) order, so both are contiguous runs. */
    auto holders = [&](const Overlap& o) {
        const auto w = touched(o);
        using Group = ReadGroups::Group;
        auto first = std::partition_point(groups.begin(), groups.end(),
                                          [&](const Group& x) { return x.end_target <= o.t_id; });
        auto end = std::partition_point(first, groups.end(), [&](const Group& x) { return x.first_target <= o.t_id; });
        first = std::partition_point(first, end, [&](const Group& x) { return x.end_window <= w.first; });
        end = std::partition_point(first, end, [&](const Group& x) { return x.first_window <= w.second; });
        return std::make_pair(static_cast<uint64_t>(first - groups.begin()), static_cast<uint64_t>(end - groups.begin()));
    };
    /* every group's overlaps in file order (a stable counting sort by group), and the first group of each aligns it */
    plan.overlap_first.assign(groups.size() + 1, 0);
    plan.aligned_in.resize(overlaps.size());
    for (uint64_t k = 0; k < overlaps.size(); ++k) {
        const auto h = holders(overlaps[k]);
        plan.aligned_in[k] = h.first;
        for (uint64_t g = h.first; g < h.second; ++g) ++plan.overlap_first[g + 1];
    }
    for (size_t g = 0; g < groups.size(); ++g) plan.overlap_first[g + 1] += plan.overlap_first[g];
    plan.overlap_order.resize(plan.overlap_first.back());
    std::vector<uint64_t> at(plan.overlap_first.begin(), plan.overlap_first.end() - 1);
    for (uint64_t k = 0; k < overlaps.size(); ++k) {
        const auto h = holders(overlaps[k]);
        for (uint64_t g = h.first; g < h.second; ++g) plan.overlap_order[at[g]++] = k;
    }
    return plan;
}

void Polisher::polish_groups(std::vector<Overlap>& overlaps, const std::function<void(const PolishedSequence&)>& sink,
                             bool drop_unpolished_sequences, size_t memory, bool banded, uint64_t read_store_bytes,
                             bool split_targets) {
    std::vector<uint32_t> distinct;
    for (uint32_t d : devices_)
        if (std::find(distinct.begin(), distinct.end(), d) == distinct.end()) distinct.push_back(d);
    if (read_store_bytes == 0) {   // half of the smallest free memory, before any store or batch object exists
        uint64_t smallest = ~0ull;
        for (uint32_t d : distinct) {
            uint64_t free_b = 0, total_b = 0;
            const rp_status s = rp_device_memory(static_cast<int>(d), &free_b, &total_b);
            if (s != RP_OK) hard_error("[racon_b200::Polisher::polish_groups] error: " + status_text(s));
            smallest = std::min(smallest, free_b);
        }
        read_store_bytes = smallest / 2;
    }
    const ReadGroups plan =
        plan_read_groups(targets_size_, sequences_, overlaps, read_store_bytes, split_targets ? window_length_ : 0);

    resident_reads_ = true;
    group_store_bytes_.clear();
    group_windows_.clear();
    group_aligned_.clear();
    failed_overlaps_.clear();
    count_coverages(overlaps);
    std::vector<uint64_t> last_group(overlaps.size(), 0);   // the last group an overlap is in
    for (size_t g = 0; g < plan.size(); ++g)
        for (uint64_t k = plan.overlap_first[g]; k < plan.overlap_first[g + 1]; ++k) last_group[plan.overlap_order[k]] = g;
    Stitch stitch;
    std::vector<size_t> failed_windows;   // whole-run indices
    uint64_t windows_before = 0;          // windows of the groups before this one
    for (size_t g = 0; g < plan.size(); ++g) {
        const ReadGroups::Group& group = plan.groups[g];
        const std::vector<uint64_t> ids(plan.overlap_order.begin() + plan.overlap_first[g],
                                        plan.overlap_order.begin() + plan.overlap_first[g + 1]);

        /* the store first, on every distinct device: the batch objects then size themselves from what is left */
        std::vector<uint8_t> members(sequences_.size(), 0);
        std::fill(members.begin() + group.first_target, members.begin() + group.end_target, 1);
        for (uint64_t k : ids) members[overlaps[k].q_id] = 1;
        run_stage([&] {
            for (uint32_t d : distinct) read_store(d, members);
        }, [&] { release_read_stores(); });
        group_store_bytes_.push_back(rp_reads_bytes(stores_.front().second));

        /* the overlaps no earlier group holds (one the device refused, or one without a match in any window, has no
         * breaking points either, so they cannot tell) */
        std::vector<uint64_t> todo;
        for (uint64_t k : ids)
            if (plan.aligned_in[k] == g) todo.push_back(k);
        group_aligned_.push_back(find_overlap_breaking_points(overlaps, todo));

        windows_.clear();
        build_windows(overlaps, ids, group.first_target, group.end_target, group.first_window, group.end_window);
        failed_windows_.clear();
        consensus(sink, stitch, drop_unpolished_sequences, memory, banded, true, true);
        for (size_t w : failed_windows_) failed_windows.push_back(windows_before + w);
        group_windows_.emplace_back(windows_before, windows_before + windows_.size());
        windows_before += windows_.size();

        release_read_stores();
        for (uint64_t k : ids)
            if (last_group[k] == g) std::vector<std::pair<uint32_t, uint32_t>>().swap(overlaps[k].breaking_points_);
    }
    windows_.clear();
    failed_windows_ = std::move(failed_windows);   // groups in target and window order: already sorted
}

}  // namespace racon_b200

/* Test hooks with the shape of oracle/ref_polisher_harness.cpp (open -> counts -> export -> polish -> polished), so
 * that tests/test_pipeline.py compares this pipeline and the unmodified reference Polisher field by field. */
namespace {
struct PolHandle {
    std::unique_ptr<racon_b200::InputSet> input;   // owns the sequence bytes when the polisher was opened on files
    std::unique_ptr<racon_b200::Polisher> polisher;
    std::vector<racon_b200::PolishedSequence> polished;
    std::vector<racon_b200::Overlap> overlaps;     // with their breaking points, when opened on arrays
    const std::vector<racon_b200::Overlap>& all_overlaps() const { return input ? input->overlaps : overlaps; }
};
}  // namespace

extern "C" void* rp_mirror_polisher_open(uint32_t n_seq, const char* bases, const char* quals, const uint64_t* seq_off,
                                         const uint8_t* seq_has_qual, uint32_t n_targets, int window_type_tgs,
                                         int fragment_correction, uint32_t n_overlaps, const uint32_t* overlaps,
                                         uint32_t window_length, double quality_threshold, int trim, int8_t match,
                                         int8_t mismatch, int8_t gap, const uint32_t* devices, uint32_t n_devices) {
    using namespace racon_b200;
    std::vector<SequenceView> seqs(n_seq);
    for (uint32_t i = 0; i < n_seq; ++i) {
        seqs[i].data = bases + seq_off[i];
        seqs[i].quality = seq_has_qual[i] ? quals + seq_off[i] : nullptr;
        seqs[i].length = static_cast<uint32_t>(seq_off[i + 1] - seq_off[i]);
    }
    std::vector<Overlap> ovl(n_overlaps);
    for (uint32_t i = 0; i < n_overlaps; ++i) {
        const uint32_t* o = overlaps + 9ull * i;
        ovl[i] = Overlap{o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7], o[8], {}, {}};
    }
    PolHandle* h = new PolHandle();
    h->polisher.reset(new Polisher(std::move(seqs), n_targets, window_type_tgs ? WindowType::kTGS : WindowType::kNGS,
                                   fragment_correction != 0, window_length, quality_threshold, trim != 0, match,
                                   mismatch, gap, std::vector<uint32_t>(devices, devices + n_devices)));
    h->polisher->initialize(ovl);
    h->overlaps = std::move(ovl);
    return h;
}

/* Host logic only (no device call): the same, with the breaking points given (bp_off in points, bp = (t, q) pairs). */
extern "C" void* rp_mirror_polisher_open_with_bp(uint32_t n_seq, const char* bases, const char* quals,
                                                 const uint64_t* seq_off, const uint8_t* seq_has_qual,
                                                 uint32_t n_targets, int window_type_tgs, int fragment_correction,
                                                 uint32_t n_overlaps, const uint32_t* overlaps, const uint64_t* bp_off,
                                                 const uint32_t* bp, uint32_t window_length, double quality_threshold) {
    using namespace racon_b200;
    std::vector<SequenceView> seqs(n_seq);
    for (uint32_t i = 0; i < n_seq; ++i) {
        seqs[i].data = bases + seq_off[i];
        seqs[i].quality = seq_has_qual[i] ? quals + seq_off[i] : nullptr;
        seqs[i].length = static_cast<uint32_t>(seq_off[i + 1] - seq_off[i]);
    }
    std::vector<Overlap> ovl(n_overlaps);
    for (uint32_t i = 0; i < n_overlaps; ++i) {
        const uint32_t* o = overlaps + 9ull * i;
        ovl[i] = Overlap{o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7], o[8], {}, {}};
        for (uint64_t b = bp_off[i]; b < bp_off[i + 1]; ++b) ovl[i].breaking_points_.emplace_back(bp[2 * b], bp[2 * b + 1]);
    }
    PolHandle* h = new PolHandle();
    h->polisher.reset(new Polisher(std::move(seqs), n_targets, window_type_tgs ? WindowType::kTGS : WindowType::kNGS,
                                   fragment_correction != 0, window_length, quality_threshold, true, 3, -5, -4, {0}));
    h->polisher->build_windows(ovl);
    h->overlaps = std::move(ovl);
    return h;
}

/* Files in: createPolisher + initialize (polisher.cpp:55-160,200-461) — reads_io's load_input, then alignment and breaking
 * points on the device (overlaps that carry a CIGAR — SAM input — keep it and need no device) and the window building.
 * NULL on an input error (message in err).  rp_mirror_polisher_stream_fasta(names = NULL) then is racon's main loop. */
extern "C" void* rp_mirror_polisher_open_files(const char* reads, const char* overlaps, const char* targets,
                                               int fragment_correction, uint32_t window_length, double quality_threshold,
                                               double error_threshold, int trim, int8_t match, int8_t mismatch, int8_t gap,
                                               const uint32_t* devices, uint32_t n_devices, int resident_reads, char* err,
                                               uint32_t err_cap) {
    using namespace racon_b200;
    try {
        std::unique_ptr<PolHandle> h(new PolHandle());
        h->input.reset(new InputSet(load_input(reads, overlaps, targets, fragment_correction != 0, error_threshold)));
        h->polisher.reset(new Polisher(h->input->views(), h->input->targets_size, h->input->window_type,
                                       fragment_correction != 0, window_length, quality_threshold, trim != 0, match,
                                       mismatch, gap, std::vector<uint32_t>(devices, devices + n_devices)));
        h->polisher->use_resident_reads(resident_reads != 0);
        h->polisher->initialize(h->input->overlaps);
        return h.release();
    } catch (const std::exception& e) {
        if (err && err_cap) {
            std::strncpy(err, e.what(), err_cap - 1);
            err[err_cap - 1] = '\0';
        }
        return nullptr;
    }
}

/* The breaking points initialize() found: those of overlap i are the (t, q) pairs pts[2 off[i]] .. pts[2 off[i + 1]]
 * (off: one entry per overlap + 1).  Returns the number of points; off / pts NULL = count only. */
extern "C" uint64_t rp_mirror_polisher_breaking_points(void* hv, uint64_t* off, uint32_t* pts) {
    const auto& overlaps = static_cast<PolHandle*>(hv)->all_overlaps();
    uint64_t n = 0;
    for (size_t i = 0; i < overlaps.size(); ++i) {
        if (off) off[i] = n;
        for (const auto& p : overlaps[i].breaking_points()) {
            if (pts) {
                pts[2 * n] = p.first;
                pts[2 * n + 1] = p.second;
            }
            ++n;
        }
    }
    if (off) off[overlaps.size()] = n;
    return n;
}

/* failed[0] = overlaps, failed[1] = windows the device could not finish (Polisher::failed_overlaps/failed_windows) */
extern "C" void rp_mirror_polisher_failed(void* hv, uint64_t* failed) {
    PolHandle* h = static_cast<PolHandle*>(hv);
    failed[0] = h->polisher->failed_overlaps().size();
    failed[1] = h->polisher->failed_windows().size();
}

extern "C" void rp_mirror_polisher_counts(void* hv, uint64_t* counts) {
    PolHandle* h = static_cast<PolHandle*>(hv);
    counts[0] = h->polisher->windows().size();
    counts[1] = counts[2] = 0;
    for (const auto& w : h->polisher->windows()) {
        counts[1] += w->sequences().size();
        for (const auto& s : w->sequences()) counts[2] += s.second;
    }
}

extern "C" void rp_mirror_polisher_export(void* hv, char* bases, char* quals, uint64_t* seq_off, uint8_t* seq_has_qual,
                                          uint32_t* seq_begin, uint32_t* seq_end, uint32_t* win_first, uint8_t* win_type,
                                          uint64_t* win_target, uint32_t* win_rank) {
    PolHandle* h = static_cast<PolHandle*>(hv);
    uint64_t nb = 0, ns = 0;
    seq_off[0] = 0;
    const auto& windows = h->polisher->windows();
    for (size_t w = 0; w < windows.size(); ++w) {
        const auto& win = windows[w];
        win_first[w] = static_cast<uint32_t>(ns);
        win_type[w] = win->type() == racon_b200::WindowType::kTGS ? 1 : 0;
        win_target[w] = win->id();
        win_rank[w] = win->rank();
        for (size_t s = 0; s < win->sequences().size(); ++s) {
            const uint32_t len = win->sequences()[s].second;
            std::memcpy(bases + nb, win->sequences()[s].first, len);
            const char* q = win->qualities()[s].first;
            if (q) {
                std::memcpy(quals + nb, q, len);
                seq_has_qual[ns] = 1;
            } else {
                std::memset(quals + nb, '!', len);
                seq_has_qual[ns] = 0;
            }
            seq_begin[ns] = win->positions()[s].first;
            seq_end[ns] = win->positions()[s].second;
            nb += len;
            seq_off[++ns] = nb;
        }
    }
    win_first[windows.size()] = static_cast<uint32_t>(ns);
}

extern "C" uint32_t rp_mirror_polisher_polish(void* hv, int drop_unpolished) {
    PolHandle* h = static_cast<PolHandle*>(hv);
    h->polisher->polish(h->polished, drop_unpolished != 0);
    return static_cast<uint32_t>(h->polished.size());
}

extern "C" uint32_t rp_mirror_polisher_window_consensus(void* hv, uint32_t w, char* out, uint32_t cap) {
    PolHandle* h = static_cast<PolHandle*>(hv);
    const std::string& c = h->polisher->windows()[w]->consensus();
    if (c.size() > cap) return 0xffffffffu;
    std::memcpy(out, c.data(), c.size());
    return static_cast<uint32_t>(c.size());
}

extern "C" uint64_t rp_mirror_polisher_polished(void* hv, uint32_t i, uint64_t* target_id, char* tags, uint32_t tags_cap,
                                                char* data, uint64_t data_cap) {
    PolHandle* h = static_cast<PolHandle*>(hv);
    const auto& s = h->polished[i];
    *target_id = s.id;
    std::strncpy(tags, s.tags.c_str(), tags_cap - 1);
    tags[tags_cap - 1] = 0;
    if (s.data.size() > data_cap) return ~0ull;
    std::memcpy(data, s.data.data(), s.data.size());
    return s.data.size();
}

/* Streaming polish straight into a FASTA file (names: NUL-separated target names, one per target id; NULL = the names
 * of the files the polisher was opened on); returns the
 * number of records written.  mem_bytes: budget per batch object (small budgets force many batches). */
extern "C" uint32_t rp_mirror_polisher_stream_fasta(void* hv, int drop_unpolished, const char* path, const char* names,
                                                     uint64_t mem_bytes, int banded, int resident_reads) {
    PolHandle* h = static_cast<PolHandle*>(hv);
    std::vector<std::string> name_of;
    for (const char* p = names; p && *p; p += std::strlen(p) + 1) name_of.emplace_back(p);
    if (!names && h->input) {
        for (uint64_t i = 0; i < h->input->targets_size; ++i) name_of.push_back(h->input->sequences[i].name);
    }
    FILE* f = std::fopen(path, "wb");
    if (!f) return 0;
    uint32_t n = 0;
    h->polisher->polish_streaming(
        [&](const racon_b200::PolishedSequence& s) {
            const std::string rec = racon_b200::format_fasta(s.id < name_of.size() ? name_of[s.id] : "?", s);
            std::fwrite(rec.data(), 1, rec.size(), f);
            ++n;
        },
        drop_unpolished != 0, static_cast<size_t>(mem_bytes), banded != 0, resident_reads != 0);
    std::fclose(f);
    return n;
}

extern "C" void rp_mirror_polisher_close(void* hv) { delete static_cast<PolHandle*>(hv); }

namespace {
/* the last rp_mirror_polish_files_grouped (rp_mirror_last_grouped_run) */
std::vector<uint64_t> g_last_group_store_bytes, g_last_failed_overlaps, g_last_failed_windows;
std::vector<uint64_t> g_last_group_windows, g_last_group_aligned;
}  // namespace

/* racon's whole run on files in target groups (Polisher::polish_groups): load_input, plan, polish, FASTA into `path`.
 * read_store_bytes: budget per device (0 = automatic); split_targets: polish a target over it in parts.  result[0] =
 * records written, [1] overlaps and [2] windows the device refused.  Returns 0, or -1 with the message in err (input
 * error, a target or window over the budget, unwritable path). */
extern "C" int rp_mirror_polish_files_grouped(const char* reads, const char* overlaps, const char* targets,
                                              int fragment_correction, uint32_t window_length, double quality_threshold,
                                              double error_threshold, int trim, int8_t match, int8_t mismatch, int8_t gap,
                                              const uint32_t* devices, uint32_t n_devices, int drop_unpolished,
                                              uint64_t mem_bytes, int banded, uint64_t read_store_bytes,
                                              int split_targets, const char* path, uint64_t* result, char* err,
                                              uint32_t err_cap) {
    using namespace racon_b200;
    auto error = [&](const std::string& what) {
        if (err && err_cap) {
            std::strncpy(err, what.c_str(), err_cap - 1);
            err[err_cap - 1] = '\0';
        }
        return -1;
    };
    InputSet input;
    try {
        input = load_input(reads, overlaps, targets, fragment_correction != 0, error_threshold);
    } catch (const std::exception& e) {
        return error(e.what());
    }
    Polisher polisher(input.views(), input.targets_size, input.window_type, fragment_correction != 0, window_length,
                      quality_threshold, trim != 0, match, mismatch, gap,
                      std::vector<uint32_t>(devices, devices + n_devices));
    FILE* f = std::fopen(path, "wb");
    if (!f) return error(std::string("cannot write ") + path);
    uint64_t n = 0;
    try {
        polisher.polish_groups(input.overlaps,
                               [&](const PolishedSequence& s) {
                                   const std::string rec = format_fasta(input.sequences[s.id].name, s);
                                   std::fwrite(rec.data(), 1, rec.size(), f);
                                   ++n;
                               },
                               drop_unpolished != 0, static_cast<size_t>(mem_bytes), banded != 0, read_store_bytes,
                               split_targets != 0);
    } catch (const TargetOverBudget& e) {   // planned before any record: no output (WindowOverBudget too)
        std::fclose(f);
        std::remove(path);
        return error(e.message(input.sequences[e.target].name));
    }
    std::fclose(f);
    g_last_group_store_bytes = polisher.group_store_bytes();
    g_last_group_windows.clear();
    for (const auto& w : polisher.group_windows()) {
        g_last_group_windows.push_back(w.first);
        g_last_group_windows.push_back(w.second);
    }
    g_last_group_aligned = polisher.group_aligned();
    g_last_failed_overlaps.assign(polisher.failed_overlaps().begin(), polisher.failed_overlaps().end());
    g_last_failed_windows.assign(polisher.failed_windows().begin(), polisher.failed_windows().end());
    result[0] = n;
    result[1] = polisher.failed_overlaps().size();
    result[2] = polisher.failed_windows().size();
    return 0;
}

/* The last rp_mirror_polish_files_grouped: counts[0] groups, [1] failed overlaps, [2] failed windows; then (any pointer
 * may be NULL) rp_reads_bytes of every group's store and the whole-run indices of the failed overlaps and windows. */
extern "C" void rp_mirror_last_grouped_run(uint64_t* counts, uint64_t* group_bytes, uint64_t* failed_overlaps,
                                           uint64_t* failed_windows) {
    counts[0] = g_last_group_store_bytes.size();
    counts[1] = g_last_failed_overlaps.size();
    counts[2] = g_last_failed_windows.size();
    if (group_bytes) std::copy(g_last_group_store_bytes.begin(), g_last_group_store_bytes.end(), group_bytes);
    if (failed_overlaps) std::copy(g_last_failed_overlaps.begin(), g_last_failed_overlaps.end(), failed_overlaps);
    if (failed_windows) std::copy(g_last_failed_windows.begin(), g_last_failed_windows.end(), failed_windows);
}

/* The same run, per group (counts[0] of rp_mirror_last_grouped_run of them): its whole-run windows
 * [group_windows[2 g], group_windows[2 g + 1]) and the number of overlaps it sent to the aligner. */
extern "C" void rp_mirror_last_grouped_run_windows(uint64_t* group_windows, uint64_t* group_aligned) {
    std::copy(g_last_group_windows.begin(), g_last_group_windows.end(), group_windows);
    std::copy(g_last_group_aligned.begin(), g_last_group_aligned.end(), group_aligned);
}

/* Host-only hook of plan_read_groups: n_seq sequences (the first n_targets are the targets) of length[i], with a quality
 * string when has_quality[i]; overlap k runs from sequence q_id[k] onto target t_id[k], over its target span
 * [t_begin[k], t_end[k]).  window_length = 0 does not split targets, and t_begin / t_end may then be NULL.
 * sizes[0] = groups, sizes[1] = entries of overlap_order (an overlap is in every part it touches); with every output
 * NULL only sizes is written.  Outputs: group g = targets [first_target[g], first_target[g + 1]) (first_target has
 * sizes[0] + 1 entries; a part's next entry is its own target until its target's last part), predicted store bytes[g],
 * its overlaps overlap_order[overlap_first[g] .. overlap_first[g + 1]), its windows [first_window[g], end_window[g])
 * when it is a part (0, 0 for whole targets), and per overlap the group that aligns it.  Returns the number of groups,
 * or -1 with the error in err (a target, or with a window length a window, over the budget). */
extern "C" int64_t rp_mirror_plan_read_groups(uint64_t n_targets, uint32_t n_seq, const uint32_t* length,
                                              const uint8_t* has_quality, uint64_t n_overlaps, const uint32_t* q_id,
                                              const uint32_t* t_id, const uint32_t* t_begin, const uint32_t* t_end,
                                              uint32_t window_length, uint64_t budget, uint64_t* sizes,
                                              uint64_t* first_target, uint64_t* bytes, uint64_t* overlap_first,
                                              uint64_t* overlap_order, uint32_t* first_window, uint32_t* end_window,
                                              uint64_t* aligned_in, char* err, uint32_t err_cap) {
    using namespace racon_b200;
    static const char kQuality[] = "";   // stands for "has a quality string": the planner only tests for null
    std::vector<SequenceView> seqs(n_seq);
    for (uint32_t i = 0; i < n_seq; ++i) seqs[i] = SequenceView{nullptr, has_quality[i] ? kQuality : nullptr, length[i]};
    std::vector<Overlap> ovl(n_overlaps);
    for (uint64_t k = 0; k < n_overlaps; ++k) {
        ovl[k].q_id = q_id[k];
        ovl[k].t_id = t_id[k];
        ovl[k].t_begin = window_length ? t_begin[k] : 0;
        ovl[k].t_end = window_length ? t_end[k] : 0;
    }
    try {
        const ReadGroups plan = plan_read_groups(n_targets, seqs, ovl, budget, window_length);
        sizes[0] = plan.size();
        sizes[1] = plan.overlap_order.size();
        if (first_target) {
            for (size_t g = 0; g < plan.size(); ++g) {
                const ReadGroups::Group& group = plan.groups[g];
                first_target[g] = group.first_target;
                bytes[g] = group.bytes;
                first_window[g] = group.first_window;
                end_window[g] = group.end_window == ReadGroups::kAllWindows ? 0 : group.end_window;
            }
            first_target[plan.size()] = n_targets;
            std::copy(plan.overlap_first.begin(), plan.overlap_first.end(), overlap_first);
            std::copy(plan.overlap_order.begin(), plan.overlap_order.end(), overlap_order);
            std::copy(plan.aligned_in.begin(), plan.aligned_in.end(), aligned_in);
        }
        return static_cast<int64_t>(plan.size());
    } catch (const std::exception& e) {
        if (err && err_cap) {
            std::strncpy(err, e.what(), err_cap - 1);
            err[err_cap - 1] = '\0';
        }
        return -1;
    }
}

/* Host-only test hook of the stitch cursor (InOrderStitcher): n_ranges contiguous ranges of counts[r] windows finish in
 * the order `completion` (a permutation of 0 .. n_ranges - 1).  order[i] = the i-th window emitted, step[i] = the position
 * in `completion` of the range whose finish emitted it.  Returns the number of windows emitted. */
extern "C" uint64_t rp_mirror_stitch_order(uint32_t n_ranges, const uint32_t* counts, const uint32_t* completion,
                                           uint64_t* order, uint32_t* step) {
    std::vector<uint64_t> first(n_ranges + 1, 0);
    for (uint32_t r = 0; r < n_ranges; ++r) first[r + 1] = first[r] + counts[r];
    racon_b200::InOrderStitcher stitcher(first[n_ranges]);
    uint64_t n = 0;
    for (uint32_t i = 0; i < n_ranges; ++i) {
        const uint32_t r = completion[i];
        stitcher.finish(first[r], counts[r], [&](size_t w) {
            order[n] = w;
            step[n++] = i;
        });
    }
    return n;
}

/* host-only: one FASTA record; returns its length (out may be NULL to size it) */
extern "C" uint64_t rp_mirror_format_fasta(const char* name, const char* tags, const char* data, uint64_t data_len,
                                           char* out, uint64_t cap) {
    racon_b200::PolishedSequence s{0, tags, std::string(data, data_len)};
    const std::string r = racon_b200::format_fasta(name, s);
    if (out && r.size() <= cap) std::memcpy(out, r.data(), r.size());
    return r.size();
}

/* Test hook: CUDAPolisher::find_overlap_breaking_points' batch loop (cudapolisher.cpp:100-213) over flat pairs:
 * fill a batch until addOverlap refuses, alignAll, generate_cigar_strings, reset, continue.  out: NUL-terminated
 * CIGARs at out + i * stride (empty when the device could not take the overlap). */
extern "C" int rp_mirror_align(uint32_t n_pairs, const char* bases, const uint64_t* q_off, const uint32_t* q_len,
                               const uint64_t* t_off, const uint32_t* t_len, uint32_t max_alignments, uint32_t device,
                               char* out, uint32_t stride) {
    using namespace racon_b200;
    uint32_t mq = 1, mt = 1;
    for (uint32_t i = 0; i < n_pairs; ++i) {
        if (q_len[i] > mq) mq = q_len[i];
        if (t_len[i] > mt) mt = t_len[i];
    }
    auto batch = createBatchAligner(mq, mt, max_alignments, device);
    std::vector<std::string> cigars(n_pairs);
    uint32_t i = 0;
    while (i < n_pairs) {
        uint32_t first = i;
        while (i < n_pairs && batch->addOverlap(bases + q_off[i], q_len[i], bases + t_off[i], t_len[i], &cigars[i])) ++i;
        if (i == first) return -1;
        batch->alignAll();
        batch->generate_cigar_strings();
        batch->reset();
    }
    for (uint32_t k = 0; k < n_pairs; ++k) {
        if (cigars[k].size() + 1 > stride) return -2;
        std::memcpy(out + static_cast<uint64_t>(k) * stride, cigars[k].c_str(), cigars[k].size() + 1);
    }
    return 0;
}

/* Test hook: drives the mirror classes exactly like CUDAPolisher::polish drives CUDABatchProcessor
 * (cudapolisher.cpp:254-276), over a flat window set. Same contract as oracle/ref_harness.cpp. */
extern "C" double rp_mirror_consensus(uint32_t n_windows, const char* bases, const char* quals,
                                      const uint64_t* seq_off, const uint8_t* seq_has_qual, const uint32_t* seq_begin,
                                      const uint32_t* seq_end, const uint32_t* win_first, const uint8_t* win_type,
                                      int8_t match, int8_t mismatch, int8_t gap, uint32_t window_length, int trim,
                                      uint32_t device, char* out, uint32_t out_stride, uint32_t* out_len,
                                      uint8_t* polished) {
    using namespace racon_b200;
    uint32_t max_bl = 1;
    for (uint32_t w = 0; w < n_windows; ++w) {
        uint32_t s0 = win_first[w];
        uint32_t bl = static_cast<uint32_t>(seq_off[s0 + 1] - seq_off[s0]);
        if (bl > max_bl) max_bl = bl;
    }
    std::string dummy(max_bl, '!');
    std::vector<std::shared_ptr<Window>> windows;
    for (uint32_t w = 0; w < n_windows; ++w) {
        uint32_t s0 = win_first[w], s1 = win_first[w + 1];
        uint64_t o = seq_off[s0];
        uint32_t bl = static_cast<uint32_t>(seq_off[s0 + 1] - o);
        bool bq = quals && seq_has_qual && seq_has_qual[s0];
        auto win = createWindow(w, w, win_type[w] ? WindowType::kTGS : WindowType::kNGS, bases + o, bl,
                                bq ? quals + o : dummy.data(), bl);
        for (uint32_t s = s0 + 1; s < s1; ++s) {
            uint64_t so = seq_off[s];
            uint32_t sl = static_cast<uint32_t>(seq_off[s + 1] - so);
            bool q = quals && seq_has_qual && seq_has_qual[s];
            win->add_layer(bases + so, sl, q ? quals + so : nullptr, q ? sl : 0, seq_begin[s], seq_end[s]);
        }
        windows.push_back(win);
    }
    auto batch = createBatch(0, device, 0, gap, mismatch, match, false, window_length, trim != 0);
    std::vector<uint8_t> flags(n_windows, 0);
    uint32_t next = 0;
    while (next < n_windows) {
        uint32_t first = next;
        batch->reset();
        while (next < n_windows && batch->addWindow(windows[next])) ++next;
        if (next == first) return -1.0;  // a single window does not fit
        const std::vector<bool>& st = batch->generateConsensus();
        for (uint32_t k = 0; k < st.size(); ++k) flags[first + k] = st[k] ? 1 : 0;
    }
    for (uint32_t w = 0; w < n_windows; ++w) {
        const std::string& c = windows[w]->consensus();
        if (c.size() > out_stride) return -2.0;
        std::memcpy(out + static_cast<uint64_t>(w) * out_stride, c.data(), c.size());
        out_len[w] = static_cast<uint32_t>(c.size());
        polished[w] = flags[w];
    }
    return 0.0;
}
