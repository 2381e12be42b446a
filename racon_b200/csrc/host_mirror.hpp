/*
 * host_mirror.hpp — C++ host-side mirror of the reference's interface for the POA hot path, written
 * over the C ABI (include/racon_b200.h).  Same names, argument meaning and error behaviour as
 *   racon::Window / createWindow / Window::add_layer        (/root/reference/src/window.hpp:25-74, window.cpp:15-63)
 *   racon::CUDABatchProcessor / createCUDABatch             (/root/reference/src/cuda/cudabatch.hpp:27-122)
 * so that racon's CUDAPolisher (src/cuda/cudapolisher.cpp:216-413) can drive it unchanged.
 */
#pragma once
#include <stdint.h>

#include <atomic>
#include <functional>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

struct rp_poa;
struct rp_aln;
struct rp_reads;

namespace racon_b200 {

enum class WindowType { kNGS, kTGS };  // src/window.hpp:20-23

class Window;
std::shared_ptr<Window> createWindow(uint64_t id, uint32_t rank, WindowType type, const char* backbone,
                                     uint32_t backbone_length, const char* quality, uint32_t quality_length);

class Window {
public:
    ~Window();
    uint64_t id() const { return id_; }
    uint32_t rank() const { return rank_; }
    const std::string& consensus() const { return consensus_; }
    WindowType type() const { return type_; }
    const std::vector<std::pair<const char*, uint32_t>>& sequences() const { return sequences_; }
    const std::vector<std::pair<const char*, uint32_t>>& qualities() const { return qualities_; }
    const std::vector<std::pair<uint32_t, uint32_t>>& positions() const { return positions_; }

    /* same checks, same silent skips and the same fatal errors as the reference (window.cpp:42-63) */
    void add_layer(const char* sequence, uint32_t sequence_length, const char* quality, uint32_t quality_length,
                   uint32_t begin, uint32_t end);

    /* Where a piece comes from: sequence `seq_id` of the caller's sequence table from `offset` on — of its reverse
     * complement when `reverse`.  A window whose backbone and every layer carry their origin can be handed to a batch by
     * reference into a device-resident read store (BatchProcessor::useReadStore) instead of by its bytes. */
    struct Origin {
        uint32_t seq_id, offset;
        bool reverse;
    };
    void set_backbone_origin(uint32_t seq_id, uint32_t offset) { origins_.assign(1, Origin{seq_id, offset, false}); }
    /* add_layer + the layer's origin (the origin is dropped with the layer when add_layer skips it) */
    void add_layer(const char* sequence, uint32_t sequence_length, const char* quality, uint32_t quality_length,
                   uint32_t begin, uint32_t end, const Origin& origin);
    const std::vector<Origin>& origins() const { return origins_; }

    friend std::shared_ptr<Window> createWindow(uint64_t id, uint32_t rank, WindowType type, const char* backbone,
                                                uint32_t backbone_length, const char* quality,
                                                uint32_t quality_length);
    friend class BatchProcessor;

private:
    Window(uint64_t id, uint32_t rank, WindowType type, const char* backbone, uint32_t backbone_length,
           const char* quality, uint32_t quality_length);
    Window(const Window&) = delete;
    const Window& operator=(const Window&) = delete;

    uint64_t id_;
    uint32_t rank_;
    WindowType type_;
    std::string consensus_;
    std::vector<std::pair<const char*, uint32_t>> sequences_;
    std::vector<std::pair<const char*, uint32_t>> qualities_;
    std::vector<std::pair<uint32_t, uint32_t>> positions_;
    std::vector<Origin> origins_;   // empty, or one per entry of sequences_
};

class BatchProcessor;
/* createCUDABatch (cudabatch.cpp:23-39) + the two things the reference fixes elsewhere: window length
 * (Polisher ctor) and the trim flag (Window::generate_consensus argument). */
std::unique_ptr<BatchProcessor> createBatch(uint32_t max_window_depth, uint32_t device, size_t avail_mem, int8_t gap,
                                            int8_t mismatch, int8_t match, bool cuda_banded_alignment,
                                            uint32_t window_length = 500, bool trim = true);

class BatchProcessor {
public:
    ~BatchProcessor();
    /* false = batch full: run generateConsensus(), reset(), add the window again (cudabatch.cpp:126-132) */
    bool addWindow(std::shared_ptr<Window> window);
    bool hasWindows() const;
    /* writes window->consensus_ for every accepted window; flag = what Window::generate_consensus returns */
    const std::vector<bool>& generateConsensus();
    /* the two halves of generateConsensus (generatePOA / getConsensus of the reference, cudabatch.cpp:193-270):
     * launch() queues H2D + kernel + D2H on the object's stream and returns, collect() waits and reads back */
    void launch();
    const std::vector<bool>& collect();
    /* true when the launched batch has finished on the device (rp_poa_query): collect() then does not wait for the
     * kernel */
    bool ready();
    void reset();
    uint32_t getBatchID() const { return bid_; }
    /* From now on windows that know the origin of all their pieces (Window::origins) are added by reference into
     * `reads` (rp_reads_create over the same sequence table, same device): no sequence byte is copied on the host, the
     * layers are extracted on the device.  nullptr switches back.  Call between batches (after reset()). */
    void useReadStore(const rp_reads* reads) { reads_ = reads; }
    /* indices (within the batch) of the windows of the last generateConsensus() that hit a device limit (soft RP_WIN_*
     * status): their flag is false and their consensus is the backbone — not what racon would produce; the reference's
     * caller re-runs such windows on the CPU (cudapolisher.cpp:354-370), a caller without a CPU path must treat them as
     * an error */
    const std::vector<uint32_t>& failedWindows() const { return failed_; }

    friend std::unique_ptr<BatchProcessor> createBatch(uint32_t, uint32_t, size_t, int8_t, int8_t, int8_t, bool,
                                                       uint32_t, bool);

private:
    BatchProcessor(uint32_t max_window_depth, uint32_t device, size_t avail_mem, int8_t gap, int8_t mismatch,
                   int8_t match, bool cuda_banded_alignment, uint32_t window_length, bool trim);
    BatchProcessor(const BatchProcessor&) = delete;
    const BatchProcessor& operator=(const BatchProcessor&) = delete;

    static std::atomic<uint32_t> batches;
    uint32_t bid_ = 0;
    rp_poa* poa_ = nullptr;
    const rp_reads* reads_ = nullptr;
    bool trim_ = true;
    std::vector<std::shared_ptr<Window>> windows_;
    std::vector<bool> window_consensus_status_;
    std::vector<uint32_t> failed_;
};

/* Mirror of racon::CUDABatchAligner (src/cuda/cudaaligner.hpp:21-92).  The reference's addOverlap takes an
 * Overlap* plus the sequence table and derives the two spans (cudaaligner.cpp:53-58); the mirror takes the spans and a
 * pointer to the std::string that plays Overlap::cigar_. */
class BatchAligner;
std::unique_ptr<BatchAligner> createBatchAligner(uint32_t max_query_size, uint32_t max_target_size,
                                                 uint32_t max_alignments, uint32_t device_id);

class BatchAligner {
public:
    ~BatchAligner();
    /* false = batch full (exceeded_max_alignments / exceeded_max_length are soft: an over-long overlap is
     * accepted and simply keeps an empty cigar, as in cudaaligner.cpp:61-77) */
    bool addOverlap(const char* q, uint32_t q_len, const char* t, uint32_t t_len, std::string* cigar);
    bool hasOverlaps() const { return !cigars_.empty(); }
    void alignAll();                  // asynchronous launch (cudaaligner.cpp:80-84)
    void generate_cigar_strings();    // sync + fill every *cigar (cudaaligner.cpp:86-104)
    void reset();
    uint32_t getBatchID() const { return bid_; }

    friend std::unique_ptr<BatchAligner> createBatchAligner(uint32_t, uint32_t, uint32_t, uint32_t);

private:
    BatchAligner(uint32_t max_query_size, uint32_t max_target_size, uint32_t max_alignments, uint32_t device_id);
    BatchAligner(const BatchAligner&) = delete;
    const BatchAligner& operator=(const BatchAligner&) = delete;

    static std::atomic<uint32_t> batches;
    uint32_t bid_ = 0;
    uint32_t max_alignments_ = 0;
    rp_aln* aln_ = nullptr;
    std::vector<std::string*> cigars_;
};

/* ------------------------------------------------------------------------------------------------------------------
 * Mirror of the device-facing half of racon::CUDAPolisher: overlaps -> (device) alignment + breaking points ->
 * windows -> (device) consensus -> stitched sequences.  Parsing and overlap filtering are reads_io.hpp's (load_input);
 * everything that touches sequence bytes in bulk runs on the GPU.
 *   find_overlap_breaking_points : src/cuda/cudapolisher.cpp:72-213  (batched aligner loop)
 *                                  + src/overlap.cpp:226-292          (breaking points, on the device here)
 *   initialize (window building) : src/polisher.cpp:383-461
 *   polish                       : src/cuda/cudapolisher.cpp:215-395 (batch loop), src/polisher.cpp:504-537 (stitch)
 * ------------------------------------------------------------------------------------------------------------------ */
struct SequenceView {        // racon::Sequence as the polisher needs it; the bytes stay owned by the caller
    const char* data;
    const char* quality;     // nullptr when the sequence has no quality string
    uint32_t length;
};

struct Overlap {             // racon::Overlap after transmute() (src/overlap.hpp:82-98)
    uint32_t q_id, t_id, strand, q_begin, q_end, q_length, t_begin, t_end, t_length;
    std::string cigar;       // only when the overlap file carried an alignment (SAM): then it is used as it is
    std::vector<std::pair<uint32_t, uint32_t>> breaking_points_;
    const std::vector<std::pair<uint32_t, uint32_t>>& breaking_points() const { return breaking_points_; }
};

/* Breaking points of an overlap that arrived WITH an alignment (SAM): the (target, query) coordinates of the first and
 * one-past-the-last aligned base pair inside every window of the target the alignment crosses — what
 * Overlap::find_breaking_points_from_cigar (overlap.cpp:226-292) finds base by base, computed run by run here.
 * (Overlaps without a CIGAR get theirs from the device: rp_aln_fetch_breaking_points.) */
void breaking_points_from_cigar(Overlap& overlap, uint32_t window_length);

struct PolishedSequence {
    uint64_t id;             // target index
    std::string tags;        // " LN:i:.. RC:i:.. XC:f:.." exactly as polisher.cpp:521-524 appends them to the name
    std::string data;
};

/* One FASTA record as racon's main prints a polished sequence (src/main.cpp:159-161): ">name tags\ndata\n". */
std::string format_fasta(const std::string& target_name, const PolishedSequence& s);

/* The stitch cursor of the polisher: ranges of windows [first, first + count) finish in any order, and emit(w) is called
 * once for every window, in window order, as soon as it and every window before it have finished.  A range that
 * finishes early waits (its windows keep their consensus) until the ranges before it are in. */
class InOrderStitcher {
public:
    explicit InOrderStitcher(size_t n_windows) : finished_(n_windows, 0) {}
    template <typename Emit>
    void finish(size_t first, size_t count, Emit&& emit) {
        for (size_t w = first; w < first + count; ++w) finished_[w] = 1;
        while (cursor_ < finished_.size() && finished_[cursor_]) emit(cursor_++);
    }
    size_t cursor() const { return cursor_; }   // windows emitted so far

private:
    std::vector<uint8_t> finished_;
    size_t cursor_ = 0;
};

/* ---- target groups: polishing a read set larger than one device's memory -------------------------------------------
 * A group is windows [first_window, end_window) of each target in [first_target, end_target), together with the read
 * store of exactly the sequences it needs: its targets and every read whose overlap onto one of them touches one of
 * those windows.  A group of whole targets has every window of its targets (end_window = kAllWindows); a part of a split
 * target is one target's windows [a, b).  Its store costs read_store_bytes() of those sequences (rp_reads_bytes' rule).
 * A read needed by two groups (racon -f, reads spanning contig ends, overlaps across a part boundary) is counted in both. */
uint64_t read_store_bytes(uint64_t sum_of_lengths, bool any_quality);

struct ReadGroups {
    static constexpr uint32_t kAllWindows = ~0u;
    struct Group {
        uint64_t first_target, end_target;
        uint32_t first_window, end_window;
        uint64_t bytes;   // predicted rp_reads_bytes of the group's store
    };
    std::vector<Group> groups;
    /* group g's overlaps, as indices into the overlaps, in their original (file) order: a window's layer order is the
     * order of its overlaps, and it decides the consensus.  They are the overlaps onto its targets whose target span
     * touches one of its windows.  group g = overlap_order[overlap_first[g] .. overlap_first[g + 1]) */
    std::vector<uint64_t> overlap_first, overlap_order;
    /* the group that aligns overlap k: the first group that holds it */
    std::vector<uint64_t> aligned_in;
    size_t size() const { return groups.size(); }
};

/* A single target whose own store exceeds the budget: it cannot be polished under that budget in one group. */
struct TargetOverBudget : std::runtime_error {
    uint64_t target, bytes, budget;
    TargetOverBudget(uint64_t target, uint64_t bytes, uint64_t budget);
    TargetOverBudget(const std::string& what, uint64_t target, uint64_t bytes, uint64_t budget)
        : std::runtime_error(what), target(target), bytes(bytes), budget(budget) {}
    virtual ~TargetOverBudget() = default;
    virtual std::string message(const std::string& target_name) const;
};

/* With split targets: one window of a target (the target and the reads touching that window) exceeds the budget, so no
 * part can hold it. */
struct WindowOverBudget : TargetOverBudget {
    uint32_t window;
    WindowOverBudget(uint64_t target, uint32_t window, uint64_t bytes, uint64_t budget);
    std::string message(const std::string& target_name) const override;
};

/* Greedy over the targets in order: a group is closed when its next target would push its store over `budget` bytes.
 * Host only.  Reads sequences[i].length and whether sequences[i].quality is set, and t_id / q_id of every overlap.
 * Throws TargetOverBudget.
 * window_length > 0 splits targets: a target whose own store exceeds the budget closes the open group and is cut into
 * maximal parts of consecutive windows (window_length bases each, as the polisher builds them), each a group of its
 * own; an overlap touches windows t_begin / window_length .. (t_end - 1) / window_length of its target (clamped to its
 * last window; an empty span touches its first window).  Targets that fit get the groups they get without splitting.
 * Throws WindowOverBudget when one window does not fit. */
ReadGroups plan_read_groups(uint64_t targets_size, const std::vector<SequenceView>& sequences,
                            const std::vector<Overlap>& overlaps, uint64_t budget, uint32_t window_length = 0);

/* The polisher runs its two device stages on a list of devices: one lane per entry (the same device may appear more than
 * once: {0, 0} = two lanes on one GPU).  The aligner has one batch object per lane, the consensus two; one host thread
 * hands every idle object the next contiguous range of overlaps / windows, launches it asynchronously and collects
 * whichever object has finished (rp_*_query), waiting for the oldest one only when none has — so devices that do not
 * finish in step never hold each other up.  Results are per overlap / per window and the stitch cursor
 * (InOrderStitcher) restores window order, so the output does not depend on the devices, their number or the order in
 * which they finish: a list of one device is the single-GPU polisher.  Every distinct device holds one copy of the
 * read store, shared by the lanes on it. */
class Polisher {
public:
    /* sequences: the targets first (targets_size of them), then the reads — the order racon::Polisher::sequences_ has;
     * devices: CUDA device indices, one lane each (not empty; each below rp_device_count() when a device is visible) */
    Polisher(std::vector<SequenceView> sequences, uint64_t targets_size, WindowType window_type, bool fragment_correction,
             uint32_t window_length, double quality_threshold, bool trim, int8_t match, int8_t mismatch, int8_t gap,
             std::vector<uint32_t> devices);
    ~Polisher();
    /* Device-resident reads: every sequence is uploaded once (rp_reads_create, at first use) and both device stages name
     * their inputs instead of copying them — the aligner its two spans per overlap (rp_aln_add_overlap_ref), the consensus
     * its window pieces (rp_poa_add_window_refs).  Call before initialize(). */
    void use_resident_reads(bool on) { resident_reads_ = on; }
    /* returns the number of overlaps sent to the device aligner */
    size_t find_overlap_breaking_points(std::vector<Overlap>& overlaps);
    void initialize(std::vector<Overlap>& overlaps);
    /* the window-building half of initialize() alone, for overlaps whose breaking points are already known */
    void build_windows(const std::vector<Overlap>& overlaps);
    void polish(std::vector<PolishedSequence>& dst, bool drop_unpolished_sequences);
    /* Streaming form (polisher.cpp:504-537 + main.cpp:159-161 as a consumer overlapped with the compute): two batch
     * objects per lane stay in flight; while they run on the GPUs the finished windows are stitched in window order, and
     * `sink` gets every polished sequence the moment its last window is stitched (e.g. a FASTA writer); stitched windows
     * are released.  `memory` =
     * device budget per batch object (0 = library default), `banded` = racon -b.  `resident_reads`: upload every sequence
     * once (rp_reads) and add the windows by reference — layer extraction on the device, no host copy of layer bytes. */
    void polish_streaming(const std::function<void(const PolishedSequence&)>& sink, bool drop_unpolished_sequences,
                          size_t memory = 0, bool banded = false, bool resident_reads = false);
    /* initialize + polish_streaming(resident_reads = true) in target groups (plan_read_groups): for each group in target
     * order, its store goes to every distinct device, the overlaps it aligns (aligned_in) are aligned, its windows built
     * from its overlaps and polished, its records streamed to `sink`, and its store released; an overlap's breaking points
     * are freed after its last group.  `read_store_bytes` = budget per device (0 = half of the smallest free memory of
     * the devices, read before anything is allocated).  The overlaps come from load_input (filter and window type over
     * the whole input); failed_overlaps / failed_windows keep their whole-run indices, RC:i: counts every overlap onto
     * the target, and the stitch carries from one group to the next, so a target's record goes to `sink` after its last
     * window.  With one group the output is that of initialize + polish_streaming.  Throws TargetOverBudget before any
     * device work.  split_targets: a target whose own store exceeds the budget is polished in parts (plan_read_groups
     * with the window length), with the output of one pass; throws WindowOverBudget (before any device work) when one
     * window does not fit. */
    void polish_groups(std::vector<Overlap>& overlaps, const std::function<void(const PolishedSequence&)>& sink,
                       bool drop_unpolished_sequences, size_t memory, bool banded, uint64_t read_store_bytes,
                       bool split_targets = false);
    /* rp_reads_bytes of each group's store in the last polish_groups (of the first device's copy) */
    const std::vector<uint64_t>& group_store_bytes() const { return group_store_bytes_; }
    /* per group of the last polish_groups: its whole-run windows [first, end), and how many overlaps it aligned */
    const std::vector<std::pair<uint64_t, uint64_t>>& group_windows() const { return group_windows_; }
    const std::vector<uint64_t>& group_aligned() const { return group_aligned_; }
    const std::vector<std::shared_ptr<Window>>& windows() const { return windows_; }
    /* Items the device could not finish (soft RP_ALN_* / RP_WIN_* status).  The reference hands such items to its CPU
     * code (cudapolisher.cpp:213 edlib, :354-370 spoa); this library has no CPU path, so a failed overlap contributes
     * no layers and a failed window keeps its backbone — the result then DIFFERS from racon's, which is why the indices
     * are reported here instead of a stderr line: a caller with a CPU implementation (the integration shim's host is
     * the reference itself) must process them, any other caller should treat a non-empty list as an error. */
    const std::vector<size_t>& failed_overlaps() const { return failed_overlaps_; }
    const std::vector<size_t>& failed_windows() const { return failed_windows_; }

private:
    Polisher(const Polisher&) = delete;
    const Polisher& operator=(const Polisher&) = delete;
    const char* reverse_complement(uint32_t id);
    const char* reverse_quality(uint32_t id);
    /* the breaking points of overlaps[ids[..]]: those with an alignment (SAM) from it, the others on the device;
     * returns the number of overlaps sent to the device aligner */
    size_t find_overlap_breaking_points(std::vector<Overlap>& overlaps, const std::vector<uint64_t>& ids);
    /* the aligner lanes of find_overlap_breaking_points over overlaps[todo[..]] */
    void align(std::vector<Overlap>& overlaps, const std::vector<uint64_t>& todo, uint32_t longest);
    /* RC:i: of every target: the number of overlaps onto it */
    void count_coverages(const std::vector<Overlap>& overlaps);
    /* windows [first_window, end_window) of every target in [first_target, end_target) (polisher.cpp:383-401), appended
     * to windows_, with the layers of overlaps[ids[..]] that fall in them */
    void build_windows(const std::vector<Overlap>& overlaps, const std::vector<uint64_t>& ids, uint64_t first_target,
                       uint64_t end_target, uint32_t first_window, uint32_t end_window);
    /* the stitch of the target whose windows are being emitted: within a run it carries from one group to the next */
    struct Stitch {
        std::string data;
        uint32_t polished_windows = 0;
    };
    /* the one batch loop + stitch of polish() and polish_streaming(); `release`: drop every window once stitched.  A
     * hard error in either stage destroys its batch objects and the read stores before the process exits. */
    void consensus(const std::function<void(const PolishedSequence&)>& sink, Stitch& stitch,
                   bool drop_unpolished_sequences, size_t memory, bool banded, bool resident_reads, bool release);
    void consensus_lanes(const std::function<void(const PolishedSequence&)>& sink, Stitch& stitch,
                         bool drop_unpolished_sequences, size_t memory, bool banded, bool resident_reads, bool release);
    void release_read_stores();
    /* the layers of overlap o in windows [first_window, end_window) of its target, whose window first_window is
     * windows_[first_window_id] (polisher.cpp:405-458) */
    void add_layers(const Overlap& o, uint64_t first_window_id, uint32_t first_window, uint32_t end_window);

    std::vector<SequenceView> sequences_;
    uint64_t targets_size_;
    WindowType window_type_;
    bool fragment_correction_;
    uint32_t window_length_;
    double quality_threshold_;
    bool trim_;
    int8_t match_, mismatch_, gap_;
    std::vector<uint32_t> devices_;
    std::string dummy_quality_;
    std::vector<std::string> reverse_complement_, reverse_quality_;
    std::vector<uint32_t> targets_coverages_;
    std::vector<std::shared_ptr<Window>> windows_;
    std::vector<size_t> failed_overlaps_, failed_windows_;
    bool resident_reads_ = false;
    std::vector<std::pair<uint32_t, rp_reads*>> stores_;   // (device, store): one per distinct device, made at first use
    std::vector<uint64_t> group_store_bytes_, group_aligned_;
    std::vector<std::pair<uint64_t, uint64_t>> group_windows_;
    /* the store on `device`; made at first use, of the sequences i with members[i] (every sequence when empty) */
    const rp_reads* read_store(uint32_t device, const std::vector<uint8_t>& members = {});
};

}  // namespace racon_b200
