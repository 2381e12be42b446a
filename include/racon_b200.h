/*
 * racon_b200.h — C ABI of the CUDA-native (sm_90a) POA consensus / pre-alignment hot path.
 *
 * Drop-in boundary for racon's GPU batch objects (SURVEY.md §8b).  Every entry point names the
 * reference interface it replaces; INTEGRATION.md shows the shim a racon maintainer adds in
 * src/cuda/cudabatch.cpp / src/cuda/cudaaligner.cpp.
 *
 * Conventions (same as the reference batch objects):
 *   - sequence / quality pointers passed to add_* are BORROWED only for the duration of the call
 *     (bytes are copied into the object's pinned staging, as cudapoa's add_poa_group does);
 *   - buffers returned by fetch_* are owned by the object and stay valid until reset/destroy;
 *   - one object is used by one host thread at a time; objects are independent (own stream, own device);
 *   - soft per-item status (window did not fit a limit) vs hard errors (negative rp_status);
 *   - no exceptions cross this ABI, no global state besides CUDA contexts;
 *   - there is NO CPU fallback behind any of these calls: without a usable CUDA device rp_*_create fails.
 */
#ifndef RACON_B200_H_
#define RACON_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int32_t rp_status;
enum {
    RP_OK = 0,
    RP_BATCH_FULL = 1,      /* item not added: run the batch, reset, add it again (cudabatch.cpp:126-132) */
    RP_NOT_READY = 2,       /* rp_poa_query / rp_aln_query: the last run is still in flight */
    RP_ERR_INVALID = -1,    /* bad argument / malformed window (the reference exit(1)s: window.cpp:19-23,49-58) */
    RP_ERR_CUDA = -2,       /* CUDA runtime failure; rp_last_error() has the text */
    RP_ERR_NOMEM = -3,
    RP_ERR_STATE = -4,      /* call order violated (e.g. fetch before run) */
    RP_ERR_NO_DEVICE = -5   /* no CUDA device: the hot path has no CPU fallback */
};

/* per-window soft status reported by rp_poa_window_status (0 = consensus produced on the GPU) */
enum {
    RP_WIN_OK = 0,
    RP_WIN_NODE_LIMIT = 1,       /* the graph outgrew the escalation pass's node budget: 8 x (6 * window_len_hint + 64)
                                    nodes, at most 65 000 (the first pass holds 6 * window_len_hint + 64) */
    RP_WIN_EDGE_LIMIT = 2,
    RP_WIN_ALIGNED_LIMIT = 3,
    RP_WIN_NEEDS_INT32 = 4,      /* the score matrix may leave int16 (|gap| > 64, |gap| * (graph depth + length) > ~31k, or
                                    max(match, mismatch) * length > ~31k) */
    RP_WIN_SEQ_TOO_LONG = 5,
    RP_WIN_STACK_LIMIT = 6,
    RP_WIN_ALPHABET_LIMIT = 7,
    RP_WIN_INTERNAL = 8,
    RP_WIN_MATRIX_LIMIT = 9      /* score matrix larger than the per-window scratch even in the escalation pass */
};

enum { RP_WINDOW_NGS = 0, RP_WINDOW_TGS = 1 }; /* racon::WindowType, src/window.hpp:20-23 */

const char* rp_strerror(rp_status s);
const char* rp_last_error(void);          /* thread-local text of the last hard error */
int rp_device_count(void);                /* cudaGetDeviceCount; <= 0 when no device (cudapolisher.cpp:48) */
/* cudaMemGetInfo on `device`: the bytes free and in all (what the batch objects size their defaults from) */
rp_status rp_device_memory(int device, uint64_t* free_bytes, uint64_t* total_bytes);
const char* rp_version(void);

/* ------------------------------------------------------------------------------------------------
 * POA consensus batch — replaces racon::CUDABatchProcessor (src/cuda/cudabatch.hpp:27-122) and the
 * cudapoa::Batch it wraps (vendor/GenomeWorks/cudapoa/include/.../batch.hpp:45-56,108-159);
 * per window it computes what Window::generate_consensus (src/window.cpp:65-149) computes.
 * ------------------------------------------------------------------------------------------------ */
typedef struct rp_poa rp_poa;

/* createCUDABatch(max_window_depth, device, avail_mem, gap, mismatch, match, banded), cudabatch.cpp:23-72.
 * mem_bytes: device-memory budget for this object (0 = 80 % of what is free).
 * window_len_hint: racon -w (sizes per-window scratch; 0 = 500).  max_depth_hint: 0 = unlimited
 * (unlike cudapoa's MAX_DEPTH 200, cudapolisher.cpp:226, no layers are dropped). */
rp_status rp_poa_create(rp_poa** out, int device, size_t mem_bytes, int8_t match, int8_t mismatch, int8_t gap,
                        int banded, uint32_t window_len_hint, uint32_t max_depth_hint);
void rp_poa_destroy(rp_poa* p);

/* CUDABatchProcessor::addWindow (cudabatch.cpp:77-175) = Window ctor + add_layer (window.cpp:30-63).
 * seq[0]/qual[0] = backbone (qual[0] may be NULL => dummy '!' quality, polisher.cpp:174,396-399);
 * seq[k>0] = layers with inclusive backbone coordinates begin[k]..end[k] (begin[0], end[0] ignored);
 * qual[k] NULL => weight 1.  Layers with len == 0 or begin == end are skipped like add_layer does.
 * Returns RP_OK, RP_BATCH_FULL, or RP_ERR_INVALID. */
rp_status rp_poa_add_window(rp_poa* p, uint32_t n_seq, const char* const* seq, const uint32_t* len,
                            const char* const* qual, const uint32_t* begin, const uint32_t* end, int window_type,
                            int trim);

/* ---- device-resident reads: windows whose layers are slices of sequences already in HBM (SURVEY §8 f2) ----------------
 * The reference builds a window from pointers into its sequences (polisher.cpp:383-461: backbone = a stretch of the
 * target, layer = a stretch of a read or of its reverse complement) and its CUDA path copies those bytes together on the
 * host, window by window (cudabatch.cpp:77-175).  With a store, every sequence is uploaded once and a window names its
 * pieces; the packed arrays the kernel reads are gathered on the device (reverse complement and quality -> weight
 * included), so no sequence byte is touched on the host when a window is added.
 *
 * rp_reads_create: data[i] / length[i] = sequence i (targets and reads, any order); quality[i] NULL (or quality NULL) =
 * no qualities.  The host arrays must stay valid while the store is alive (backbone copies of windows with < 3 sequences
 * and the rare exact alphabet scan read them).  One store can serve any number of batch objects on the same device, on
 * any of their streams: nothing writes to a store after rp_reads_create has returned (its upload is complete by then).
 * A sequence given with length 0 (its data may then be NULL) is absent: it costs nothing, and a window piece or an
 * overlap that names it with a non-empty span is refused with RP_ERR_INVALID.  A store can so hold a subset of a
 * sequence table under the table's own ids. */
typedef struct rp_reads rp_reads;
rp_status rp_reads_create(rp_reads** out, int device, uint32_t n_seqs, const char* const* data,
                          const char* const* quality, const uint32_t* length);
void rp_reads_destroy(rp_reads* r);
/* Device bytes the store occupies, exactly: (sum of length[i] + 16) bytes of bases, and the same again for qualities
 * when any sequence of non-zero length has a quality string.  Callers size their stores with this rule. */
uint64_t rp_reads_bytes(const rp_reads* r);

/* rp_poa_add_window with the pieces named instead of passed: piece k = length[k] bases of sequence seq_id[k] starting at
 * offset[k]; reverse[k] != 0: offset counts in the reverse complement of the sequence (racon's
 * `reverse_complement()[offset]`), and the piece is read back to front, complemented, its qualities reversed.  Piece 0 is
 * the backbone (never reverse; begin/end ignored).  Same checks, skips, statuses and results as rp_poa_add_window.
 * A batch holds either windows added this way (all from one store) or windows added by pointer: RP_ERR_STATE otherwise. */
rp_status rp_poa_add_window_refs(rp_poa* p, const rp_reads* reads, uint32_t n_seq, const uint32_t* seq_id,
                                 const uint32_t* offset, const uint32_t* length, const uint8_t* reverse,
                                 const uint32_t* begin, const uint32_t* end, int window_type, int trim);

/* Bulk form of rp_poa_add_window_refs: windows [first, first + count) of a flat description — pieces
 * win_first[w] .. win_first[w + 1] of the piece arrays belong to window w, backbone first (win_type NULL = all TGS).
 * Stops at the first window that does not fit; *added = how many were taken (RP_OK when > 0, else RP_BATCH_FULL). */
rp_status rp_poa_add_window_set_refs(rp_poa* p, const rp_reads* reads, uint32_t first, uint32_t count,
                                     const uint32_t* seq_id, const uint32_t* offset, const uint32_t* length,
                                     const uint8_t* reverse, const uint32_t* begin, const uint32_t* end,
                                     const uint32_t* win_first, const uint8_t* win_type, int trim, uint32_t* added);

/* Bulk form of rp_poa_add_window over flat arrays (see racon_b200/windows.py): adds windows
 * [first, first + count) of the set until the batch is full; *added = how many were taken. */
rp_status rp_poa_add_window_set(rp_poa* p, uint32_t first, uint32_t count, const char* bases, const char* quals,
                                const uint64_t* seq_off, const uint8_t* seq_has_qual, const uint32_t* seq_begin,
                                const uint32_t* seq_end, const uint32_t* win_first, const uint8_t* win_type, int trim,
                                uint32_t* added);

uint32_t rp_poa_size(const rp_poa* p);    /* windows in the batch (CUDABatchProcessor::hasWindows) */

/* CUDABatchProcessor::generateConsensus = generate_poa + get_consensus (cudabatch.cpp:193-270):
 * rp_poa_run = upload + launch + download, asynchronous on the object's stream; rp_poa_sync waits. */
rp_status rp_poa_run(rp_poa* p);
rp_status rp_poa_sync(rp_poa* p);
/* Non-blocking completion test of the last run: RP_OK when it has finished (rp_poa_sync then returns without waiting
 * for the device, unless windows have to be escalated), RP_NOT_READY while it is in flight, RP_ERR_STATE when nothing
 * was launched since the last reset.  Lets one host thread keep batch objects on several devices busy. */
rp_status rp_poa_query(rp_poa* p);
/* the three stages separately (bench.py times rp_poa_launch alone with inputs resident in HBM) */
rp_status rp_poa_upload(rp_poa* p);
rp_status rp_poa_launch(rp_poa* p);
rp_status rp_poa_download(rp_poa* p);

/* Window::consensus() + the bool generate_consensus returns (window.cpp:65-149); coverage = per-base
 * coverage of the returned consensus (Graph::GenerateConsensus summary, graph.cpp:377-398), saturated at 65 535
 * (cudapoa's uint16).  The device counts sequences through a node in 32 bits, and the trim compares the exact sum. */
rp_status rp_poa_fetch(rp_poa* p, uint32_t i, const char** consensus, uint32_t* len, const uint16_t** coverage,
                       int* polished);
rp_status rp_poa_window_status(rp_poa* p, uint32_t i, uint32_t* status);
/* bulk fetch: out is n x stride bytes; any output pointer may be NULL */
rp_status rp_poa_fetch_all(rp_poa* p, char* out, uint32_t stride, uint32_t* lens, uint8_t* polished,
                           uint32_t* status);

rp_status rp_poa_reset(rp_poa* p);        /* CUDABatchProcessor::reset (cudabatch.cpp:272-278) */

/* stream / measurement hooks */
rp_status rp_poa_set_stream(rp_poa* p, void* cuda_stream);   /* use the caller's cudaStream_t */
/* info[0] kernel launches so far, [1] last H2D bytes, [2] last D2H bytes, [3] worker warps,
 * [4] scratch bytes per warp; with counters enabled: [5] alignments done, [6] DP cells sum (L+1)(N+1),
 * [7] predecessor cells sum (L+1)*E (E = sum over rows of max(1, in-degree)) — SURVEY.md §8(d) byte model.
 * L = read length, N = graph rows of the alignment (the subgraph's for a partial-span layer); an alignment accepted
 * inside the band counts the band width in place of L+1.
 * [5]-[7] are per launch, not cumulative: every rp_poa_launch (and so every rp_poa_run) starts them from zero, and
 * rp_poa_download reads back those of the launch before it (all three 0 when counters were off at that download, or
 * the batch had no GPU window).  They count the first pass only: the escalation pass rp_poa_sync runs for windows over
 * a first-pass limit is not counted, so such a window contributes the alignments it finished before it failed the
 * first pass (none, when its backbone is over the node budget or its first layer over the length limit).  Windows of
 * fewer than 3 sequences and windows over the alphabet limit never reach the device and count nothing. */
rp_status rp_poa_info(rp_poa* p, uint64_t info[8]);
rp_status rp_poa_enable_counters(rp_poa* p, int on);
/* racon -b / --cuda-banded-alignment (createCUDABatch's `banded`, cudabatch.cpp:56-59): after a run (counts of the
 * last launch's first pass, like rp_poa_info's [5]-[7]),
 * info[0] = 1 when the object is banded, [1] alignments tried inside the band, [2] alignments whose band result
 * was refused by the device-side check and that were redone with the full matrix on the device, [3] band width
 * in columns, [4] (only with the environment variable RP_BAND_AUDIT=1, a test mode that recomputes every accepted
 * band result with the full matrix) accepted band alignments that differ from the full-matrix alignment, [5] 1 when the
 * band layout is in use: a banded object uses it for windows of 768 bases or more (where it is the faster kernel) or when
 * the environment variables RP_POA_BAND_K (band columns per lane) / RP_POA_GROUP (lanes per window) ask for it; each
 * layout has a kernel and a launch shape of its own.  Otherwise -b runs the full matrix, which returns the same results
 * faster.
 * Banded and unbanded objects return identical results (tests/test_gpu_poa.py). */
rp_status rp_poa_band_info(rp_poa* p, uint64_t info[8]);

/* ------------------------------------------------------------------------------------------------
 * Pre-alignment batch — replaces racon::CUDABatchAligner (src/cuda/cudaaligner.hpp:21-92) and the
 * cudaaligner::Aligner it wraps (vendor/GenomeWorks/cudaaligner/include/.../aligner.hpp:56-82); per overlap it
 * computes what Overlap::align_overlaps (src/overlap.cpp:205-224) computes with edlib:
 * edlibAlign(query, target, NW, k = -1, TASK_PATH) -> edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD).
 * The CIGAR is byte-identical to edlib's (tests/test_gpu_aln.py).  An overlap the device cannot take
 * (band wider than 16384 rows, sequence longer than the object's limit, > 16 distinct characters) gets a soft
 * status and an empty CIGAR, exactly like a cudaaligner failure: the caller's CPU edlib call then handles it
 * (src/cuda/cudapolisher.cpp:213, "overlaps whose cigar_ is still empty").
 * ------------------------------------------------------------------------------------------------ */
typedef struct rp_aln rp_aln;

enum {
    RP_ALN_OK = 0,
    RP_ALN_BAND_LIMIT = 1,
    RP_ALN_ALPHABET_LIMIT = 2,
    RP_ALN_STORE_LIMIT = 3,
    RP_ALN_INTERNAL = 4,
    RP_ALN_RUN_LIMIT = 5,
    RP_ALN_TOO_LONG = 6
};

/* createCUDABatchAligner(max_query, max_target, max_alignments, device), src/cuda/cudaaligner.cpp:18-49.
 * max_len: longest query/target this object accepts (0 = 65536); mem_bytes: device budget (0 = 40 % of free). */
rp_status rp_aln_create(rp_aln** out, int device, size_t mem_bytes, uint32_t max_len);
void rp_aln_destroy(rp_aln* a);
/* CUDABatchAligner::addOverlap (cudaaligner.cpp:51-78): query = read span, target = contig span, in racon's
 * orientation (overlap.cpp:193-197).  RP_OK | RP_BATCH_FULL | RP_ERR_INVALID. */
rp_status rp_aln_add(rp_aln* a, const char* q, uint32_t ql, const char* t, uint32_t tl);
/* Breaking points on the device (Overlap::find_breaking_points_from_cigar, src/overlap.cpp:226-292): set the window
 * length (Polisher::window_length_) on an empty batch, add overlaps with their coordinates — t_begin = Overlap::t_begin_,
 * q_start = strand ? q_length - q_end : q_begin (overlap.cpp:241) — and fetch, after the run, the (t, q) points the
 * reference would have stored in Overlap::breaking_points_ (uint32 pairs, two points per window with a match). */
rp_status rp_aln_set_window_length(rp_aln* a, uint32_t window_length);
rp_status rp_aln_add_overlap(rp_aln* a, const char* q, uint32_t ql, const char* t, uint32_t tl, uint32_t t_begin,
                             uint32_t q_start);
/* The same overlap named instead of passed (device-resident reads, rp_reads_create): query = q_len bases of sequence q_id
 * from q_start on — of its reverse complement when q_reverse (racon's `reverse_complement()[q_length - q_end]`,
 * overlap.cpp:193-195) —, target = t_len bases of sequence t_id from t_begin on.  The spans are gathered on the device;
 * nothing but the descriptor crosses the bus.  A batch holds overlaps of one kind (by pointer, or by reference into one
 * store): RP_ERR_STATE otherwise. */
rp_status rp_aln_add_overlap_ref(rp_aln* a, const rp_reads* reads, uint32_t q_id, uint32_t q_start, uint32_t q_len,
                                 int q_reverse, uint32_t t_id, uint32_t t_begin, uint32_t t_len);
rp_status rp_aln_fetch_breaking_points(rp_aln* a, uint32_t i, const uint32_t** points, uint32_t* n_points);
uint32_t rp_aln_size(const rp_aln* a);
/* CUDABatchAligner::alignAll (async) / generate_cigar_strings (sync), cudaaligner.cpp:80-104 */
rp_status rp_aln_run(rp_aln* a);
rp_status rp_aln_sync(rp_aln* a);
/* rp_poa_query for the aligner: RP_OK (finished), RP_NOT_READY (in flight) or RP_ERR_STATE (nothing launched) */
rp_status rp_aln_query(rp_aln* a);
rp_status rp_aln_upload(rp_aln* a);
rp_status rp_aln_launch(rp_aln* a);
rp_status rp_aln_download(rp_aln* a);
/* Overlap::cigar_ for overlap i (NUL-terminated; empty when status != RP_ALN_OK), its edit distance, soft status */
rp_status rp_aln_fetch_cigar(rp_aln* a, uint32_t i, const char** cigar, uint32_t* len, int32_t* edit_distance,
                             uint32_t* status);
rp_status rp_aln_reset(rp_aln* a);
rp_status rp_aln_set_stream(rp_aln* a, void* cuda_stream);
/* info[0] kernel launches, [1] last H2D bytes, [2] last D2H bytes, [3] worker warps, [4] scratch bytes per warp */
rp_status rp_aln_info(rp_aln* a, uint64_t info[8]);

#ifdef __cplusplus
}
#endif
#endif /* RACON_B200_H_ */
