/*
 * racon_main.cpp — the racon_b200 command line: racon's arguments in, racon's polished FASTA on stdout.
 *
 *   racon_b200 [options ...] <sequences> <overlaps> <target sequences> > polished.fasta
 *
 * The option table and its parsing are racon 1.5.0's with CUDA support (getopt_long over "ufw:q:e:m:x:g:t:hbc::", atoi /
 * atof conversions, int8_t scores, `-c` taking its count from the next word when that word is not an option).  The run is
 * the host layer's: load_input (parsing + racon's overlap filter), then Polisher on every visible GPU (alignment,
 * breaking points and consensus on the device) in target groups whose sequences fit the device read store budget
 * (polish_groups, RP_READ_STORE_BYTES; with --split-targets a target that does not fit on its own is polished in window
 * ranges that do), whose sink writes each record to stdout the moment it is stitched.
 *
 * Exit status: 0 = racon's bytes; 1 = an error (bad argument, bad input, no device, a target over the read store budget
 * (with --split-targets: a window over it), a device error, a failed write);
 * 2 = the output was written, but the device refused some overlaps or windows (a soft RP_ALN_* / RP_WIN_* status).  racon
 * redoes such items on its CPU; this program has no CPU path, so its output then differs from racon's.
 */
#include <getopt.h>
#include <signal.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <cerrno>
#include <cstring>
#include <exception>
#include <string>
#include <vector>

#include "host_mirror.hpp"
#include "racon_b200.h"
#include "reads_io.hpp"

namespace {

constexpr int kCudaAlignerBatches = 10000;     // long options without a short form
constexpr int kCudaAlignerBandWidth = 10001;
constexpr int kSplitTargets = 10002;

const struct option kOptions[] = {
    {"include-unpolished", no_argument, nullptr, 'u'},
    {"fragment-correction", no_argument, nullptr, 'f'},
    {"window-length", required_argument, nullptr, 'w'},
    {"quality-threshold", required_argument, nullptr, 'q'},
    {"error-threshold", required_argument, nullptr, 'e'},
    {"no-trimming", no_argument, nullptr, 'T'},
    {"match", required_argument, nullptr, 'm'},
    {"mismatch", required_argument, nullptr, 'x'},
    {"gap", required_argument, nullptr, 'g'},
    {"threads", required_argument, nullptr, 't'},
    {"version", no_argument, nullptr, 'v'},
    {"help", no_argument, nullptr, 'h'},
    {"cudapoa-batches", optional_argument, nullptr, 'c'},
    {"cuda-banded-alignment", no_argument, nullptr, 'b'},
    {"cudaaligner-batches", required_argument, nullptr, kCudaAlignerBatches},
    {"cudaaligner-band-width", required_argument, nullptr, kCudaAlignerBandWidth},
    {"split-targets", no_argument, nullptr, kSplitTargets},
    {nullptr, 0, nullptr, 0}};

void usage(FILE* out) {
    fputs(
        "usage: racon_b200 [options ...] <sequences> <overlaps> <target sequences>\n"
        "\n"
        "Polishes the target sequences with the sequences and their overlaps, as racon does, and writes the polished\n"
        "sequences to stdout in FASTA.  Overlap alignment and window consensus run on every visible CUDA device\n"
        "(select them with CUDA_VISIBLE_DEVICES); there is no CPU path.\n"
        "\n"
        "    <sequences>         FASTA/FASTQ reads (.fasta .fa .fna .fastq .fq, each also .gz)\n"
        "    <overlaps>          MHAP/PAF/SAM overlaps of the reads with the targets (.mhap .paf .sam, each also .gz)\n"
        "    <target sequences>  FASTA/FASTQ sequences to polish\n"
        "\n"
        "options (racon's, with racon's defaults):\n"
        "    -u, --include-unpolished       also print target sequences no window of which was polished\n"
        "    -f, --fragment-correction      fragment correction instead of contig polishing (dual/self overlaps)\n"
        "    -w, --window-length <int>      default 500: window length of the consensus\n"
        "    -q, --quality-threshold <float> default 10.0: lowest average base quality of a window piece\n"
        "    -e, --error-threshold <float>  default 0.3: highest error rate of an overlap that is kept\n"
        "    --no-trimming                  keep the low-coverage ends of every window consensus\n"
        "    -m, --match <int>              default 3: match score\n"
        "    -x, --mismatch <int>           default -5: mismatch score\n"
        "    -g, --gap <int>                default -4: gap penalty (not positive)\n"
        "    -b, --cuda-banded-alignment    banded consensus alignment (same output wherever the band holds the optimum)\n"
        "    -c, --cudapoa-batches [<int>]  default 1: lanes per GPU; a lane is one aligner and two consensus batches\n"
        "                                   (a count below 1 is taken as 1)\n"
        "    --split-targets                polish a target whose sequences do not fit the read store budget in\n"
        "                                   consecutive window ranges that do, with the output of one pass; a single\n"
        "                                   window that does not fit is an error (status 1)\n"
        "    --version                      print the library version\n"
        "    -h, --help                     print this text\n"
        "\n"
        "accepted so that racon command lines keep working, without effect:\n"
        "    -t, --threads <int>            the host work runs on one thread\n"
        "    --cudaaligner-batches <int>    alignment always runs on the device; the lanes decide the batches\n"
        "    --cudaaligner-band-width <int> alignment is always exact (edlib's result)\n"
        "\n"
        "environment:\n"
        "    RP_READ_STORE_BYTES=<bytes>    device memory per GPU for the sequences of one group of targets: the targets\n"
        "                                   are polished in consecutive groups whose sequences fit it, with the output of\n"
        "                                   one pass.  Unset or 0: half of the smallest free GPU memory.  A target whose\n"
        "                                   own sequences do not fit is an error (status 1),\n"
        "                                   unless --split-targets is given\n"
        "\n"
        "exit status: 0 = output written; 1 = error; 2 = output written, but the device refused some overlaps or\n"
        "windows, which racon would have redone on its CPU: the output then differs from racon's.\n",
        out);
}

/* RP_READ_STORE_BYTES: the read store budget per device, in bytes (unset, empty or 0 = automatic: half of the smallest
 * free device memory).  false when it is not a plain decimal number that fits 64 bits. */
bool read_store_budget(uint64_t* bytes) {
    *bytes = 0;
    const char* s = getenv("RP_READ_STORE_BYTES");
    if (s == nullptr || *s == '\0') return true;
    for (const char* c = s; *c; ++c) {
        if (*c < '0' || *c > '9') return false;
    }
    errno = 0;
    const unsigned long long v = strtoull(s, nullptr, 10);
    if (errno == ERANGE) return false;
    *bytes = v;
    return true;
}

/* thrown by the output sink: unwinds through the polisher, whose batch objects and read stores are released on the way */
struct WriteError : std::exception {
    int error;
    explicit WriteError(int e) : error(e) {}
};

}  // namespace

int main(int argc, char** argv) {
    uint32_t window_length = 500;
    double quality_threshold = 10.0;
    double error_threshold = 0.3;
    bool trim = true;
    int8_t match = 3, mismatch = -5, gap = -4;
    bool fragment_correction = false;
    bool drop_unpolished_sequences = true;
    int lanes_per_device = 1;
    bool banded = false;
    bool split_targets = false;

    int argument;
    while ((argument = getopt_long(argc, argv, "ufw:q:e:m:x:g:t:hbc::", kOptions, nullptr)) != -1) {
        switch (argument) {
            case 'u': drop_unpolished_sequences = false; break;
            case 'f': fragment_correction = true; break;
            case 'w': window_length = static_cast<uint32_t>(atoi(optarg)); break;
            case 'q': quality_threshold = atof(optarg); break;
            case 'e': error_threshold = atof(optarg); break;
            case 'T': trim = false; break;
            case 'm': match = static_cast<int8_t>(atoi(optarg)); break;
            case 'x': mismatch = static_cast<int8_t>(atoi(optarg)); break;
            case 'g': gap = static_cast<int8_t>(atoi(optarg)); break;
            case 't': break;
            case 'v': printf("%s\n", rp_version()); return 0;
            case 'h': usage(stdout); return 0;
            case 'c':
                /* racon's rule: without an attached value the next word is the count unless it looks like an option */
                lanes_per_device = 1;
                if (optarg == nullptr && optind < argc && argv[optind][0] != '-') lanes_per_device = atoi(argv[optind++]);
                if (optarg != nullptr) lanes_per_device = atoi(optarg);
                break;
            case 'b': banded = true; break;
            case kCudaAlignerBatches: break;
            case kCudaAlignerBandWidth: break;
            case kSplitTargets: split_targets = true; break;
            default: return 1;   // getopt_long has named the option on stderr
        }
    }
    if (argc - optind < 3) {
        fprintf(stderr, "[racon_b200::main] error: missing input file(s)!\n");
        usage(stderr);
        return 1;
    }
    const std::string reads_path = argv[optind], overlaps_path = argv[optind + 1], targets_path = argv[optind + 2];

    /* racon's order of checks: window length, the three file extensions, then the files themselves — all before any
     * device is looked for */
    if (window_length == 0) {
        fprintf(stderr, "[racon_b200::main] error: invalid window length!\n");
        return 1;
    }
    uint64_t read_store_bytes = 0;
    if (!read_store_budget(&read_store_bytes)) {
        fprintf(stderr, "[racon_b200::main] error: RP_READ_STORE_BYTES must be a decimal byte count, not \"%s\"!\n",
                getenv("RP_READ_STORE_BYTES"));
        return 1;
    }
    racon_b200::InputSet input;
    try {
        input = racon_b200::load_input(reads_path, overlaps_path, targets_path, fragment_correction, error_threshold);
    } catch (const std::exception& e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }

    const int device_count = rp_device_count();
    if (device_count <= 0) {
        fprintf(stderr, "[racon_b200::main] error: %s\n", rp_strerror(RP_ERR_NO_DEVICE));
        return 1;
    }
    /* lane round r on every device before round r + 1 on any: the first batches go to all GPUs */
    std::vector<uint32_t> devices;
    for (int r = 0; r < std::max(lanes_per_device, 1); ++r) {
        for (int d = 0; d < device_count; ++d) devices.push_back(static_cast<uint32_t>(d));
    }

    /* a closed pipe must end the run with status 1 from a failed write, not kill it silently */
    signal(SIGPIPE, SIG_IGN);
    static char out_buffer[1 << 20];
    setvbuf(stdout, out_buffer, _IOFBF, sizeof(out_buffer));

    size_t failed_overlaps = 0, failed_windows = 0;
    try {
        racon_b200::Polisher polisher(input.views(), input.targets_size, input.window_type, fragment_correction,
                                      window_length, quality_threshold, trim, match, mismatch, gap, devices);
        polisher.polish_groups(
            input.overlaps,
            [&](const racon_b200::PolishedSequence& s) {
                const std::string record = racon_b200::format_fasta(input.sequences[s.id].name, s);
                if (fwrite(record.data(), 1, record.size(), stdout) != record.size()) throw WriteError(errno);
            },
            drop_unpolished_sequences, 0, banded, read_store_bytes, split_targets);
        failed_overlaps = polisher.failed_overlaps().size();
        failed_windows = polisher.failed_windows().size();
    } catch (const WriteError& e) {
        fprintf(stderr, "[racon_b200::main] error: writing the output failed: %s\n", strerror(e.error));
        return 1;
    } catch (const racon_b200::TargetOverBudget& e) {   // a target, or with --split-targets a window, over the budget
        fprintf(stderr, "%s\n", e.message(input.sequences[e.target].name).c_str());
        if (!split_targets) {
            fprintf(stderr, "[racon_b200::main] note: --split-targets polishes such a target in window ranges that fit\n");
        }
        return 1;
    }
    if (fflush(stdout) != 0 || ferror(stdout)) {
        fprintf(stderr, "[racon_b200::main] error: writing the output failed: %s\n", strerror(errno));
        return 1;
    }
    if (failed_overlaps > 0 || failed_windows > 0) {
        fprintf(stderr,
                "[racon_b200::main] warning: the device refused %zu overlap(s) and %zu window(s); racon would redo them "
                "on its CPU, so this output differs from racon's\n",
                failed_overlaps, failed_windows);
        return 2;
    }
    return 0;
}
