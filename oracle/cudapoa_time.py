"""Times the reference's own GPU path (GenomeWorks cudapoa, unmodified, oracle/_ref/libref_cudapoa.so) on the bench
workload and prints one JSON line.  Run as a separate process by bench.py's cpu_baseline leg (a CUDA error in the
reference library must not take the bench down):
  python -m oracle.cudapoa_time --windows 10000 [--banded] [--devices N --batches B]
--devices N drives `B` batch objects on each of N GPUs from one host thread each, exactly the shape of the reference's
CUDAPolisher::polish (cudapolisher.cpp:226-345; racon -c B on an N-GPU box); --windows is then the TOTAL."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=2000)
    ap.add_argument("--banded", action="store_true")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--devices", type=int, default=0, help="0: single batch object on --device (round-1 harness)")
    ap.add_argument("--batches", type=int, default=2)
    a = ap.parse_args()
    from oracle import bindings as ob
    from racon_b200 import windows
    if not ob.have_ref_cudapoa():
        print(json.dumps({"unavailable": "oracle/_ref/libref_cudapoa.so not built"}))
        return
    ws, _ = windows.synth_windows(a.windows, err=0.12, state=42)
    band = "static band 256" if a.banded else "full band"
    if a.devices > 0:
        warm = ws.subset(range(min(400, a.windows)))
        ob.ref_cudapoa_multi(warm, banded=a.banded, n_devices=a.devices, batches_per_device=a.batches)
        ok, wall = ob.ref_cudapoa_multi(ws, banded=a.banded, n_devices=a.devices, batches_per_device=a.batches)
        print(json.dumps({"kind": "reference GPU path: GenomeWorks cudapoa (unmodified, sm_90, %s), %d batch objects on "
                                  "each of %d GPU(s), one host thread per batch object, as CUDAPolisher::polish"
                                  % (band, a.batches, a.devices),
                          "n_gpus": a.devices, "batches_per_gpu": a.batches, "windows": a.windows, "windows_ok": ok,
                          "value": a.windows / wall, "unit": "windows/s", "wall_s": wall}))
        return
    ob.ref_cudapoa_consensus(ws.subset(range(min(200, a.windows))), banded=a.banded, device=a.device)   # warm-up
    cons, ok, wall, gpu = ob.ref_cudapoa_consensus(ws, banded=a.banded, device=a.device)
    print(json.dumps({"kind": "reference GPU path: GenomeWorks cudapoa (unmodified, sm_90, %s), driven as "
                              "CUDABatchProcessor does" % band,
                      "windows": a.windows, "windows_ok": ok, "value": a.windows / wall, "unit": "windows/s",
                      "wall_s": wall, "gpu_call_s": gpu, "value_gpu_calls_only": a.windows / gpu if gpu else None,
                      "mean_consensus_len": float(sum(len(c) for c in cons)) / max(1, ok)}))


if __name__ == "__main__":
    main()
