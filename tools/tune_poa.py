"""Kernel-only throughput of rp_poa_kernel over its launch-shape knobs (lanes per window, blocks per SM, banded),
inputs resident in HBM, CUDA-event timed.  A tuning aid; bench.py is the judged measurement.
  python tools/tune_poa.py [--windows 10000] [--configs "banded,lanes,blocks_per_sm[,band columns per lane];..."]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--configs", default="0,32,4;0,16,4;0,8,4;1,16,4;1,8,4;1,8,3;1,8,2;0,8,3;0,16,3;1,16,3")
    ap.add_argument("--two-streams", action="store_true", help="also time launches alternating between two objects")
    ap.add_argument("--wlen", type=int, default=500, help="window length of the synthetic windows")
    ap.add_argument("--replicate", type=int, default=1, help="every window this many times in a row (lock-step experiment)")
    args = ap.parse_args()
    import torch
    from racon_b200 import api, windows
    ws, _ = windows.synth_windows(args.windows // args.replicate, truth_len=args.wlen, err=0.12)
    import numpy as np
    if args.replicate > 1:
        ws = ws.subset(np.repeat(np.arange(ws.n_windows), args.replicate))
    stride = int(2 * np.diff(ws.seq_off.astype(np.int64)).max() + 64)
    ref = None
    for cfg in args.configs.split(";"):
        f = [int(x) for x in cfg.split(",")]
        banded, g, bps = f[:3]
        k = f[3] if len(f) > 3 else 16
        os.environ["RP_POA_GROUP"] = str(g)
        os.environ["RP_BLOCKS_PER_SM"] = str(bps)
        os.environ["RP_POA_BAND_K"] = str(k)
        try:
            b = api.PoaBatch(device=0, window_length=args.wlen, banded=bool(banded), mem_bytes=int(30e9))
            st = torch.cuda.current_stream()
            b.set_stream(st.cuda_stream)
            assert b.add_window_set(ws) == ws.n_windows
            b.run()
            b.sync()
            out, lens, pol, status = b.fetch_all(stride)
            ck = "%016x" % windows.fnv1a64([out[i, :lens[i]].tobytes() for i in range(min(ws.n_windows, 200))])
            full = windows.fnv1a64([out[i, :lens[i]].tobytes() for i in range(ws.n_windows)])
            if ref is None:
                ref = full
            bi = b.band_info()
            b.upload()
            b.launch()
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.reps + 1)]
            ev[0].record(st)
            for kk in range(args.reps):
                b.launch()
                ev[kk + 1].record(st)
            torch.cuda.synchronize()
            ms = [ev[kk].elapsed_time(ev[kk + 1]) for kk in range(args.reps)]
            info = b.info()
            res = {"banded": banded, "lanes": g, "blocks_per_sm": bps, "band_cols_per_lane": k, "ms": [round(x, 2) for x in ms],
                   "windows_per_s": round(ws.n_windows / (min(ms) * 1e-3)), "workers": info["workers"],
                   "scratch_MB_per_worker": round(info["scratch_bytes_per_worker"] / 1e6, 2),
                   "bad_status": int((status != 0).sum()), "fnv200": ck, "same_as_first": full == ref,
                   "band": bi}
            if args.two_streams:
                b2 = api.PoaBatch(device=0, window_length=args.wlen, banded=bool(banded), mem_bytes=int(30e9))
                s2 = torch.cuda.Stream()
                b2.set_stream(s2.cuda_stream)
                assert b2.add_window_set(ws) == ws.n_windows
                b2.upload()
                b2.launch()
                torch.cuda.synchronize()
                e0, e1, eb = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record(st)
                s2.wait_event(e0)
                K = 6
                for kk in range(K):
                    (b if kk % 2 == 0 else b2).launch()
                eb.record(s2)
                st.wait_event(eb)
                e1.record(st)
                torch.cuda.synchronize()
                res["two_stream_windows_per_s"] = round(K * ws.n_windows / (e0.elapsed_time(e1) * 1e-3))
                b2.close()
            b.close()
        except Exception as e:  # noqa: BLE001
            res = {"banded": banded, "lanes": g, "blocks_per_sm": bps, "error": str(e)[:300]}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
