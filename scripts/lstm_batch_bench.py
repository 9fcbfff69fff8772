"""Time the LSTM recurrence above 256 rows: one JSON document per run.

    python scripts/lstm_batch_bench.py [--out DIR] [--H 512,768,1024] [--B 257,384,512] [--T 500]

`qb_lstm_tc` runs a batch as ceil(B / 128) launches of at most 128 rows, one after the other, so its time grows in steps of
128 rows.  Builds made before the mma.sync recurrence (`qb_lstm`, one launch over all rows) was removed still export it;
point QB_LIB at such a build and the script times that kernel on the same inputs too, and reports how far its output is from
`qb_lstm_tc`'s.  Times are CUDA-event means over at least half a second per shape, after a warm-up, with the card's name,
power limit and max SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clk = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(name=name, power_limit=power, clocks_max_sm=clk)


def timed(fn, min_s=0.5):
    """Mean ms per call over a window of at least min_s seconds of CUDA-event time, after a warm-up."""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record(); torch.cuda.synchronize()
    reps = max(3, int(min_s * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def mma_lstm(lib):
    """The mma.sync recurrence of an older build, or None"""
    try:
        run, ws_bytes = lib.qb_lstm, lib.qb_lstm_workspace_bytes
    except AttributeError:
        return None
    vp, i64 = C.c_void_p, C.c_int64
    run.restype, run.argtypes = C.c_int, [vp, vp, vp, i64, i64, i64, vp, vp, vp, vp]
    ws_bytes.restype, ws_bytes.argtypes = i64, [i64, i64]
    return run, ws_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for lstm_batch_bench.json (default: print only)")
    ap.add_argument("--H", default="512,768,1024")
    ap.add_argument("--B", default="257,384,512")
    ap.add_argument("--T", type=int, default=500)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lstm_batch_bench: needs a CUDA device")
    from unified_audio_b200 import _lib, ops
    lib = _lib.load()
    mma = mma_lstm(lib)
    stream = torch.cuda.current_stream().cuda_stream
    T, rows = args.T, []
    for H in (int(v) for v in args.H.split(",")):
        U = ops.lstm_tc_units(H)
        g = torch.Generator(device="cuda").manual_seed(H)
        whh = (torch.rand(4 * H, H, generator=g, device="cuda") * 2 - 1) / math.sqrt(H)
        whh_perm, whh16 = ops.lstm_tc_permute(whh, U), whh.half().contiguous()
        for B in (int(v) for v in args.B.split(",")):
            xp = torch.randn(B, T, 4 * H, generator=g, device="cuda")
            out = ops.Planes.zeros((B, T, H), True, "cuda")
            ws = torch.zeros(ops.lstm_tc_workspace_bytes(B, H), dtype=torch.uint8, device="cuda")
            r = dict(H=H, B=B, T=T, units=U, launches=-(-B // 128),
                     lstm_tc_ms=round(timed(lambda: ops.lstm_tc(xp, whh_perm, U, B, T, H, out, ws)), 3))
            if mma is not None:
                run, ws_bytes = mma
                out2 = ops.Planes.zeros((B, T, H), True, "cuda")
                ws2 = torch.zeros(int(ws_bytes(B, H)), dtype=torch.uint8, device="cuda")
                args2 = [xp.data_ptr(), whh16.data_ptr(), None, B, T, H, out2.hi.data_ptr(), out2.lo.data_ptr(),
                         ws2.data_ptr(), stream]
                r["lstm_mma_ms"] = round(timed(lambda: _lib.check(run(*args2))), 3)
                r["mma_over_tc"] = round(r["lstm_mma_ms"] / r["lstm_tc_ms"], 3)
                r["max_abs_diff"] = float((out.float() - out2.float()).abs().max())
                del out2, ws2
            print(json.dumps(r), flush=True)
            rows.append(r)
            del xp, out, ws
        torch.cuda.empty_cache()
    doc = dict(card=card(), lib=_lib.LIB_PATH, mma_available=mma is not None, rows=rows)
    print(json.dumps(doc))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "lstm_batch_bench.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
