"""Times ``opb_topk10_rows`` (csrc/recall.cu) on the retrieval-evaluation shape: a 5,000 x 25,010 fp32 similarity matrix
(COCO 5k images x 25,010 captions), N(0, 1) entries.  With several --lib builds of the extension, the launches alternate
between them in the same process, and their outputs on the timed matrix must agree (ties are absent from N(0, 1) data, so
any correct ranking gives the same indices).

Each figure is the median over --repeat windows of --iters launches, timed with CUDA events, after --warmup launches per
build.  Bytes moved: R * C * 4 read + R * 10 * 8 written.  Prints one JSON line with the card's name and power limit.

    python scripts/bench_topk10.py [--lib path/to/libonepeace_b200.so ...] [--rows 5000] [--cols 25010]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_classify_step import card  # noqa: E402


def load(path):
    lib = ctypes.CDLL(path)
    fn = lib.opb_topk10_rows
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    return fn


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--lib", action="append", default=None, help="extension build to time (repeatable)")
    p.add_argument("--rows", type=int, default=5000)
    p.add_argument("--cols", type=int, default=25010)
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--repeat", type=int, default=15)
    p.add_argument("--warmup", type=int, default=10)
    a = p.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from one_peace_b200 import _lib
    libs = a.lib or [_lib.LIB_PATH]
    fns = [load(os.path.abspath(x)) for x in libs]
    R, C = a.rows, a.cols
    sim = torch.randn(R, C, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    stream = torch.cuda.current_stream().cuda_stream
    idx = [torch.empty(R, 10, dtype=torch.int32, device="cuda") for _ in fns]
    val = [torch.empty(R, 10, device="cuda") for _ in fns]

    def launch(i):
        assert fns[i](sim.data_ptr(), C, idx[i].data_ptr(), val[i].data_ptr(), R, C, stream) == 0

    for i in range(len(fns)):
        for _ in range(a.warmup):
            launch(i)
    torch.cuda.synchronize()
    want = sim.topk(10, dim=1)
    for i in range(len(fns)):
        assert torch.equal(idx[i].long(), want.indices) and torch.equal(val[i], want.values), f"{libs[i]}: wrong top-10"
    times = [[] for _ in fns]
    ev = torch.cuda.Event
    for _ in range(a.repeat):
        for i in range(len(fns)):                       # alternate the builds window by window
            s, e = ev(enable_timing=True), ev(enable_timing=True)
            s.record()
            for _ in range(a.iters):
                launch(i)
            e.record()
            torch.cuda.synchronize()
            times[i].append(s.elapsed_time(e) / a.iters)
    nbytes = R * C * 4 + R * 10 * 8
    res = {"card": card(), "rows": R, "cols": C, "builds": []}
    for i, t in enumerate(times):
        ms = statistics.median(t)
        res["builds"].append({"lib": os.path.relpath(os.path.abspath(libs[i]), os.path.dirname(HERE)), "median_ms": round(ms, 4),
                              "min_ms": round(min(t), 4), "max_ms": round(max(t), 4), "GB_per_s": round(nbytes / ms / 1e6, 1)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
