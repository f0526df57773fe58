#!/usr/bin/env python
"""Per-pass cost of the headline transform: one lone 2^20-point f64 forward FFT through `phastft_fft_dit_f64_dev`.

Each round times `--steps` transforms replayed from a CUDA graph over 16 rotating device signals (256 MiB, more than the L2, as
in bench.py), then the per-pass device times of `--profile` calls of `phastft_fft_dit_f64_dev_profile`.  Prints one JSON line:
the card's name and power limit, the plan, and per round the µs per step and per pass, with the median and spread over the
rounds.  To compare two builds, run it on each in turn, alternating, in one session (PHASTFT_LIB selects the library).

    python tools/pass_times.py --rounds 5 --steps 20000 --label branch
"""
import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import phastft_b200 as pf  # noqa: E402
from phastft_b200 import _lib  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20000)
    ap.add_argument("--profile", type=int, default=200, help="profiled calls per round (per-pass CUDA events)")
    ap.add_argument("--label", default="")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    n, nbuf = 1 << 20, 16
    planner = pf.PlannerDit64(n, 0)
    planner.reserve(1)
    g = torch.Generator(device=dev)
    g.manual_seed(1234)
    bufs = [(torch.rand(n, dtype=torch.float64, device=dev, generator=g) * 2 - 1,
             torch.rand(n, dtype=torch.float64, device=dev, generator=g) * 2 - 1) for _ in range(nbuf)]
    f = _lib.fn("phastft_fft_dit_{s}_dev", "f64")
    fprof = _lib.fn("phastft_fft_dit_{s}_dev_profile", "f64")
    stream = torch.cuda.Stream(dev)

    def step(i):
        re, im = bufs[i % nbuf]
        _lib.check(f(planner._h, C.c_void_p(re.data_ptr()), C.c_void_p(im.data_ptr()), 1, 1, n, C.c_void_p(stream.cuda_stream)))

    with torch.cuda.stream(stream):
        for i in range(nbuf):
            step(i)
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            for i in range(nbuf):
                step(i)
        stream.synchronize()
    reps = max(1, a.steps // nbuf)
    pass_ms = (C.c_float * 3)()
    npass = C.c_int(0)
    rounds = []
    for r in range(a.rounds + 1):                  # round 0 warms up and is not reported
        with torch.cuda.stream(stream):
            for _ in range(max(1, reps // 10)):
                graph.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(reps):
                graph.replay()
            e1.record(stream)
        e1.synchronize()
        us_step = e0.elapsed_time(e1) * 1e3 / (reps * nbuf)
        acc = [0.0, 0.0, 0.0]
        for i in range(a.profile):
            re, im = bufs[i % nbuf]
            _lib.check(fprof(planner._h, C.c_void_p(re.data_ptr()), C.c_void_p(im.data_ptr()), 1, 1, n,
                             C.c_void_p(stream.cuda_stream), pass_ms, C.byref(npass)))
            for j in range(npass.value):
                acc[j] += pass_ms[j]
        if r:
            rounds.append({"us_per_step": us_step, "us_per_pass": [acc[j] * 1e3 / a.profile for j in range(npass.value)]})
    steps = [x["us_per_step"] for x in rounds]
    passes = list(zip(*[x["us_per_pass"] for x in rounds]))
    print(json.dumps({
        "label": a.label, "card": card(), "plan": planner.describe(), "steps_per_round": reps * nbuf,
        "us_per_step_median": statistics.median(steps), "us_per_step_spread": max(steps) - min(steps),
        "us_per_pass_median": [statistics.median(p) for p in passes], "us_per_pass_spread": [max(p) - min(p) for p in passes],
        "rounds": rounds}), flush=True)


if __name__ == "__main__":
    main()
