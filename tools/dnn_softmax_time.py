"""Device time of K2's normaliser (dnn_softmax_kernel) by frame count and logit distribution.

The normaliser replays addlog_array: a serial chain of dependent table loads over the outputs that survive its drop
rule, so its cost depends on how peaked the logits are.  This runs a single-layer net whose logits are chosen per frame
(one-hot inputs select a designed column), times the kernel with torch.profiler over repeated calls, and prints one JSON
line per (logits, T).  The library is the one julius_b200.capi loads (JB200_LIB overrides it), so two builds can be
compared by running this once with each.

    python tools/dnn_softmax_time.py [--n 3000] [--frames 1,32,1024,132000] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from julius_b200 import capi, desc  # noqa: E402
from util import dnn_blob, random_prior  # noqa: E402

K = 64   # designed columns per net


def design(kind, n, rng):
    if kind == "flat":                      # every output survives the drop rule: the longest chain
        return np.zeros((n, K), np.float32)
    if kind == "broad":                     # random-init output layer
        return rng.standard_normal((n, K)).astype(np.float32)
    # peaked like a trained model: one output 10, the rest N(-4, 1), so about half lie more than 13.8 below the peak
    w = (rng.standard_normal((n, K)) - 4.0).astype(np.float32)
    w[rng.integers(0, n, K), np.arange(K)] = 10.0
    return w


def kernel_ms(scorer, x, reps):
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):
        scorer.score(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            scorer.score(x)
        torch.cuda.synchronize()
    times = [e.device_time_total / e.count for e in prof.key_averages() if "dnn_softmax_kernel" in e.key]
    if not times:
        raise SystemExit("no dnn_softmax_kernel in the trace")
    return times[0] / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3000)
    ap.add_argument("--frames", default="1,32,1024,132000")
    ap.add_argument("--kinds", default="flat,broad,peaked")
    ap.add_argument("--out", default=None, help="also append the JSON lines to DIR/dnn_softmax_time.jsonl")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    torch.cuda.init()
    dev = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    rng = np.random.default_rng(0)
    lines = []
    for kind in a.kinds.split(","):
        w = design(kind, a.n, rng)
        ds = desc.Descriptors(dnn_blob([w], [np.zeros(a.n, np.float32)], random_prior(rng, a.n)))
        scorer = capi.DnnScorer(ds)
        for T in (int(t) for t in a.frames.split(",")):
            x = np.zeros((T, K), np.float32)
            x[np.arange(T), rng.integers(0, K, T)] = 1.0
            reps = max(3, min(50, 200000 // T))
            ms = kernel_ms(scorer, x, reps)
            line = dict(kernel="dnn_softmax_kernel", logits=kind, N=a.n, T=T, reps=reps, ms=round(ms, 4),
                        us_per_frame=round(1000.0 * ms / T, 4), lib=capi.LIBPATH, device=dev, power_limit=power)
            print(json.dumps(line), flush=True)
            lines.append(line)
        scorer.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "dnn_softmax_time.jsonl"), "a") as f:
            f.writelines(json.dumps(line) + "\n" for line in lines)


if __name__ == "__main__":
    main()
