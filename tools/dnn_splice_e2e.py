"""End-to-end cost of handing a DNN-HMM decoder front-end frames (spliced on the device, jb200_dnn_set_context) instead
of spliced vectors, on the dnn20k network shape (48 x 11 = 528 inputs, 7 x 2048 logistic, 3000 states, 20k-word tree).

Four legs, each run once with spliced vectors on a context-1 DNN ("spliced") and once with frames on a context-11 DNN
("frames"):
  batch   jb200_decode_batch_host, U utterances of T decoded frames (T + 10 input frames each);
  stream  U streams fed F frames at a time until each has decoded T frames, then an end mark.
Input frames are seeded synthetic trajectories (synth.sample_dnn_input); the spliced leg gets the same frames spliced on
the host, so both legs decode the same network inputs -- the script checks that their results are bit-identical.

Per leg one JSON line: decoded frames/s from CUDA events around whole steps (a batch, or a whole utterance of feeds)
after warm-up, the bytes uploaded per step (from the shapes), and for the batch legs jb200_decoder_last_timing()[0]
(the upload, ms).  Needs an sm_90 GPU and the dnn20k workload (__graft_entry__.build()); there is no CPU path.

    python tools/dnn_splice_e2e.py [--utts 132] [--frames 1000] [--feed 10] [--steps 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from julius_b200 import capi, desc, synth, workload  # noqa: E402

CTX, FL = 11, 48


def splice(f, ctx):
    T = max(0, len(f) - ctx + 1)
    return np.concatenate([f[j:j + T] for j in range(ctx)], axis=1)


def same(a, b):
    return all(x["status"] == y["status"] and x["n_frames"] == y["n_frames"] and x["words"] == y["words"]
               and np.float32(x["score"]).view(np.uint32) == np.float32(y["score"]).view(np.uint32)
               and len(x["atoms"]) == len(y["atoms"]) and x["atoms"].tobytes() == y["atoms"].tobytes() for x, y in zip(a, b))


def timed(torch, fn, steps, warmup):
    """mean ms per call of fn, from CUDA events around each call after warmup calls"""
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.mean(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=132)
    ap.add_argument("--frames", type=int, default=1000, help="decoded frames per utterance")
    ap.add_argument("--feed", type=int, default=10, help="frames per stream feed")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dnn_splice_e2e: no CUDA device (there is no CPU path)")
    if not workload.ready("dnn20k"):
        raise SystemExit("dnn_splice_e2e: workload dnn20k is not prepared (run __graft_entry__.build())")
    ds = desc.Descriptors(workload.load_model("dnn20k"))
    assert ds.dnn.in_dim == CTX * FL
    U, T, F = a.utts, a.frames, a.feed
    N = T + CTX - 1
    rng = np.random.default_rng(a.seed)
    frames = [synth.sample_dnn_input(rng, N, FL) for _ in range(U)]
    spliced = [np.ascontiguousarray(splice(f, CTX), np.float32) for f in frames]
    host = {"frames": torch.from_numpy(np.concatenate(frames, 0)).pin_memory(),
            "spliced": torch.from_numpy(np.concatenate(spliced, 0)).pin_memory()}
    offs = {"frames": np.arange(U + 1, dtype=np.int32) * N, "spliced": np.arange(U + 1, dtype=np.int32) * T}

    am = capi.GmmScorer(ds, gmm_desc=ds.cd_only_gmm())
    decs, dnns = {}, {}
    for leg, ctx in (("spliced", 1), ("frames", CTX)):
        dnns[leg] = capi.DnnScorer(ds, context_len=ctx)
        decs[leg] = capi.Decoder(ds, am, max_utts=U, max_frames=U * T)
        decs[leg].attach_dnn(dnns[leg])
    lib = capi.lib()
    results, lines = {}, []

    # ---- batch: jb200_decode_batch_host on pinned host buffers
    for leg in ("spliced", "frames"):
        dec, hb, off = decs[leg], host[leg], offs[leg]

        def step():
            capi._check(lib.jb200_decode_batch_host(dec.handle_ptr(), C.cast(hb.data_ptr(), desc.F), off.ctypes.data_as(desc.I), U),
                        "jb200_decode_batch_host")
        ms = timed(torch, step, a.steps, a.warmup)
        dec._last_n = U
        results[("batch", leg)] = dec.results()
        width = FL if leg == "frames" else CTX * FL
        lines.append(dict(leg="batch", input=leg, utts=U, decoded_frames_per_utt=T, frames_per_s=U * T / (ms / 1000.0),
                          step_ms=ms, upload_bytes_per_step=int(off[-1]) * width * 4, h2d_ms=dec.timing()["h2d"]))

    # ---- streams: U streams, F input frames per feed each (context 1: F spliced vectors), then an end mark
    for leg in ("spliced", "frames"):
        dec = decs[leg]
        x = frames if leg == "frames" else spliced
        n_in = len(x[0])

        def utterance():
            dec.stream_open(U)
            for t in range(0, n_in, F):
                dec.stream_feed([xu[t:t + F] for xu in x])
            dec.stream_feed([None] * U, last=[1] * U)
        ms = timed(torch, utterance, a.steps, a.warmup)
        results[("stream", leg)] = [dec.stream_result(s) for s in range(U)]
        width = FL if leg == "frames" else CTX * FL
        n_feeds = (n_in + F - 1) // F
        lines.append(dict(leg="stream", input=leg, streams=U, frames_per_feed=F, decoded_frames_per_utt=T, feeds=n_feeds + 1,
                          frames_per_s=U * T / (ms / 1000.0), utterance_ms=ms, upload_bytes_per_step=U * n_in * width * 4,
                          upload_bytes_per_feed=U * F * width * 4, h2d_ms=None))

    ok = {k: same(results[(k, "spliced")], results[(k, "frames")]) for k in ("batch", "stream")}
    ok["stream_vs_batch"] = same(results[("stream", "frames")], results[("batch", "frames")])
    gpu = torch.cuda.get_device_name(0)
    try:    # the power limit is part of the numbers
        gpu += ", power limit " + subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                                                 capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        gpu += ", power limit unknown"
    for ln in lines:
        ln["gpu"] = gpu
        print(json.dumps(ln))
    print(json.dumps({"identical_results": ok, "gpu": gpu}))
    if not all(ok.values()):
        raise SystemExit("dnn_splice_e2e: the two inputs decoded differently")


if __name__ == "__main__":
    main()
