"""What a decoder group (jb200_group_*, Julius multi-decoding) saves over separate decoders, on the bench workloads.

For each workload (tri20k: GMM; dnn20k: DNN-HMM) and N = 1, 2, 3 recognition instances -- the workload's tree at beam
widths 800, 600 and 400, all on one acoustic model -- one batch of B utterances x T frames (B = one resident wave of the
widest member), features resident in device memory, is decoded two ways:
  group     one jb200_group_decode_batch_device: the batch is scored once, then every member's beam runs on its stream;
  separate  jb200_decode_batch_device on each of the N decoders in turn (each scores the batch itself; the decoders'
            streams let the calls overlap on the device).
Per way one JSON line: ms per step and frames/s per instance (B * T / step time), from a host clock around whole steps
that end in a device synchronise, after warm-up; for the group the phase times of jb200_group_last_timing (scoring, and
beams = end of scoring to end of the last member's beam); and the device memory the way's objects hold beyond the scorer (cudaMemGetInfo before and
after they are created and warmed).  Both ways must give the same results; the script checks it.  Needs an sm_90 GPU and
the prepared workloads (__graft_entry__.build()); there is no CPU path.

    python tools/group_decode_time.py [--workloads tri20k dnn20k] [--frames 1000] [--steps 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from julius_b200 import capi, desc, workload  # noqa: E402

BEAMS = (800, 600, 400)


def timed(torch, fn, steps, warmup):
    """mean ms per call of fn after warmup calls, from a host clock around each call and the device synchronise that ends
    it (the decoders and the group work on streams of their own, which events on torch's stream would not bracket)"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1000.0)
    return float(np.mean(ms))


def same(a, b):
    return all(x["status"] == y["status"] and x["words"] == y["words"] and x["atoms"].tobytes() == y["atoms"].tobytes()
               and np.float32(x["score"]).view(np.uint32) == np.float32(y["score"]).view(np.uint32) for x, y in zip(a, b))


def variant(blob, beam):
    b = dict(blob)
    b["tree.beam_width"] = np.array([beam], b["tree.beam_width"].dtype)
    return desc.Descriptors(b)


def used(torch):
    free, total = torch.cuda.mem_get_info()
    return total - free


def run(torch, name, T, steps, warmup, seed):
    blob = workload.load_model(name)
    ds = desc.Descriptors(blob)
    dnn = None
    if ds.dnn is not None:
        am = capi.GmmScorer(ds, gmm_desc=ds.cd_only_gmm())
        dnn = capi.DnnScorer(ds)
    else:
        am = capi.GmmScorer(ds, mode=capi.GMM_EXACT)
    dss = [variant(blob, b) for b in BEAMS]
    probe = capi.Decoder(dss[0], am, max_utts=1, max_frames=8)
    B = max(1, probe.resident_utts())
    probe.close()
    feats = np.concatenate(workload.sample_inputs(name, workload.synth_model(name), B, T, seed=seed), 0)
    d_feats = torch.from_numpy(feats).cuda()
    off = np.arange(B + 1, dtype=np.int32) * T
    offp = off.ctypes.data_as(C.POINTER(C.c_int32))
    lib = capi.lib()
    # the scorers' own scratch grows on first use: let it, before any memory is counted
    warm = capi.Decoder(dss[0], am, max_utts=B, max_frames=B * T)
    if dnn is not None:
        warm.attach_dnn(dnn)
    capi._check(lib.jb200_decode_batch_device(warm.handle_ptr(), d_feats.data_ptr(), offp, B), "jb200_decode_batch_device")
    torch.cuda.synchronize()
    warm.close()
    lines = []
    for n in (1, 2, 3):
        torch.cuda.synchronize()
        m0 = used(torch)
        decs = []
        for ds_k in dss[:n]:
            d = capi.Decoder(ds_k, am, max_utts=B, max_frames=B * T)
            if dnn is not None:
                d.attach_dnn(dnn)
            decs.append(d)

        def separate():
            for d in decs:
                capi._check(lib.jb200_decode_batch_device(d.handle_ptr(), d_feats.data_ptr(), offp, B), "jb200_decode_batch_device")

        ms_sep = timed(torch, separate, steps, warmup)
        m_sep = used(torch) - m0
        want = []
        for d in decs:
            d._last_n = B
            want.append(d.results())
        g = capi.DecoderGroup(decs)
        ms_grp = timed(torch, lambda: g.decode_device(d_feats.data_ptr(), off, fetch=False), steps, warmup)
        m_grp = used(torch) - m0
        t = g.timing()
        ok = all(same(d.results(), w) for d, w in zip(decs, want))
        base = dict(workload=name, instances=n, beams=list(BEAMS[:n]), utts=B, frames_per_utt=T)
        lines.append(dict(base, way="separate", ms_per_step=ms_sep, frames_per_s_per_instance=B * T / (ms_sep / 1000.0),
                          device_mb=m_sep / 2 ** 20))
        lines.append(dict(base, way="group", ms_per_step=ms_grp, frames_per_s_per_instance=B * T / (ms_grp / 1000.0),
                          score_ms=t["score"], beams_ms=t["beams"], device_mb=m_grp / 2 ** 20, same_results=ok))
        g.close()
        for d in decs:
            d.close()
        if not ok:
            raise SystemExit(f"group_decode_time: {name} N={n}: the group's results differ from the separate decodes")
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["tri20k", "dnn20k"])
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=100)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("group_decode_time: no CUDA device (there is no CPU path)")
    for name in a.workloads:
        if not workload.ready(name):
            raise SystemExit(f"group_decode_time: workload {name} is not prepared (run __graft_entry__.build())")
    p = torch.cuda.get_device_properties(0)
    print(json.dumps(dict(device=p.name)))
    for name in a.workloads:
        for line in run(torch, name, a.frames, a.steps, a.warmup, a.seed):
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
