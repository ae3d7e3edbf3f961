"""Experiment driver (GPU box): one model, one set of inputs, several decoder configurations back to back.

    python tools/exp_pipeline.py [workload] [steps]

For every configuration: W warm-up + K timed batches (device-resident features, CUDA events on the decoder's streams),
the per-phase cycle counters, and a fingerprint of the results (atom count, score bits and word sequence of every
utterance) -- configurations that decode the same utterances must agree bit for bit.
"""
import ctypes as C
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from julius_b200 import capi, desc, workload


def fingerprint(res):
    h = hashlib.sha1()
    for r in res:
        h.update(np.int32(len(r["atoms"])).tobytes()); h.update(np.float32(r["score"]).tobytes())
        h.update(np.asarray(r["words"], np.int32).tobytes()); h.update(r["atoms"].tobytes())
    return h.hexdigest()[:16]


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "tri20k"
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    T = 1000
    blob = workload.load_model(name)
    ds = desc.Descriptors(blob)
    am = capi.GmmScorer(ds, device=0, mode=capi.GMM_EXACT)
    probe = capi.Decoder(ds, am, max_utts=1, max_frames=8)
    resident = probe.resident_utts(); probe.close()
    m = workload.synth_model(name)
    t0 = time.time()
    nmax = max(resident, int(os.environ.get("EXP_MAX_UTTS", "0")))
    batches = [np.concatenate(workload.sample_inputs(name, m, nmax, T, seed=100 + 1000 * bi), 0) for bi in range(2)]
    dev = [torch.from_numpy(b).cuda() for b in batches]
    print(f"# {name}: resident {resident}, inputs sampled in {time.time() - t0:.1f}s", flush=True)
    lib = capi.lib()
    # (label, utterances, pipeline frames)
    B3 = (resident * 3) // 4
    configs = [
        ("base", resident, 0),
        ("b3_pipe32", B3, 32),
        ("b3_nopipe", B3, 0),
        ("b3_pipe250", B3, 250),
        ("b3_pipe125", B3, 125),
        ("b3_pipe64", B3, 64),
        ("b4_pipe125", resident, 125),
    ]
    if len(sys.argv) > 3:
        # either names of the presets above, or explicit label:utterances:pipe_frames triples
        sel = sys.argv[3].split(",")
        if all(":" in x for x in sel):
            configs = [(x.split(":")[0], int(x.split(":")[1]), int(x.split(":")[2])) for x in sel]
        else:
            configs = [c for c in configs if c[0] in set(sel)]
    B3 = min(c[1] for c in configs)
    fps = {}
    for label, B, pipe in configs:
        dec = capi.Decoder(ds, am, max_utts=B, max_frames=B * T)
        dec.set_pipeline(pipe)
        off = (np.arange(B + 1, dtype=np.int32) * T)
        offp = off.ctypes.data_as(C.POINTER(C.c_int32))
        def step(i):
            capi._check(lib.jb200_decode_batch_device(dec.handle_ptr(), dev[i % 2].data_ptr(), offp, B), "decode")
        for w in range(2):
            step(w)
        torch.cuda.synchronize()
        sc, bm, busy = [], [], []
        t1 = time.perf_counter()
        for k in range(steps):
            step(k)
            capi._check(lib.jb200_decoder_sync_timing(dec.handle_ptr()), "sync")
            tm = dec.timing(); sc.append(tm["score"]); bm.append(tm["beam"]); busy.append(dec.pipeline_info()["score_busy_ms"])
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t1) * 1000.0 / steps
        capi._check(lib.jb200_decoder_fetch(dec.handle_ptr()), "fetch")
        dec._last_n = B
        res = dec.results()
        ok = sum(1 for r in res if r["status"] == 0 and r["overflow"] == 0)
        fp = fingerprint(res[:B3])                       # the first B3 utterances are common to every configuration
        phase = dec.phase_cycles(min(B, 64)).mean(0) / T
        out = {"config": label, "utts": B, "pipe_frames": pipe, "slices": dec.pipeline_info()["slices"], "ms_per_step": round(wall, 2),
               "frames_per_s": round(B * T / (wall / 1000.0)), "score_exposed_ms": round(float(np.mean(sc)), 2),
               "beam_ms": round(float(np.mean(bm)), 2), "score_busy_ms": round(float(np.mean(busy)), 2), "decoded_ok": f"{ok}/{B}",
               "fingerprint": fp, "phase_cycles_per_frame": [round(float(x)) for x in phase], "cut": dec.heap_stats()}
        print(json.dumps(out), flush=True)
        fps[label] = (fp, (steps - 1) % 2)
        dec.close()
    vals = {v[0] for v in fps.values()}
    print("# fingerprints", "AGREE" if len(vals) == 1 else f"DIFFER: {fps}", flush=True)


if __name__ == "__main__":
    main()
