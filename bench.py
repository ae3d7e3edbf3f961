#!/usr/bin/env python
"""bench.py -- frames/sec of the acoustic-scoring + pass-1 beam hot path (BASELINE.json metric).

    python bench.py --gpus N --steps K --warmup W [--impl reference] [--workload tri20k]
    (N>1: launched by torch.distributed.run, one rank per GPU)

A step = one pass of the hot path over one batch of synthetic utterances on every rank:
    [H2D of the MFCC batch] -> K1 GMM state scoring -> K3 pass-1 beam -> [D2H of word trellis]
`value`  : frames/s with the feature batch already resident in HBM, results left in HBM.
`e2e`    : frames/s through the C-ABI call a host makes (jb200_decode_batch_host): pinned host
           features in, word trellis + pass-1 best out, copies inside the timed region.
`--impl reference` : the UNMODIFIED reference (oracle/_ref/jref, compiled from /root/reference by
           oracle/Makefile) decoding the same workload on the host cores, as many processes as
           there are cores; each step is a bounded sample.
Utterances shard across ranks with no data-path collective (weak scaling: fixed batch per GPU);
the only collective is the init-time NCCL broadcast of the flattened model from rank 0.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

ALG_GMM_BYTES_PER_GAUSS = 320          # SURVEY 8d: (2D+2)*4 for D=39, streamed once per launch
ALG_FLOPS_PER_GAUSS_FRAME = 162        # SURVEY 8d
ALG_BEAM_BYTES_PER_TOKEN = 180         # SURVEY 8d per surviving token per frame


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="jb200", choices=["jb200", "reference"])
    ap.add_argument("--workload", default="tri20k")
    ap.add_argument("--utts", type=int, default=0, help="utterances per GPU per step (0 = one resident wave)")
    ap.add_argument("--frames", type=int, default=1000, help="frames per utterance")
    ap.add_argument("--mode", default="exact", choices=["exact", "fast"])
    ap.add_argument("--pipe-frames", type=int, default=-1,
                    help="GMM workloads: frames per time slice of the batch pipeline (scoring of slice c+1 beside the beam of slice c); "
                         "0 = off (one launch per batch), -1 = the default of this build")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-shim-leg", action="store_true", help="skip the reference-host-with-GPU-shim point (64 files through oracle/_ref/jref_gpu)")
    ap.add_argument("--no-extra-legs", action="store_true", help="skip the 1-utterance / 16-utterance points and the short DNN-HMM leg")
    ap.add_argument("--cpu-sample-utts", type=int, default=0)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step returned (pass-1 best and, for a fixed sample of utterances, the word "
                         "trellis) as DIR/<name>.npy, so that two builds can be compared output for output")
    return ap.parse_args()


# --------------------------------------------------------------------------------------- clocks
class ClockSampler:
    FIELDS = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
              "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
              "clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.rows = []
        self.proc = None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(index), f"--query-gpu={self.FIELDS}",
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.th = threading.Thread(target=self._read, daemon=True)
            self.th.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), line.strip()))

    def stop(self, t0: float, t1: float) -> dict:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.25)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        for ts, line in self.rows:
            if ts < t0 - 0.1 or ts > t1 + 0.1:
                continue
            f = [x.strip() for x in line.split(",")]
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except Exception:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            for ts, line in self.rows[-3:]:
                f = [x.strip() for x in line.split(",")]
                try:
                    sm.append(float(f[0])); mx.append(float(f[1]))
                except Exception:
                    pass
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3), not measured"


# --------------------------------------------------------------------------------------- reference arm
def host_cpus() -> dict:
    """What this process may actually use: affinity mask and cgroup CPU quota, not os.cpu_count()."""
    info = {"cpu_count": os.cpu_count() or 1}
    try:
        info["affinity"] = len(os.sched_getaffinity(0))
    except Exception:
        info["affinity"] = info["cpu_count"]
    quota = None
    try:                                                  # cgroup v2
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            quota = float(q) / float(per)
    except Exception:
        try:                                              # cgroup v1
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                quota = q / per
        except Exception:
            pass
    info["cgroup_quota"] = quota
    tpc = 1
    try:
        sib = open("/sys/devices/system/cpu/cpu0/topology/thread_siblings_list").read().strip()
        tpc = max(1, len([x for part in sib.split(",") for x in ([part] if "-" not in part else
                                                                 range(int(part.split("-")[0]), int(part.split("-")[1]) + 1))]))
    except Exception:
        pass
    info["threads_per_core"] = tpc
    usable = info["affinity"] if quota is None else max(1, min(info["affinity"], int(quota)))
    info["usable_threads"] = usable
    return info


def ref_procs(info: dict | None = None) -> int:
    """One reference process per physical core this process may use: the decoder is single-threaded and
    memory-bound, and two processes sharing a core's hardware threads are slower in aggregate.  JB200_REF_PROCS overrides."""
    if os.environ.get("JB200_REF_PROCS"):
        return max(1, int(os.environ["JB200_REF_PROCS"]))
    info = info or host_cpus()
    # usable_threads = min(affinity, cgroup quota); physical cores inside the affinity mask = affinity / threads per core.
    # A quota smaller than the mask still lets every process have a core of its own.
    physical = max(1, info["affinity"] // info["threads_per_core"])
    return max(1, min(info["usable_threads"], physical))


def run_reference(workload_name: str, n_procs: int, n_timed: int, n_frames: int, seed: int, warm_frames: int = 100,
                  binary: str = "jref"):
    """n_procs independent reference processes, each loading the model once and decoding one short warm-up
    utterance followed by n_timed utterances of n_frames frames.  Returns per-process
    (timed frames, timed decode seconds); decode time = between PASS1_BEGIN and PASS1_END of each utterance."""
    from julius_b200 import workload
    jref = os.path.join(ROOT, "oracle", "_ref", binary)
    if not os.path.exists(jref):
        raise RuntimeError(f"oracle/_ref/{binary} is missing (built by __graft_entry__.build() where /root/reference exists)")
    m = workload.synth_model(workload_name)
    tmp = tempfile.mkdtemp(prefix="jb200_ref_")
    rng = np.random.default_rng(seed)
    procs = []
    env = dict(os.environ, JREF_QUIET="1", JREF_PER_UTT="1")
    for pi in range(n_procs):
        files = []
        for ui in range(n_timed + 1):
            fn = os.path.join(tmp, f"p{pi}_u{ui}.mfc")
            x = workload.sample_inputs(workload_name, m, 1, warm_frames if ui == 0 else n_frames, seed=int(rng.integers(1 << 30)))[0]
            workload.write_input(workload_name, fn, x)
            files.append(fn)
        args = [jref, "-dump", "/dev/null"] + workload.ref_args(workload_name)
        p = subprocess.Popen(args, stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
        p.stdin.write("\n".join(files) + "\n")
        p.stdin.close()
        procs.append(p)
    per_proc = []
    last_out = ""
    for p in procs:
        out = p.stdout.read()
        p.wait()
        last_out = f"[exit code {p.returncode}] " + out
        fr, sec = 0, 0.0
        for line in out.splitlines():
            if line.startswith("JREF_UTT"):
                kv = dict(x.split("=") for x in line.split()[1:])
                if int(kv["idx"]) >= 1:                   # idx 0 is the warm-up utterance
                    fr += int(kv["frames"]); sec += float(kv["decode_sec"])
        if fr:
            per_proc.append((fr, sec))
    for f in os.listdir(tmp):
        os.remove(os.path.join(tmp, f))
    os.rmdir(tmp)
    if not per_proc:
        raise RuntimeError("reference produced no timing lines: " + last_out[-400:].replace("\n", " | "))
    return per_proc


def reference_measure(workload_name: str, n_timed: int, n_frames: int, seed: int) -> dict:
    """The reference CPU arm, sized to the cores this process may use.  A 1-process probe gives the uncontended
    per-process rate; if the per-process rate of the full run falls below half of it the cores are oversubscribed
    (a CPU-restricted lease that affinity/cgroup do not show) and the process count is halved and the run repeated."""
    info = host_cpus()
    n = ref_procs(info)
    probe = run_reference(workload_name, 1, 1, min(n_frames, 300), seed + 7)
    probe_rate = probe[0][0] / probe[0][1]
    tried = []
    while True:
        pp = run_reference(workload_name, n, n_timed, n_frames, seed)
        frames = sum(f for f, _ in pp)
        slowest = max(s for _, s in pp)
        rates = [f / s for f, s in pp]
        per_proc = float(np.median(rates))
        tried.append({"nproc": n, "frames_per_s": frames / slowest, "frames_per_s_per_process": per_proc})
        if per_proc >= 0.5 * probe_rate or n == 1 or len(tried) >= 4 or os.environ.get("JB200_REF_PROCS"):
            break
        n = max(1, n // 2)
    best = max(tried, key=lambda r: r["frames_per_s"])
    last = tried[-1]
    # report the configuration with the highest aggregate rate among those tried (the reference's best showing)
    return {"value": best["frames_per_s"], "nproc": best["nproc"], "frames_per_s_per_process": best["frames_per_s_per_process"],
            "probe_frames_per_s_1proc": probe_rate, "oversubscribed": bool(last["frames_per_s_per_process"] < 0.5 * probe_rate),
            "tried": tried, "timed_sec_slowest_process": (n_timed * n_frames * best["nproc"]) / best["frames_per_s"],
            "cpu_count": info["cpu_count"], "affinity": info["affinity"], "cgroup_quota": info["cgroup_quota"],
            "threads_per_core": info["threads_per_core"]}


def reference_cuda_dnn(workload_name: str, n_frames: int) -> dict:
    """The only GPU code the reference ships: its CUDA DNN forward (libsent/src/phmm/calc_dnn_cuda.cu, per-frame GEMV
    kernels, 15 launches and two PCIe copies a frame, SURVEY 2a), built by oracle/Makefile as oracle/_ref/jref_cuda.
    Whole pass 1 (CUDA DNN scoring + the host's beam), 1 process and one process per usable core sharing the GPU."""
    out = {}
    for tag, n in (("1_process", 1), ("per_core", ref_procs())):
        pp = run_reference(workload_name, n, 1, n_frames, 777, binary="jref_cuda")
        out[tag] = {"nproc": n, "frames_per_s": sum(f for f, _ in pp) / max(s for _, s in pp),
                    "frames_per_s_per_process": float(np.median([f / s for f, s in pp]))}
    return out


def reference_main(a):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    upp = a.cpu_sample_utts or 1
    n_timed = a.steps * upp
    r = reference_measure(a.workload, n_timed, a.frames, 1000)
    v = r["value"]
    sample = (f"{r['nproc']} independent reference processes (one per usable physical core; affinity {r['affinity']}, "
              f"cgroup quota {r['cgroup_quota']}, cpu_count {r['cpu_count']}), each loads the model once, decodes a 100-frame warm-up "
              f"utterance and then {a.steps} steps x {upp} utterances x {a.frames} frames; decode time between PASS1_BEGIN/END, "
              f"slowest process; {r['frames_per_s_per_process']:.0f} frames/s per process (1-process probe {r['probe_frames_per_s_1proc']:.0f})")
    line = {
        "impl": "reference", "metric": "frames/sec (xRT) 20k-word triphone decode", "value": v, "unit": "frames/s",
        "xRT": v / 100.0, "n_gpus": a.gpus, "steps": a.steps, "warmup": a.warmup,
        "ms_per_step": 1000.0 * r["timed_sec_slowest_process"] / max(a.steps, 1), "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": workload_label(a.workload), "utts_per_step": r["nproc"] * upp, "frames_per_utt": a.frames,
                   "parallelism": f"{r['nproc']} independent single-threaded reference processes on the host cores"},
        "cpu_baseline": {"value": v, "unit": "frames/s", "cores": r["nproc"], "kind": "reference", "sample": sample,
                         **{k: r[k] for k in ("nproc", "cpu_count", "affinity", "cgroup_quota", "frames_per_s_per_process",
                                              "probe_frames_per_s_1proc", "oversubscribed", "tried")}},
        "e2e": {"value": v, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))
    return 0


WORKLOAD_LABELS = {
    "tri20k": "tri20k: tied-state triphone GMM 3000 states x 16 mix x 39 dim, 20k-word 2-gram (BASELINE configs[1]), beam 800, pass 1",
    "tri20k_gbeam": "tri20k_gbeam: the same triphone GMM with -gprune beam (BASELINE configs[2]), 20k-word 2-gram, beam 800, pass 1",
    "tri20k_mp": "tri20k_mp: the triphone GMM on the multipath tree (-multipath), 20k-word 2-gram, beam 800, pass 1",
    "dnn20k": "dnn20k: DNN-HMM 528 -> 7 x 2048 logistic -> 3000 states (BASELINE configs[3] shape), 20k-word 2-gram, beam 800, pass 1",
    "dnn60k_mp": "dnn60k_mp: DNN-HMM 528 -> 7 x 2048 -> 3000 states, 60k-word multipath tree, -iwsp -iwcd1 max -b 4000 (BASELINE configs[4]), pass 1",
    "mono100": "mono100: monophone GMM 16 mix x 39 dim, 100-word grammar (BASELINE configs[0])",
}


def workload_label(name: str) -> str:
    return WORKLOAD_LABELS.get(name, name)


# --------------------------------------------------------------------------------------- product arm
def fp32_peak():
    """FP32 SIMT peak for the GMM scoring roofline: the H100 SXM data sheet's dense FP32 rate (132 SMs x 128 lanes x 2 flop
    at the boost clock).  A power-limited card reaches less."""
    return 67.0, "H100 SXM data sheet, dense FP32 (67 TFLOP/s), not measured"


# frames per time slice of the batch pipeline for GMM workloads (DESIGN.md section 4, "batch pipeline")
PIPE_FRAMES_DEFAULT = 32


DUMP_SAMPLE_UTTS = 16                  # utterances whose full word trellis --dump-outputs writes
DUMP_MAX_BYTES = 48 << 20


def dump_outputs(res, out_dir: str) -> None:
    """The results of one batch as float64 arrays: per utterance (status, overflow, frames, atoms, score) and the pass-1
    best word ids (-1 padded) for all utterances; the word trellis (utterance, wid, begin, end, backscore, lscore, last)
    of a fixed seeded sample of utterances, as many of them as fit in DUMP_MAX_BYTES."""
    os.makedirs(out_dir, exist_ok=True)
    n = len(res)
    info = np.array([[r["status"], r["overflow"], r["n_frames"], len(r["atoms"]), r["score"]] for r in res], np.float64).reshape(n, 5)
    words = np.full((n, max([len(r["words"]) for r in res] + [1])), -1.0)
    for i, r in enumerate(res):
        words[i, :len(r["words"])] = r["words"]
    sample = np.sort(np.random.default_rng(0).choice(n, min(n, DUMP_SAMPLE_UTTS), replace=False))
    rows, nbytes = [], 0
    for i in sample:
        a = res[i]["atoms"]
        if nbytes + len(a) * 7 * 8 > DUMP_MAX_BYTES:
            break
        rows.append(np.stack([np.full(len(a), i), a["wid"], a["begin"], a["end"], a["backscore"], a["lscore"], a["last"]], 1).astype(np.float64))
        nbytes += len(a) * 7 * 8
    np.save(os.path.join(out_dir, "utterances.npy"), info)
    np.save(os.path.join(out_dir, "best_words.npy"), words)
    np.save(os.path.join(out_dir, "trellis_sample.npy"), np.concatenate(rows, 0) if rows else np.zeros((0, 7)))


def measure_workload(ctx, name, B, T, steps, warmup, mode="exact", want_e2e=True, n_batches=2, seed0=100, pipe_frames=0,
                     dump_dir=None):
    """W warm-up + K timed steps of one workload at B utterances x T frames per GPU; returns the measured figures.
    ctx: dict(rank, local, world, device, torch, dist).  dump_dir: write the last timed step's results there (rank 0)."""
    torch, dist = ctx["torch"], ctx["dist"]
    from julius_b200 import capi, desc, workload
    from julius_b200.dist import broadcast_blob
    rank, local, world, device = ctx["rank"], ctx["local"], ctx["world"], ctx["device"]
    if rank == 0 and not workload.ready(name):
        raise SystemExit(f"workload {name} is not prepared (run __graft_entry__.build() where the reference is available)")
    blob = workload.load_model(name) if rank == 0 else None
    blob = broadcast_blob(blob, rank, world, device)
    ds = desc.Descriptors(blob)
    use_dnn = ds.dnn is not None
    dnn = None
    if use_dnn:
        S, M_total, D = ds.n_states, 0, ds.dnn.in_dim
        am = capi.GmmScorer(ds, device=local, gmm_desc=ds.cd_only_gmm())
        dnn = capi.DnnScorer(ds, device=local)
        dnn_flops_per_frame = 2.0 * sum(int(ds.dnn.layer_in[i]) * int(ds.dnn.layer_out[i]) for i in range(ds.dnn.n_layers))
    else:
        S, M_total, D = ds.gmm.n_states, ds.gmm.n_gauss, ds.gmm.dim
        am = capi.GmmScorer(ds, device=local, mode=capi.GMM_EXACT if mode == "exact" else capi.GMM_FAST)
    probe = capi.Decoder(ds, am, max_utts=1, max_frames=8)
    resident = max(1, probe.resident_utts())       # one resident wave of thread blocks
    probe.close()
    # the pipeline is meant for where a K1 block beside three beam blocks beats a fourth beam block: GMM scoring on normal
    # trees; the multipath kernel loses more from the missing block than the overlap returns
    pipe = 0 if (use_dnn or int(ds.tree.multipath)) else max(0, pipe_frames)
    if not B:
        # the pipeline needs room for one scoring thread block beside the beam's on every SM: 3/4 of a resident wave
        B = (resident * 3) // 4 if pipe else resident
    dec = capi.Decoder(ds, am, max_utts=B, max_frames=B * T)
    if use_dnn:
        dec.attach_dnn(dnn)
    if pipe:
        dec.set_pipeline(pipe)

    # synthetic input, different per rank and batch: B DISTINCT utterances per batch (no tiling: identical blocks would
    # walk the same tree nodes, bigram rows and memo entries in step and flatter the cache hit rates)
    m = workload.synth_model(name)
    off = np.arange(B + 1, dtype=np.int32) * T
    host_batches, dev_batches = [], []
    for bi in range(n_batches):
        feats = np.concatenate(workload.sample_inputs(name, m, B, T, seed=seed0 + 17 * rank + 1000 * bi), 0)
        hb = torch.from_numpy(feats).pin_memory()
        host_batches.append(hb)
        dev_batches.append(hb.to(device))
    torch.cuda.synchronize()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    lib = capi.lib()
    offp = off.ctypes.data_as(C.POINTER(C.c_int32))

    def step_device(i):
        db = dev_batches[i % n_batches]
        capi._check(lib.jb200_decode_batch_device(dec.handle_ptr(), db.data_ptr(), offp, B), "decode_batch_device")

    def step_host(i):
        hb = host_batches[i % n_batches]
        capi._check(lib.jb200_decode_batch_host(dec.handle_ptr(), C.cast(hb.data_ptr(), C.POINTER(C.c_float)), offp, B), "decode_batch_host")

    # ---------------- value: device-resident input ----------------
    for w in range(warmup):
        step_device(w)
    barrier()
    sampler = ClockSampler(local) if rank == 0 else None
    l0 = capi.launch_count()
    t_wall0 = time.time()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    score_ms, beam_ms, busy_ms = [], [], []
    for k in range(steps):
        step_device(k)
        capi._check(lib.jb200_decoder_sync_timing(dec.handle_ptr()), "sync_timing")   # CUDA events on the decoder's stream
        tm = dec.timing()
        score_ms.append(tm["score"]); beam_ms.append(tm["beam"])
        busy_ms.append(dec.pipeline_info()["score_busy_ms"])
    pinfo = dec.pipeline_info()
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    t_wall1 = time.time()
    launches = capi.launch_count() - l0
    dev_ms = sum(score_ms) + sum(beam_ms)
    barrier()
    clocks = sampler.stop(t_wall0, t_wall1) if sampler else None
    if dump_dir and rank == 0:
        dec._last_n = B
        dump_outputs(dec.results(), dump_dir)

    # ---------------- e2e: host buffers through the C-ABI ----------------
    e2e_ms = h2d = d2h = 0
    if want_e2e:
        for w in range(max(1, min(warmup, 2))):
            step_host(w)
        barrier()
        t2 = time.perf_counter()
        for k in range(steps):
            step_host(k)
            h2d += host_batches[k % n_batches].numel() * 4
            d2h += dec.last_d2h_bytes()
        torch.cuda.synchronize()
        e2e_ms = (time.perf_counter() - t2) * 1000.0
        barrier()

    dec._last_n = B
    res = dec.results()
    phase = dec.phase_cycles(min(B, 64)).mean(0)
    n_ok = sum(1 for r in res if r["status"] == 0 and r["overflow"] == 0)
    failures = [{"utt": i, "status": r["status"], "overflow": r["overflow"]} for i, r in enumerate(res) if r["status"] != 0 or r["overflow"] != 0][:8]
    counts = dec.frame_counts(0, T)
    hs = dec.heap_stats()

    vals = torch.tensor([dev_ms, (t1 - t0) * 1000.0, e2e_ms], dtype=torch.float64, device=device)
    if world > 1:
        dist.all_reduce(vals, op=dist.ReduceOp.MAX)
    dev_ms_max, wall_ms_max, e2e_ms_max = [float(x) for x in vals.cpu()]
    out = dict(name=name, ds=ds, use_dnn=use_dnn, B=B, T=T, S=S, M_total=M_total, D=D, resident=resident, steps=steps,
               dev_ms=dev_ms_max, wall_ms=wall_ms_max, e2e_ms=e2e_ms_max, h2d=h2d, d2h=d2h, launches=int(launches),
               score_ms=float(np.mean(score_ms)), beam_ms=float(np.mean(beam_ms)), clocks=clocks, phase=phase,
               n_ok=n_ok, n_res=len(res), failures=failures, tokens_per_frame=float(counts[:, 1].mean()), created_per_frame=float(counts[:, 0].mean()),
               heap=hs, misspec=dec.misspeculations(), beam_width=int(ds.tree.beam_width), multipath=int(ds.tree.multipath),
               pipe_frames=pipe, pipe_slices=pinfo["slices"], score_busy_ms=float(np.mean(busy_ms)))
    if use_dnn:
        out["dnn_flops_per_frame"] = dnn_flops_per_frame
        out["dnn_layers"] = int(ds.dnn.n_layers); out["dnn_hidden"] = int(ds.dnn.layer_out[0])
    dec.close()
    if dnn is not None:
        dnn.close()
    am.close()
    return out


def rooflines(r, world):
    """roofline objects of one measured workload: the kernel with the larger share against HBM (the contract's
    `roofline`), and the scoring kernel against the pipe that binds it (`roofline_scoring`)."""
    B, T, S = r["B"], r["T"], r["S"]
    peak, peak_src = peaks()
    gmm_ms, bm_ms = r["score_ms"], r["beam_ms"]
    piped = r.get("pipe_slices", 1) > 1
    if piped:
        # sliced batch: score_ms is only the scoring the beam had to wait for (slice 0); the scoring kernel's own time is
        # the span its stream was busy, most of it beside the beam kernel
        gmm_ms = r["score_busy_ms"]
    gmm_bytes = r["M_total"] * ALG_GMM_BYTES_PER_GAUSS + B * T * (r["D"] * 4 + 4 * S)
    beam_bytes = B * T * r["tokens_per_frame"] * ALG_BEAM_BYTES_PER_TOKEN
    beam_name = "beam_kernel_mp" if r["multipath"] else "beam_kernel"
    score_name = "dnn_gemm_wgmma (x%d layers)" % r["dnn_layers"] if r["use_dnn"] else "gmm_score_kernel"
    if bm_ms >= gmm_ms:
        dom, dom_ms, dom_bytes = beam_name, bm_ms, beam_bytes
    else:
        dom, dom_ms, dom_bytes = score_name, gmm_ms, gmm_bytes
    ach = dom_bytes / (dom_ms / 1000.0) / 1e9
    hs = r["heap"]
    roof = {"bound": "hbm", "kernel": dom, "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
            "algorithmic_bytes": dom_bytes, "peak_source": peak_src,
            "kernel_ms": {score_name: gmm_ms, beam_name: bm_ms},
            "pipeline": ({"slices": r["pipe_slices"], "frames_per_slice": r["pipe_frames"], "scoring_exposed_ms": r["score_ms"],
                          "scoring_stream_busy_ms": r["score_busy_ms"], "beam_and_overlapped_scoring_ms": r["beam_ms"],
                          "note": "scoring of slice c+1 runs on its own stream beside the token passing of slice c; "
                                  "kernel_ms are spans, they overlap"} if piped else None),
            "beam_phase_cycles_per_frame": {n: round(float(c) / T, 1) for n, c in zip(
                ("clear", "count_atoms", "expand", "creators", "order_sort", "materialise_outprob", "beam_cut", "heap_build"), r["phase"])},
            "beam_tokens_per_frame": r["tokens_per_frame"], "beam_created_per_frame": r["created_per_frame"],
            "beam_cut": {"upward_selects": hs["upward_selects"], "closed_form": hs["closed_form"],
                         "closed_form_frac": round(hs["closed_form"] / max(hs["upward_selects"], 1), 4),
                         "closed_form_with_relocations": hs.get("closed_form_relocated", 0),
                         "replayed_extractions": hs["extractions"],
                         "replay_ticks_per_extraction": round(hs["levels"] / max(hs["extractions"], 1), 3)}}
    if r["use_dnn"]:
        pk = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
        tpeak = float(pk.get("bf16_tflops_sustained", 989.0))
        tach = B * T * r["dnn_flops_per_frame"] / (gmm_ms / 1000.0) / 1e12
        scoring = {"bound": "tensor", "kernel": score_name, "achieved": tach, "peak": tpeak, "unit": "TFLOP/s", "frac": tach / tpeak,
                   "ms": gmm_ms, "frames_per_s": B * T / (gmm_ms / 1000.0),
                   "note": "algorithmic flops (2*in*out per layer per frame); the kernel issues 3 bf16 MMAs per product term "
                           "(hi.hi+hi.lo+lo.hi) to meet the 1e-4 tolerance, so 1/3 of peak is the ceiling of this formulation",
                   "peak_source": "MEASURED_PEAKS.json bf16_tflops_sustained" if pk else "H100 SXM data sheet, dense BF16 (989 TFLOP/s), not measured"}
    else:
        fpeak, fsrc = fp32_peak()
        fach = B * T * r["M_total"] * ALG_FLOPS_PER_GAUSS_FRAME / (gmm_ms / 1000.0) / 1e12
        scoring = {"bound": "fp32", "kernel": score_name, "achieved": fach, "peak": fpeak, "unit": "TFLOP/s", "frac": fach / fpeak,
                   "ms": gmm_ms, "frames_per_s": B * T / (gmm_ms / 1000.0), "hbm_gbs": gmm_bytes / (gmm_ms / 1000.0) / 1e9,
                   "hbm_frac": gmm_bytes / (gmm_ms / 1000.0) / 1e9 / peak,
                   "note": "algorithmic flops (162 per Gaussian-frame, SURVEY 8d); a parameter record is reused for 256 frames, so the "
                           "batch kernel is FP32-issue bound, not HBM bound (ridge ~20 flop/B on an H100)",
                   "peak_source": fsrc}
    return roof, scoring


def shim_leg(name: str, n_files: int, T: int, ahead: int) -> dict:
    """What the real host gets: oracle/_ref/jref_gpu = the unmodified Julius host with the pass-1 beam externs linked to
    the GPU shim (INTEGRATION.md 3), decoding a list of n_files utterances one utterance per call, and with the shim's
    decode-ahead over the same list (JB200_FILELIST).  Rates are frames / time between PASS1_BEGIN and PASS1_END."""
    from julius_b200 import workload
    jref_gpu = os.path.join(ROOT, "oracle", "_ref", "jref_gpu")
    if not os.path.exists(jref_gpu) or name in workload.DNN_SHAPES:
        return {"unavailable": "oracle/_ref/jref_gpu not built" if not os.path.exists(jref_gpu) else "GMM workloads only"}
    m = workload.synth_model(name)
    tmp = tempfile.mkdtemp(prefix="jb200_shim_")
    feats = workload.sample_inputs(name, m, n_files, T, seed=31337)
    files = []
    for i, x in enumerate(feats):
        fn = os.path.join(tmp, f"u{i}.mfc")
        workload.write_input(name, fn, x)
        files.append(fn)
    lst = os.path.join(tmp, "files.lst")
    with open(lst, "w") as f:
        f.write("\n".join(files) + "\n")
    out = {"files": n_files, "frames_per_file": T}
    for tag, env_extra in (("one_utterance_per_call", {}), ("decode_ahead", {"JB200_FILELIST": lst, "JB200_AHEAD": str(ahead)})):
        env = dict(os.environ, JREF_QUIET="1", JB200_SHIM_VERBOSE="1", **env_extra)
        args = [jref_gpu, "-dump", "/dev/null"] + workload.ref_args(name)
        p = subprocess.run(args, input="\n".join(files) + "\n", text=True, capture_output=True, env=env)
        kv = {}
        for line in p.stdout.splitlines():
            if line.startswith("JREF_SUMMARY"):
                kv = dict(x.split("=") for x in line.split()[1:])
        if not kv:
            out[tag] = {"failed": (p.stdout[-300:] + p.stderr[-300:])}
            continue
        sec = float(kv["decode_sec"])
        out[tag] = {"decode_sec": sec, "frames_per_s": int(kv["frames"]) / sec, "ms_per_file": 1000.0 * sec / max(int(kv["utts"]), 1)}
        if env_extra:
            out[tag]["answered_from_batches"] = p.stdout.count("from_cache")
            out[tag]["batches"] = [ln.split("batch ", 1)[1] for ln in p.stdout.splitlines() if ln.startswith("JB200_SHIM batch")]
    if "frames_per_s" in out.get("decode_ahead", {}) and "frames_per_s" in out.get("one_utterance_per_call", {}):
        out["speedup"] = out["decode_ahead"]["frames_per_s"] / out["one_utterance_per_call"]["frames_per_s"]
        out["ahead"] = ahead
    for f in os.listdir(tmp):
        os.remove(os.path.join(tmp, f))
    os.rmdir(tmp)
    return out


def product_main(a):
    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != a.gpus:
        if world == 1 and a.gpus > 1:
            raise SystemExit("launch with torch.distributed.run for --gpus > 1")
    host_shim = None
    if world == 1 and not a.no_extra_legs and not a.no_shim_leg:
        # the host-with-shim point runs other processes on the same GPU: before this process creates its CUDA context
        try:
            host_shim = shim_leg(a.workload, 64, a.frames, 32)
        except Exception as e:
            host_shim = {"failed": str(e)}
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    ctx = dict(rank=rank, local=local, world=world, device=device, torch=torch, dist=dist)

    pf = PIPE_FRAMES_DEFAULT if a.pipe_frames < 0 else a.pipe_frames
    r = measure_workload(ctx, a.workload, a.utts, a.frames, a.steps, a.warmup, mode=a.mode, pipe_frames=pf, dump_dir=a.dump_outputs)
    B, T = r["B"], r["T"]
    extra = {}
    if world == 1 and not a.no_extra_legs:
        # what one host thread sees: a single utterance, and a batch of 16 (the drop-in beam shim decodes one
        # utterance per call); device-event time of scoring + beam, features resident
        for tag, b in (("latency_1utt", 1), ("batch16", 16)):
            q = measure_workload(ctx, a.workload, b, T, 3, 2, mode=a.mode, want_e2e=True)
            extra[tag] = {"utterances": b, "frames_per_utt": T, "ms_device": q["dev_ms"] / q["steps"], "ms_e2e": q["e2e_ms"] / q["steps"],
                          "frames_per_s_e2e": b * T * q["steps"] / (q["e2e_ms"] / 1000.0)}
        if r["pipe_slices"] > 1:
            # the same workload, one scoring launch then one beam launch per batch at a full resident wave: the kernels'
            # durations ALONE (in the sliced headline run they overlap and slow each other down)
            q = measure_workload(ctx, a.workload, r["resident"], T, 3, 2, mode=a.mode, want_e2e=False, pipe_frames=0)
            qroof, qscoring = rooflines(q, world)
            extra["unsliced"] = {"utts_per_gpu": q["B"], "frames_per_utt": T, "value": q["B"] * T * q["steps"] / (q["wall_ms"] / 1000.0),
                                 "unit": "frames/s", "ms_per_step": q["wall_ms"] / q["steps"], "kernel_ms": qroof["kernel_ms"],
                                 "roofline": {k: qroof[k] for k in ("kernel", "achieved", "peak", "unit", "frac", "algorithmic_bytes")},
                                 "roofline_scoring": {k: qscoring[k] for k in ("kernel", "achieved", "peak", "unit", "frac", "ms")},
                                 "beam_phase_cycles_per_frame": qroof["beam_phase_cycles_per_frame"], "decoded_ok": f"{q['n_ok']}/{q['n_res']}"}
        if host_shim is not None:
            extra["host_shim"] = host_shim
        # K2 on the driver's record: a short leg of the DNN-HMM workload (BASELINE configs[3]) unless it is the headline
        if a.workload != "dnn20k":
            from julius_b200 import workload as _w
            if _w.ready("dnn20k"):
                q = measure_workload(ctx, "dnn20k", a.utts or min(r["resident"], torch.cuda.get_device_properties(device).multi_processor_count),
                                     T, 2, 2, want_e2e=True)
                qroof, qscoring = rooflines(q, world)
                extra["dnn20k"] = {"config": {"workload": workload_label("dnn20k"), "utts_per_gpu": q["B"], "frames_per_utt": T},
                                   "value": q["B"] * T * q["steps"] / (q["wall_ms"] / 1000.0), "unit": "frames/s",
                                   "e2e": {"value": q["B"] * T * q["steps"] / (q["e2e_ms"] / 1000.0), "unit": "frames/s",
                                           "h2d_bytes_per_step": q["h2d"] // q["steps"], "d2h_bytes_per_step": q["d2h"] // q["steps"]},
                                   "roofline_scoring": qscoring, "kernel_ms": qroof["kernel_ms"], "decoded_ok": f"{q['n_ok']}/{q['n_res']}"}

    if rank == 0:
        frames_total = world * B * T * a.steps
        value = frames_total / (r["wall_ms"] / 1000.0)
        e2e = frames_total / (r["e2e_ms"] / 1000.0)
        roof, scoring = rooflines(r, world)
        if "unsliced" in extra:
            roof["alone"] = {"note": "the same kernel timed without the scoring kernel beside it (leg `unsliced`, %d utterances)" % extra["unsliced"]["utts_per_gpu"],
                             **{k: extra["unsliced"]["roofline"][k] for k in ("achieved", "frac")},
                             "ms": extra["unsliced"]["kernel_ms"].get(roof["kernel"])}
            scoring["alone"] = {k: extra["unsliced"]["roofline_scoring"][k] for k in ("achieved", "frac", "ms")}
        line = {
            "metric": "frames/sec (xRT) 20k-word triphone decode", "value": value, "unit": "frames/s", "xRT": value / 100.0,
            "n_gpus": world, "steps": a.steps, "warmup": a.warmup, "ms_per_step": r["wall_ms"] / a.steps, "device_event_ms_per_step": r["dev_ms"] / a.steps,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16x3 (scoring) + f32 (beam)" if r["use_dnn"] else "f32", "data": "synthetic",
            "config": {"workload": workload_label(a.workload) + (f"; {B} utterances x {T} frames per GPU per step" +
                                                                (", bf16x3 tensor-core arithmetic" if r["use_dnn"] else f", GMM arithmetic mode {a.mode}")),
                       "utts_per_gpu": B, "frames_per_utt": T, "resident_utts_per_gpu": r["resident"], "beam": r["beam_width"],
                       "l2": "per-step working set (score matrix %.1f GB) exceeds L2; %d distinct utterances per batch, two batches alternate" % (B * T * r["S"] * 4 / 1e9, B),
                       "parallelism": f"utterance-sharded x{world}, no per-frame collective",
                       "pipeline": (f"batch cut into {r['pipe_slices']} time slices of {r['pipe_frames']} frames: GMM scoring of slice c+1 on a second "
                                    f"stream beside the beam kernel of slice c" if r["pipe_slices"] > 1 else "off: one scoring launch, then one beam launch per batch")},
            "roofline": roof, "roofline_scoring": scoring,
            "e2e": {"value": e2e, "unit": "frames/s", "h2d_bytes_per_step": r["h2d"] // a.steps, "d2h_bytes_per_step": r["d2h"] // a.steps,
                    "ms_per_step": r["e2e_ms"] / a.steps},
            "gpu_launches": r["launches"],
            "decoded_ok": f"{r['n_ok']}/{r['n_res']}", "decode_failures": r["failures"], "heap_misspeculations": r["misspec"], "clocks": r["clocks"],
        }
        line.update(extra)
        if world == 1 and not a.no_cpu_baseline and r["use_dnn"] and os.path.exists(os.path.join(ROOT, "oracle", "_ref", "jref_cuda")):
            try:
                line["reference_cuda_dnn"] = reference_cuda_dnn(a.workload, T)
            except Exception as e:
                line["reference_cuda_dnn"] = {"failed": str(e)[-300:]}
        if world == 1 and not a.no_cpu_baseline:
            try:
                upp = a.cpu_sample_utts or 1
                rr = reference_measure(a.workload, upp, T, 4242)
                line["cpu_baseline"] = {"value": rr["value"], "unit": "frames/s", "cores": rr["nproc"], "kind": "reference",
                                        "sample": f"{rr['nproc']} reference processes (one per usable core) x {upp} utterances x {T} frames of the "
                                                  f"same workload after a 100-frame warm-up utterance; decode time between PASS1_BEGIN/END, slowest process",
                                        **{k: rr[k] for k in ("nproc", "cpu_count", "affinity", "cgroup_quota", "frames_per_s_per_process",
                                                              "probe_frames_per_s_1proc", "oversubscribed")}}
            except Exception as e:   # the bench line must still print
                line["cpu_baseline"] = {"value": None, "unit": "frames/s", "cores": 0, "kind": "reference", "sample": f"failed: {e}"}
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    args = parse()
    sys.exit(reference_main(args) if args.impl == "reference" else product_main(args))
