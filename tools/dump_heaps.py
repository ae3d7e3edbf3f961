"""Test tooling: decode a few synthetic utterances of a workload with the CPU restatement (oracle/) and record
every beam cut (token count, beam width, scores in token-index order) for `beamcut --dump` (tools/beamcut.cpp).

    python tools/dump_heaps.py tri20k /tmp/hd/tri20k.heaps [n_utts] [n_frames]
"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from julius_b200 import desc as D, refdump, workload
from oracle import ffi


def main():
    name, out = sys.argv[1], sys.argv[2]
    n_utts = int(sys.argv[3]) if len(sys.argv) > 3 else 2
    T = int(sys.argv[4]) if len(sys.argv) > 4 else 300
    ds = D.Descriptors(workload.load_model(name))
    m = workload.synth_model(name)
    feats = workload.sample_inputs(name, m, n_utts, T, seed=4242)
    lib = ffi.lib()
    lib.oracle_set_heap_dump.argtypes = [C.c_char_p]
    lib.oracle_set_heap_dump(out.encode())
    for x in feats:
        st = ffi.dnn_score(ds, x) if workload.is_dnn(name) else ffi.gmm_score(ds, x)
        r = ffi.beam_decode(ds, st)
        print("decoded", len(r["atoms"]), "atoms", r["words"][:8])
    lib.oracle_set_heap_dump(b"")


if __name__ == "__main__":
    main()
