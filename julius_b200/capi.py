"""ctypes binding of libjb200.so (include/julius_b200.h) -- the product's host-side mirror.

Fails loudly when the CUDA library is missing or no H100 is visible: there is no CPU path here.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import desc as D

HERE = os.path.dirname(os.path.abspath(__file__))
# JB200_LIB (the variable the C plugin and the beam shim honour too) selects another build of the library
LIBPATH = os.environ.get("JB200_LIB") or os.path.join(HERE, "libjb200.so")

GMM_EXACT, GMM_FAST = 0, 1

ATOM_DT = np.dtype([("wid", "<i4"), ("begin", "<i4"), ("end", "<i4"),
                    ("backscore", "<f4"), ("lscore", "<f4"), ("last", "<i4")])
UTT_DT = np.dtype([("status", "<i4"), ("n_frames", "<i4"), ("n_atoms", "<i4"), ("n_words", "<i4"),
                   ("score", "<f4"), ("_pad", "<i4"), ("atom_offset", "<i8"), ("word_offset", "<i4"), ("overflow", "<i4")])

_lib = None


class Jb200Error(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIBPATH):
            raise Jb200Error(f"{LIBPATH} is missing: run `python -m julius_b200.build` (no CPU fallback exists)")
        L = C.CDLL(LIBPATH)
        L.jb200_last_error.restype = C.c_char_p
        L.jb200_launch_count.restype = C.c_int64
        vp = C.c_void_p
        L.jb200_gmm_create.argtypes = [C.POINTER(D.GmmDesc), C.c_int, C.c_int, C.POINTER(vp)]
        L.jb200_gmm_destroy.argtypes = [vp]
        for f in ("jb200_gmm_score_stride", "jb200_gmm_n_states", "jb200_gmm_n_cdsets"):
            getattr(L, f).argtypes = [vp]
        L.jb200_gmm_score_host.argtypes = [vp, D.F, C.c_int, D.F]
        L.jb200_gmm_score_rows_host.argtypes = [vp, D.F, C.c_int, D.F]
        L.jb200_gmm_score_device.argtypes = [vp, vp, C.c_int, vp, vp]
        L.jb200_gmm_cdsets_device.argtypes = [vp, vp, C.c_int, vp]
        L.jb200_gmm_gauss_host.argtypes = [vp, D.F, D.F]
        if hasattr(L, "jb200_dnn_create"):
            L.jb200_dnn_create.argtypes = [C.POINTER(D.DnnDesc), C.c_int, C.POINTER(vp)]
            L.jb200_dnn_destroy.argtypes = [vp]
            L.jb200_dnn_in_dim.argtypes = [vp]
            L.jb200_dnn_out_dim.argtypes = [vp]
            L.jb200_dnn_score_host.argtypes = [vp, D.F, C.c_int, D.F]
            L.jb200_dnn_set_context.argtypes = [vp, C.c_int]
            L.jb200_decoder_attach_dnn.argtypes = [vp, vp]
        if hasattr(L, "jb200_decoder_create"):
            L.jb200_decoder_create.argtypes = [C.POINTER(D.TreeDesc), vp, C.c_int, C.c_int, C.POINTER(vp)]
            L.jb200_decoder_destroy.argtypes = [vp]
            L.jb200_decode_batch_host.argtypes = [vp, D.F, D.I, C.c_int]
            L.jb200_decode_batch_scores_host.argtypes = [vp, D.F, D.I, C.c_int]
            L.jb200_decode_batch_device.argtypes = [vp, vp, D.I, C.c_int]
            L.jb200_decoder_fetch.argtypes = [vp]
            L.jb200_decoder_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
            L.jb200_decoder_last_timing.argtypes = [vp, D.F]
            L.jb200_decoder_frame_counts.argtypes = [vp, C.c_int, D.I, C.c_int]
            L.jb200_decoder_sync_timing.argtypes = [vp]
            L.jb200_decoder_last_d2h_bytes.argtypes = [vp]
            L.jb200_decoder_last_d2h_bytes.restype = C.c_int64
            L.jb200_decoder_resident_utts.argtypes = [vp]
            L.jb200_decoder_misspeculations.argtypes = [vp]
            L.jb200_decoder_misspeculations.restype = C.c_int64
            L.jb200_decoder_heap_stats.argtypes = [vp, C.POINTER(C.c_int64)]
            L.jb200_decoder_select_stats.argtypes = [vp, C.POINTER(C.c_int64)]
            L.jb200_decoder_relocated_selects.argtypes = [vp]
            L.jb200_decoder_relocated_selects.restype = C.c_int64
            L.jb200_decoder_cut_placement.argtypes = [vp, C.POINTER(C.c_int64)]
            L.jb200_decoder_phase_cycles.argtypes = [vp, C.POINTER(C.c_int64), C.c_int]
            U8 = C.POINTER(C.c_uint8)
            L.jb200_decoder_set_pipeline.argtypes = [vp, C.c_int]
            L.jb200_decoder_pipeline_info.argtypes = [vp, D.I, D.F]
            L.jb200_stream_open.argtypes = [vp, C.c_int]
            L.jb200_stream_restart.argtypes = [vp, C.c_int]
            L.jb200_stream_feed_host.argtypes = [vp, D.F, D.I, U8, C.c_int]
            L.jb200_stream_feed_scores_host.argtypes = [vp, D.F, D.I, U8, C.c_int]
            L.jb200_stream_status.argtypes = [vp, C.c_int, D.I, D.I, D.I]
            L.jb200_stream_partial.argtypes = [vp, C.c_int, D.I, C.c_int, D.I, D.F, D.I]
            L.jb200_stream_result.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
        if hasattr(L, "jb200_group_create"):
            U8 = C.POINTER(C.c_uint8)
            L.jb200_group_create.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(vp)]
            L.jb200_group_destroy.argtypes = [vp]
            L.jb200_group_set_active.argtypes = [vp, C.c_int, C.c_int]
            L.jb200_group_decode_batch_host.argtypes = [vp, D.F, D.I, C.c_int]
            L.jb200_group_decode_batch_device.argtypes = [vp, vp, D.I, C.c_int]
            L.jb200_group_decode_batch_scores_host.argtypes = [vp, D.F, D.I, C.c_int]
            L.jb200_group_stream_open.argtypes = [vp, C.c_int]
            L.jb200_group_stream_restart.argtypes = [vp, C.c_int]
            L.jb200_group_stream_feed_host.argtypes = [vp, D.F, D.I, U8, C.c_int]
            L.jb200_group_stream_feed_scores_host.argtypes = [vp, D.F, D.I, U8, C.c_int]
            L.jb200_group_last_timing.argtypes = [vp, D.F]
        _lib = L
    return _lib


def _check(rc: int, what: str):
    if rc != 0:
        raise Jb200Error(f"{what} failed ({rc}): {lib().jb200_last_error().decode()}")


def launch_count() -> int:
    return int(lib().jb200_launch_count())


def _f(a):
    return a.ctypes.data_as(D.F)


def _utt_result(u, pa: int, pw: int) -> dict:
    """one jb200_utt_result as a dict; its atoms and words are copied from the atom base pa and the word base pw"""
    na, nw = int(u["n_atoms"]), int(u["n_words"])
    atoms = np.ctypeslib.as_array(C.cast(pa + int(u["atom_offset"]) * ATOM_DT.itemsize, C.POINTER(C.c_uint8)),
                                  shape=(max(na, 0) * ATOM_DT.itemsize,)).view(ATOM_DT).copy() if na > 0 else np.zeros(0, ATOM_DT)
    words = np.ctypeslib.as_array(C.cast(pw + int(u["word_offset"]) * 4, D.I), shape=(nw,)).copy().tolist() if nw > 0 else []
    return dict(status=int(u["status"]), n_frames=int(u["n_frames"]), atoms=atoms, words=words,
                score=float(u["score"]), overflow=int(u["overflow"]))


def _offsets(lengths):
    off = np.zeros(len(lengths) + 1, np.int32)
    np.cumsum(np.asarray(lengths, np.int64), out=off[1:])
    return off


def _batch(fn, h, arrays, what: str):
    """one call of a host batch entry point on the concatenated arrays and their offsets"""
    off = _offsets([len(x) for x in arrays])
    cat = np.ascontiguousarray(np.concatenate(arrays, 0), np.float32)
    _check(fn(h, _f(cat), off.ctypes.data_as(D.I), len(arrays)), what)


def _feed(fn, h, n: int, chunks, last, interim: bool, what: str):
    """one call of a stream feed entry point: the chunks packed stream-major, their counts and the end flags"""
    dim = None
    for c in chunks:
        if c is not None and len(c):
            dim = c.shape[1]
    n_new = np.array([0 if c is None else len(c) for c in chunks], np.int32)
    parts = [np.asarray(c, np.float32) for c in chunks if c is not None and len(c)]
    cat = np.ascontiguousarray(np.concatenate(parts, 0)) if parts else np.zeros((1, dim or 1), np.float32)
    lastv = np.zeros(n, np.uint8) if last is None else np.asarray(last, np.uint8)
    _check(fn(h, _f(cat), n_new.ctypes.data_as(D.I), lastv.ctypes.data_as(C.POINTER(C.c_uint8)), 1 if interim else 0), what)


class GmmScorer:
    """All-state GMM scoring on the GPU (outprob_state/calc_mix/gprune_*/addlog_array/outprob_cd)."""

    def __init__(self, ds: D.Descriptors, device: int = 0, mode: int = GMM_EXACT, gmm_desc=None):
        self.ds = ds
        self._h = C.c_void_p()
        g = gmm_desc if gmm_desc is not None else ds.gmm
        _check(lib().jb200_gmm_create(C.byref(g), device, mode, C.byref(self._h)), "jb200_gmm_create")
        self.n_states = lib().jb200_gmm_n_states(self._h)
        self.n_cdsets = lib().jb200_gmm_n_cdsets(self._h)
        self.stride = lib().jb200_gmm_score_stride(self._h)
        self.dim = g.dim

    @property
    def handle(self):
        return self._h

    def score(self, feats: np.ndarray) -> np.ndarray:
        feats = np.ascontiguousarray(feats, np.float32)
        T = feats.shape[0]
        out = np.empty((T, self.n_states), np.float32)
        _check(lib().jb200_gmm_score_host(self._h, _f(feats), T, _f(out)), "jb200_gmm_score_host")
        return out

    def score_rows(self, feats: np.ndarray) -> np.ndarray:
        feats = np.ascontiguousarray(feats, np.float32)
        T = feats.shape[0]
        out = np.empty((T, self.stride), np.float32)
        _check(lib().jb200_gmm_score_rows_host(self._h, _f(feats), T, _f(out)), "jb200_gmm_score_rows_host")
        return out

    def score_device(self, d_feats_ptr: int, T: int, d_rows_ptr: int, stream: int = 0):
        _check(lib().jb200_gmm_score_device(self._h, d_feats_ptr, T, d_rows_ptr, stream or None), "jb200_gmm_score_device")

    def gauss(self, feat: np.ndarray) -> np.ndarray:
        feat = np.ascontiguousarray(feat, np.float32)
        out = np.empty(self.ds.gmm.n_gauss, np.float32)
        _check(lib().jb200_gmm_gauss_host(self._h, _f(feat), _f(out)), "jb200_gmm_gauss_host")
        return out

    def close(self):
        if self._h:
            lib().jb200_gmm_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DnnScorer:
    """DNN-HMM forward on the tensor cores (dnn_calc_outprob).  With context_len > 1 (the dnnconf's context_len) the
    network input is spliced on the device: score(), and the Decoder it is attached to, take front-end frames
    in_dim / context_len wide, and N frames give max(0, N - context_len + 1) decoded frames."""

    def __init__(self, ds: D.Descriptors, device: int = 0, context_len: int = 1):
        self.ds = ds
        self._h = C.c_void_p()
        _check(lib().jb200_dnn_create(C.byref(ds.dnn), device, C.byref(self._h)), "jb200_dnn_create")
        self.in_dim = lib().jb200_dnn_in_dim(self._h)
        self.out_dim = lib().jb200_dnn_out_dim(self._h)
        if context_len != 1:
            _check(lib().jb200_dnn_set_context(self._h, context_len), "jb200_dnn_set_context")
        self.context_len = context_len
        self.frame_len = self.in_dim // context_len

    @property
    def handle(self):
        return self._h

    def score(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, np.float32)
        N = x.shape[0]
        out = np.empty((max(0, N - self.context_len + 1), self.out_dim), np.float32)
        _check(lib().jb200_dnn_score_host(self._h, _f(x), N, _f(out)), "jb200_dnn_score_host")
        return out

    def close(self):
        if self._h:
            lib().jb200_dnn_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Decoder:
    """Batched pass-1 decoder (get_back_trellis_* / outprob_style / factoring lookups on the GPU)."""

    def __init__(self, ds: D.Descriptors, am: GmmScorer, max_utts: int, max_frames: int):
        self.ds, self.am = ds, am
        self._h = C.c_void_p()
        _check(lib().jb200_decoder_create(C.byref(ds.tree), am.handle, max_utts, max_frames, C.byref(self._h)),
               "jb200_decoder_create")
        self.dnn = None

    def attach_dnn(self, dnn: "DnnScorer"):
        _check(lib().jb200_decoder_attach_dnn(self._h, dnn.handle), "jb200_decoder_attach_dnn")
        self.dnn = dnn

    def decode(self, feats_list):
        """feats_list: list of [T_u, dim] arrays (host; front-end frames [N_u, frame_len] when the attached DNN splices).
        Returns list of result dicts."""
        _batch(lib().jb200_decode_batch_host, self._h, feats_list, "jb200_decode_batch_host")
        self._last_n = len(feats_list)
        return self.results()

    def decode_scores(self, scores_list):
        _batch(lib().jb200_decode_batch_scores_host, self._h, scores_list, "jb200_decode_batch_scores_host")
        self._last_n = len(scores_list)
        return self.results()

    def decode_device(self, d_feats_ptr: int, frame_off: np.ndarray, fetch: bool = True):
        frame_off = np.ascontiguousarray(frame_off, np.int32)
        _check(lib().jb200_decode_batch_device(self._h, d_feats_ptr, frame_off.ctypes.data_as(D.I), len(frame_off) - 1),
               "jb200_decode_batch_device")
        self._last_n = len(frame_off) - 1
        if fetch:
            _check(lib().jb200_decoder_fetch(self._h), "jb200_decoder_fetch")

    def raw_results(self):
        pu, pa, pw = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _check(lib().jb200_decoder_results(self._h, C.byref(pu), C.byref(pa), C.byref(pw)), "jb200_decoder_results")
        return pu.value, pa.value, pw.value

    def results(self, n_utts: int | None = None):
        pu, pa, pw = self.raw_results()
        n = self._last_n if n_utts is None else n_utts
        utts = np.ctypeslib.as_array(C.cast(pu, C.POINTER(C.c_uint8)), shape=(n * UTT_DT.itemsize,)).view(UTT_DT)
        return [_utt_result(u, pa, pw) for u in utts]

    # the *_host entry points remember the batch size for results()
    _last_n = 0

    # ---- batch pipeline: scoring of time slice c+1 beside the token passing of slice c
    def set_pipeline(self, frames_per_slice: int):
        _check(lib().jb200_decoder_set_pipeline(self._h, int(frames_per_slice)), "jb200_decoder_set_pipeline")

    def pipeline_info(self) -> dict:
        n, ms = C.c_int32(0), C.c_float(0)
        _check(lib().jb200_decoder_pipeline_info(self._h, C.byref(n), C.byref(ms)), "jb200_decoder_pipeline_info")
        return {"slices": int(n.value), "score_busy_ms": float(ms.value)}

    # ---- frame-synchronous operation (jb200_stream_*): the call sequence get_back_trellis_init/_proceed/_end
    def stream_open(self, n_streams: int = 1):
        _check(lib().jb200_stream_open(self._h, n_streams), "jb200_stream_open")
        self._st_n = n_streams

    def stream_restart(self, stream: int):
        _check(lib().jb200_stream_restart(self._h, stream), "jb200_stream_restart")

    def stream_feed(self, chunks, last=None, interim: bool = False, scores: bool = False):
        """chunks: one [n_new, dim] array (or None / empty) per stream; last: per-stream end-of-utterance flags."""
        fn = lib().jb200_stream_feed_scores_host if scores else lib().jb200_stream_feed_host
        _feed(fn, self._h, self._st_n, chunks, last, interim, "jb200_stream_feed")

    def stream_status(self, stream: int) -> dict:
        a, b, c = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        _check(lib().jb200_stream_status(self._h, stream, C.byref(a), C.byref(b), C.byref(c)), "jb200_stream_status")
        return {"frames": int(a.value), "alive": bool(b.value), "ended": bool(c.value)}

    def stream_partial(self, stream: int) -> dict:
        w = np.zeros(160, np.int32)
        n, sc, fr = C.c_int32(0), C.c_float(0), C.c_int32(0)
        _check(lib().jb200_stream_partial(self._h, stream, w.ctypes.data_as(D.I), 160, C.byref(n), C.byref(sc), C.byref(fr)),
               "jb200_stream_partial")
        return {"words": w[:n.value].tolist(), "score": float(sc.value), "frame": int(fr.value)}

    def stream_result(self, stream: int) -> dict:
        pu, pa, pw = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _check(lib().jb200_stream_result(self._h, stream, C.byref(pu), C.byref(pa), C.byref(pw)), "jb200_stream_result")
        u = np.ctypeslib.as_array(C.cast(pu.value, C.POINTER(C.c_uint8)), shape=(UTT_DT.itemsize,)).view(UTT_DT)[0]
        return _utt_result(u, pa.value, pw.value)

    def handle_ptr(self):
        return self._h

    def last_d2h_bytes(self) -> int:
        return int(lib().jb200_decoder_last_d2h_bytes(self._h))

    def misspeculations(self) -> int:
        return int(lib().jb200_decoder_misspeculations(self._h))

    def heap_stats(self) -> dict:
        """beam-cut replay counters since create"""
        v = (C.c_int64 * 3)()
        _check(lib().jb200_decoder_heap_stats(self._h, v), "jb200_decoder_heap_stats")
        w = (C.c_int64 * 2)()
        _check(lib().jb200_decoder_select_stats(self._h, w), "jb200_decoder_select_stats")
        return {"fallbacks": int(v[0]), "levels": int(v[1]), "extractions": int(v[2]),
                "upward_selects": int(w[0]), "closed_form": int(w[1]),
                "closed_form_relocated": int(lib().jb200_decoder_relocated_selects(self._h))}

    def cut_placement(self) -> dict:
        """where the heap-select array lives, and the replays of a global-memory heap since create by copy strategy"""
        v = (C.c_int64 * 3)()
        _check(lib().jb200_decoder_cut_placement(self._h, v), "jb200_decoder_cut_placement")
        return {"heap_global": bool(v[0]), "whole_copy_replays": int(v[1]), "top_tail_replays": int(v[2])}

    def resident_utts(self) -> int:
        return int(lib().jb200_decoder_resident_utts(self._h))

    def phase_cycles(self, n_utts: int) -> np.ndarray:
        c = np.zeros((n_utts, 8), np.int64)
        _check(lib().jb200_decoder_phase_cycles(self._h, c.ctypes.data_as(C.POINTER(C.c_int64)), n_utts), "jb200_decoder_phase_cycles")
        return c

    def timing(self):
        ms = np.zeros(4, np.float32)
        _check(lib().jb200_decoder_last_timing(self._h, _f(ms)), "jb200_decoder_last_timing")
        return dict(h2d=float(ms[0]), score=float(ms[1]), beam=float(ms[2]), d2h=float(ms[3]))

    def frame_counts(self, u: int, T: int):
        c = np.zeros((T, 2), np.int32)
        _check(lib().jb200_decoder_frame_counts(self._h, u, c.ctypes.data_as(D.I), T), "jb200_decoder_frame_counts")
        return c

    def close(self):
        if self._h:
            lib().jb200_decoder_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DecoderGroup:
    """Recognition instances on one acoustic model (Julius multi-decoding): each batch or stream feed is scored once and
    decoded by every active member.  Per-member results come from the members' own Decoder methods (results(),
    stream_status(), stream_partial(), stream_result()).  Close the group before its members."""

    def __init__(self, decoders):
        self.members = list(decoders)
        self._h = C.c_void_p()
        hs = (C.c_void_p * max(len(self.members), 1))(*[d.handle_ptr() for d in self.members])
        _check(lib().jb200_group_create(hs, len(self.members), C.byref(self._h)), "jb200_group_create")
        self._active = [True] * len(self.members)
        self._st_n = 0                  # until stream_open: the library refuses a feed

    def set_active(self, member: int, active: bool):
        _check(lib().jb200_group_set_active(self._h, member, 1 if active else 0), "jb200_group_set_active")
        self._active[member] = bool(active)

    def _results(self, n):
        for d, a in zip(self.members, self._active):
            if a:
                d._last_n = n
        return [d.results() if a else None for d, a in zip(self.members, self._active)]

    def decode(self, feats_list):
        """-> one list of result dicts per member (None for an inactive member)"""
        _batch(lib().jb200_group_decode_batch_host, self._h, feats_list, "jb200_group_decode_batch_host")
        return self._results(len(feats_list))

    def decode_scores(self, scores_list):
        _batch(lib().jb200_group_decode_batch_scores_host, self._h, scores_list, "jb200_group_decode_batch_scores_host")
        return self._results(len(scores_list))

    def decode_device(self, d_feats_ptr: int, frame_off: np.ndarray, fetch: bool = True):
        frame_off = np.ascontiguousarray(frame_off, np.int32)
        n = len(frame_off) - 1
        _check(lib().jb200_group_decode_batch_device(self._h, d_feats_ptr, frame_off.ctypes.data_as(D.I), n),
               "jb200_group_decode_batch_device")
        for d, a in zip(self.members, self._active):
            if a:
                d._last_n = n
                if fetch:
                    _check(lib().jb200_decoder_fetch(d.handle_ptr()), "jb200_decoder_fetch")

    def stream_open(self, n_streams: int = 1):
        _check(lib().jb200_group_stream_open(self._h, n_streams), "jb200_group_stream_open")
        self._st_n = n_streams
        for d in self.members:
            d._st_n = n_streams

    def stream_restart(self, stream: int):
        _check(lib().jb200_group_stream_restart(self._h, stream), "jb200_group_stream_restart")

    def stream_feed(self, chunks, last=None, interim: bool = False, scores: bool = False):
        """as Decoder.stream_feed, for every active member"""
        fn = lib().jb200_group_stream_feed_scores_host if scores else lib().jb200_group_stream_feed_host
        _feed(fn, self._h, self._st_n, chunks, last, interim, "jb200_group_stream_feed")

    def timing(self):
        ms = np.zeros(4, np.float32)
        _check(lib().jb200_group_last_timing(self._h, _f(ms)), "jb200_group_last_timing")
        return dict(h2d=float(ms[0]), score=float(ms[1]), beams=float(ms[2]), d2h=float(ms[3]))

    def close(self):
        if self._h:
            lib().jb200_group_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
