"""ctypes loader of libhx_callers.so — the C++ host harness (host/hx_callers.cpp over host/vector_index.hpp) that plays the
reference's calling pattern: N concurrent callers, one query per call (read_index.rs:81-101)."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

_LIB = None
MODES = {"blocking": 0, "tasks": 1, "direct": 2}


class CallersReport(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("seconds", "qps", "mean_us", "p50_us", "p90_us", "p99_us", "max_us")] + \
               [("completed", C.c_uint64), ("errors", C.c_uint64)]

    def as_dict(self):
        return {n: (round(float(getattr(self, n)), 2) if t is C.c_double else int(getattr(self, n))) for n, t in self._fields_}


def load():
    global _LIB
    if _LIB is None:
        from . import load_library
        load_library()   # libhelix_b200.so first (the harness links against it)
        p = Path(__file__).resolve().parent / "libhx_callers.so"
        if not p.exists():
            raise RuntimeError(f"{p} is missing: run helix-db_b200/build.sh")
        L = C.CDLL(str(p))
        L.hx_callers_run.restype = C.c_int
        L.hx_callers_run.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_float), C.c_size_t, C.c_uint32,
                                     C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_double, C.POINTER(C.c_uint64),
                                     C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(CallersReport)]
        L.hx_callers_run_restricted.restype = C.c_int
        L.hx_callers_run_restricted.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_size_t, C.c_uint32,
                                                C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_void_p,
                                                C.c_uint32, C.c_uint32, C.c_int, C.c_double, C.POINTER(C.c_uint64),
                                                C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(CallersReport)]
        _LIB = L
    return _LIB


def run(service, index, queries, k, ef, n_callers, mode="blocking", n_threads=0, seconds=1.0):
    """Drive `n_callers` concurrent one-query callers for ~`seconds`.  Returns (report dict, ids[nq,k], scores, counts):
    the answer recorded for every query index (each query is answered at least once)."""
    L = load()
    q = np.ascontiguousarray(queries, dtype=np.float32)
    nq, dim = q.shape
    ids = np.zeros((nq, k), dtype=np.uint64)
    sc = np.zeros((nq, k), dtype=np.float32)
    cnt = np.zeros(nq, dtype=np.uint32)
    rep = CallersReport()
    rc = L.hx_callers_run(service.h if service is not None else None, index.h if index is not None else None, ef,
                          q.ctypes.data_as(C.POINTER(C.c_float)), nq, dim, k, n_callers, n_threads, MODES[mode], seconds,
                          ids.ctypes.data_as(C.POINTER(C.c_uint64)), sc.ctypes.data_as(C.POINTER(C.c_float)),
                          cnt.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(rep))
    d = rep.as_dict()
    d.update(mode=mode, callers=n_callers, threads=(n_threads if mode == "tasks" else n_callers), rc=rc)
    return d, ids, sc, cnt


def run_restricted(service, index, queries, k, n_callers, cand_ids=None, cand_offsets=None, sets=None, mode="blocking",
                   n_threads=0, seconds=1.0):
    """search_restricted callers: query i scans cand_ids[cand_offsets[i]:cand_offsets[i+1]], or the DeviceCandidates
    sets[i].  Modes as in run(); "direct" is one blocking B = 1 hx_search_restricted (hx_search_restricted_sets) per call.
    Returns (report dict, ids[nq,k], scores, counts)."""
    L = load()
    q = np.ascontiguousarray(queries, dtype=np.float32)
    nq, dim = q.shape
    ids = np.zeros((nq, k), dtype=np.uint64)
    sc = np.zeros((nq, k), dtype=np.float32)
    cnt = np.zeros(nq, dtype=np.uint32)
    rep = CallersReport()
    cp = op = sp = None
    if sets is not None:
        assert len(sets) == nq
        sarr = (C.c_void_p * nq)(*[s.h for s in sets])
        sp = C.cast(sarr, C.c_void_p)
    else:
        ca = np.ascontiguousarray(cand_ids, dtype=np.uint64)
        oa = np.ascontiguousarray(cand_offsets, dtype=np.uint64)
        assert oa.size == nq + 1
        cp, op = ca.ctypes.data_as(C.POINTER(C.c_uint64)), oa.ctypes.data_as(C.POINTER(C.c_uint64))
    rc = L.hx_callers_run_restricted(service.h if service is not None else None, index.h if index is not None else None,
                                     q.ctypes.data_as(C.POINTER(C.c_float)), nq, dim, k, cp, op, sp, n_callers, n_threads,
                                     MODES[mode], seconds, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                     sc.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_uint32)),
                                     C.byref(rep))
    d = rep.as_dict()
    d.update(mode=mode, callers=n_callers, threads=(n_threads if mode == "tasks" else n_callers), rc=rc)
    return d, ids, sc, cnt
