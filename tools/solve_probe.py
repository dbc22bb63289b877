"""Timing of the triangular-solve step alone (b = 4096): the library's DMMA kernel vs cusolverDnDpotrs, for the right-hand-side
counts of the 1/2/4/8-GPU column-sharded solve."""
import ctypes as C
import json
import sys

import numpy as np

sys.path.insert(0, ".")
import keystone_b200 as ks
from keystone_b200._capi import check, lib

n = 4096
rng = np.random.default_rng(0)
A = rng.standard_normal((n + 64, n))
H = np.asfortranarray(A.T @ A + np.eye(n))
with ks.Context(0) as ctx:
    for k in (1000, 500, 250, 125):
        B = np.asfortranarray(rng.standard_normal((n, k)))
        out = {}
        for use_cusolver in (0, 1):
            X = np.empty((n, k), order="F"); ms = C.c_double(0)
            check(ctx.handle, lib().ks_debug_chol_solve(ctx.handle, H.ctypes.data_as(C.c_void_p), n, B.ctypes.data_as(C.c_void_p), k,
                                                       use_cusolver, X.ctypes.data_as(C.c_void_p), C.byref(ms)))
            out["potrs_ms" if use_cusolver else "dmma_kernel_ms"] = round(ms.value, 3)
            out["err" + str(use_cusolver)] = float(np.abs(H @ X - B).max())
        print(json.dumps({"probe": "solve", "n": n, "k": k, **out}), flush=True)
