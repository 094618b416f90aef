"""ctypes binding of tests/hnsw_delete_oracle.c (TEST INFRASTRUCTURE ONLY): delete_embedding restated on the CPU with the
deviations of cdb_index_delete_rows.  The delete oracle #includes the insert oracle's source, so its ig_delete_rows works on
the graph handles of tests/pyinsert.py.  The shared object is compiled on first use into a temporary directory (keyed by
the sources' contents) and links the checker library oracle/libcosdata_oracle.so."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import pyoracle as po
from tests import pyinsert

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRC = os.path.join(_HERE, "hnsw_delete_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    po.lib()   # builds oracle/libcosdata_oracle.so if needed
    h = hashlib.sha256()
    for p in (_SRC, os.path.join(_HERE, "hnsw_insert_oracle.c"), os.path.join(_ORACLE, "hnsw_build_internal.h"),
              os.path.join(_ORACLE, "cosdata_oracle.h")):
        with open(p, "rb") as f:
            h.update(f.read())
    out = os.path.join(tempfile.gettempdir(), f"cdb_delete_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(out):
        tmp = out + f".{os.getpid()}"
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-std=gnu11", "-I", _ORACLE,
                        "-I", _HERE, "-o", tmp, _SRC, "-L", _ORACLE, "-lcosdata_oracle", f"-Wl,-rpath,{_ORACLE}", "-lm"], check=True)
        os.replace(tmp, out)
    L = C.CDLL(out)
    L.ig_delete_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    _lib = L
    return L


class Graph(pyinsert.Graph):
    """pyinsert.Graph plus deletes; `deleted` is the deletion mask over the code table (grown with set_table)"""

    def set_table(self, codes, mags):
        super().set_table(codes, mags)
        old = getattr(self, "deleted", np.zeros(0, np.uint8))
        self.deleted = np.zeros(len(self.mags), np.uint8)
        self.deleted[: old.size] = old[: len(self.mags)]

    def delete(self, rows, shortlist_size=64):
        """delete_embedding for rows, one at a time in list order -> status u8[len(rows)]"""
        r = np.ascontiguousarray(rows, dtype=np.uint32)
        st = np.zeros(max(r.size, 1), np.uint8)
        lib().ig_delete_rows(self.h, r.ctypes.data, r.size, shortlist_size, self.deleted.ctypes.data, st.ctypes.data)
        return st[: r.size]
