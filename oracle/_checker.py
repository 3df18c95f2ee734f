"""TEST INFRASTRUCTURE ONLY — what the checker modules (oracle.ldpc, turbo, dump, meteor, hrpt, eos, fsk, gac, xband) share: their
libraries loaded by ctypes from a signature table, the handle of one checker instance, and the loop over the pieces of a stream."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def ref_path(name):
    """oracle/_ref/libsatref_<name>.so: the checker built from the unmodified reference by oracle/Makefile"""
    return os.path.join(HERE, "_ref", f"libsatref_{name}.so")


class Library:
    """One checker's library per implementation, {impl: (path, symbol prefix)}, loaded on first use. sigs lists (name without the
    prefix, restype, argtypes). A library must export every name except those in `optional`, which are left out where missing (turbo's
    port has no encoder). Calling it returns {name: function}."""

    def __init__(self, paths, sigs, optional=()):
        self.paths, self.sigs, self.optional, self.fns = paths, sigs, optional, {}

    def available(self, impl="ref"):
        return os.path.exists(self.paths[impl][0])

    def __call__(self, impl="ref"):
        if impl not in self.fns:
            path, pfx = self.paths[impl]
            L = C.CDLL(path)
            fns = {}
            for name, res, args in self.sigs:
                if name in self.optional and not hasattr(L, pfx + name):
                    continue
                f = getattr(L, pfx + name)
                f.restype, f.argtypes = res, args
                fns[name] = f
            self.fns[impl] = fns
        return self.fns[impl]


class Handle:
    """One instance of a checker's module loop: self.h from L[kind + "_create"](*args), destroyed with L[kind + "_destroy"]."""

    def __init__(self, L, kind, *args):
        self.L, self._kind = L, kind
        self.h = L[kind + "_create"](*args)

    def __del__(self):
        if getattr(self, "h", None):
            self.L[self._kind + "_destroy"](self.h)
            self.h = None


def pieces(n, cuts=()):
    """(start, end) of the pieces that `cuts` splits [0, n) into"""
    return zip([0, *cuts], [*cuts, n])


def run_pieces(d, soft, cuts=()):
    """d.run over soft pushed in the pieces cut at `cuts`: its arrays concatenated, its other results (the stats) listed per piece."""
    rs = [d.run(soft[a:b]) for a, b in pieces(soft.size, cuts)]
    return {k: np.concatenate([r[k] for r in rs]) if isinstance(v, np.ndarray) else [r[k] for r in rs] for k, v in rs[0].items()}
