"""TEST INFRASTRUCTURE: a stand-in for strelka_b200.api.Context on a machine without a GPU, for checking the PLUMBING of multi-kernel
device-resident pipelines (struct fields, buffer sizes, what is passed where).  "Device memory" is host memory; every `*_dev` entry
point the pipelines call is answered by the host-compiled device body of that kernel (tests/cpp/k7*_core_host.cpp) or, for the kernels
that have none (K1, K6), by the CPU oracle reading the same structs.  Nothing here is part of the product."""
import ctypes as C

import numpy as np

import reflib
from strelka_b200 import _abi as A
from strelka_b200 import api
from strelka_b200 import batch as B


class _Timing:
    kernel_ms = 0.0
    launches = 0


class _MockLib:
    def __init__(self):
        self._bufs = {}
        reflib.k7core_enumerate(None)  # builds / loads the host-compiled bodies
        self.k7 = reflib._k7core
        eb = None
        del eb

    # ---- memory
    def sx_dev_alloc(self, h, n):
        buf = np.full(int(n) + 64, 0xEE, np.uint8)  # poisoned, like device memory is not zeroed
        self._bufs[buf.ctypes.data] = buf
        return buf.ctypes.data

    def sx_dev_free(self, h, p):
        self._bufs.pop(p, None)

    def sx_memcpy_h2d(self, h, dst, src, n):
        C.memmove(dst, src, n)
        return 0

    def sx_memcpy_d2h(self, h, dst, src, n):
        C.memmove(dst, src, n)
        return 0

    # ---- host-only entries
    def sx_default_window_opts(self, batch):
        A.load().sx_default_window_opts(batch)

    # ---- kernels
    def sx_alignment_indels_dev(self, h, batch, regions, seq4, ref, kio, ki, out):
        return reflib._k7acore.k7acore_run(batch, regions, seq4, ref, kio, ki, out)

    def sx_enumerate_alignments_dev(self, h, batch, out):
        maxA = batch._obj.opts.max_alns_per_read
        return self.k7.k7core_run(batch, out, maxA)

    def sx_link_alignments_dev(self, h, batch, enum_out, n_alns, kio, ki, out):
        return reflib._k8core.k8core_run(batch, enum_out, n_alns, kio, ki, out)

    def sx_score_alignments_dev(self, h, batch, lnp):
        return reflib.oracle().ox_score_alignments(batch, lnp)

    def sx_score_indels_dev(self, h, batch, lnp, out):
        o = out._obj
        lib = reflib.oracle()
        lib.ox_score_indels.argtypes = [C.POINTER(A.SxScoreIndelsBatch)] + [C.c_void_p] * 5
        return lib.ox_score_indels(batch, lnp, o.recs, o.n_rec, o.max_aln, o.eval_aln)


    def sx_realign_gates_dev(self, h, batch, out):
        return reflib._k7acore.k7gcore_run(batch, out)

    def sx_choose_realignment_dev(self, h, batch, lnp, out):
        return reflib._k9core.k9core_run(batch, lnp, out)


class MockContext:
    def __init__(self, eb, pools):
        # load the host-compiled bodies the mock forwards to
        reflib.k7acore_prepare(eb, pools)
        out = reflib.ox_enumerate_alignments(eb)
        reflib.k8core_link(eb, out, pools.regions)
        reflib.k9core_choose(B.RealignBatch(eb, out), np.zeros(int(out.totals[0]) + 1))
        reflib._k7acore.k7gcore_run.argtypes = [C.POINTER(A.SxGateBatch), C.POINTER(A.SxGateOut)]
        self.lib = _MockLib()
        self.h = 1

    def _chk(self, rc):
        if rc != 0:
            raise api.SxError(rc, "mock")

    def timing(self):
        return _Timing()

    def last_error(self):
        return "mock"

    enumerate_alignments_dev = api._enumerate_alignments_dev
