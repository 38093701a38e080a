"""Freezes the reference's answers for the somatic window pass in callable mode into tests/golden/somatic_callable_window_digests.json: for
each two-sample window of tests/test_zzzzzzzzzzzzz_gpu_somatic_callable.py (the seeded windows and the bench-shaped one, with and without
tier2 evidence), a digest of QSS, NQSS and the callable intervals that the reference's position_somatic_snv_call(..., true, sgt) and
SomaticCallableProcessor give on the columns of that window (callable_gen.reference_window_digest).  The columns come from one callable-mode
pass, so this needs a GPU as well as oracle/_ref (the reference tree at build time).

    python tests/golden/make_somatic_callable_window_golden.py [out.json]"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]

import callable_gen as G  # noqa: E402
import test_zzzzzzzzzzzzz_gpu_somatic_callable as T  # noqa: E402
from strelka_b200.api import Context  # noqa: E402

assert G.have_ref(), "needs oracle/_ref/libstrelka_ref_somatic_callable.so"
ctx = Context(0)
out = {}
for key, normal, tumor, loci, key_gid, forced, opts, tier2 in list(T.seeded_window_inputs()) + [T.synthetic_window_inputs(t) for t in (False, True)]:
    _, _, pb = T.callable_pass(ctx, normal, tumor, loci, key_gid, forced, opts=opts, use_tier2=tier2)
    out[key] = G.reference_window_digest(ctx.params, pb, forced, normal.report_begin)
ctx.close()
path = sys.argv[1] if len(sys.argv) > 1 else G.WINDOW_GOLDEN
with open(path, "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
print(path, len(out), "windows")
