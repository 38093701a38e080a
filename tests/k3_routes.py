"""K3 (sx_global_align) routing restated in Python, and a seeded case generator that puts problems on every route.

Each DP problem of a batch goes down one of these paths, picked from its shape and from the batch's scores:
  group kernel     kg_align_kernel<T>, T = ceil(Q/8), four reference-length classes   Q <= 128, R <= 255, every score within +-4096
  warp kernel      register strip dp_register_strip<T>, T = ceil(Q/32) <= 4           the other problems with Q <= 128
                   shared-memory strip dp_shared_strip, T >= 5                        Q > 128
  status 2         no result: k3_slot_bytes(Q, R) exceeds the opt-in shared memory per block, or Q == 0 or R == 0 (device entry)
and the warp kernel's launch runs 4, 2 or 1 warps per CTA, whichever is the most that fit the batch's largest slot.
(k3_group.cu: kg_bucket, sx_k3_group_run; k3_global_align.cu: k3_run, k3_global_align_kernel; k3_common.cuh: k3_slot_bytes.)
test_k3_routes.py checks the constants below against those sources, so a routing change cannot leave this mirror behind.
"""
from __future__ import annotations

import numpy as np

from strelka_b200 import _abi as A

KG_MAX_Q = 128  # group kernel: longest query
KG_MAX_R = 255  # group kernel: longest reference
KG_G = 8  # group kernel: lanes per matrix
KG_RCLASSES = 4  # group kernel: reference-length classes per T (R >> 6, capped)
KG_SCORE_MAX = 4096  # group kernel: every score within +-4096 (it keeps 64 * score in 32 bits)
K3_WARPS = 4  # warp kernel: most warps per CTA
H100_SMEM_OPTIN = 232448  # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100

SCORE_FIELDS = ("match", "mismatch", "open", "extend", "offEdge", "insertDelete")


def pad16(x: int) -> int:
    return (x + 15) & ~15


def k3_slot_bytes(Q: int, R: int) -> int:
    """shared memory of one warp-kernel problem: pointer matrix, score strips, query, reference, traceback steps"""
    T = (Q + 31) // 32
    return pad16((Q + 1) * (R + 1)) + 3 * 32 * T * 4 + pad16(Q + 8) + pad16(R + 8) + pad16(Q + R + 8)


def group_kernel_allowed(scores: A.SxGaScores) -> bool:
    return all(-KG_SCORE_MAX <= getattr(scores, f) <= KG_SCORE_MAX for f in SCORE_FIELDS)


def k3_route(Q: int, R: int, scores: A.SxGaScores, smem_optin: int):
    """("group", T, rclass) | ("warp_reg", T) | ("warp_smem", T) | "status2" | "empty" """
    if Q == 0 or R == 0:
        return "empty"
    if group_kernel_allowed(scores) and Q <= KG_MAX_Q and R <= KG_MAX_R:
        return ("group", (Q + KG_G - 1) // KG_G, min(KG_RCLASSES - 1, R >> 6))
    if k3_slot_bytes(Q, R) > (smem_optin & ~15):
        return "status2"
    T = (Q + 31) // 32
    return ("warp_reg", T) if T <= 4 else ("warp_smem", T)


def route_kind(route) -> str:
    return route if isinstance(route, str) else route[0]


def k3_warp_launch_warps(shapes, scores: A.SxGaScores, smem_optin: int):
    """warps per CTA of the batch's warp-kernel launch; None when every problem goes to the group kernel"""
    large = [(Q, R) for Q, R in shapes if route_kind(k3_route(Q, R, scores, smem_optin)) != "group"]
    if not large:
        return None
    slot = pad16(max([k3_slot_bytes(Q, R) for Q, R in large if Q and R], default=0))
    warps = K3_WARPS
    while warps > 1 and slot * warps > smem_optin:
        warps >>= 1
    return warps


def reg_strip_r_last(Q: int) -> int:
    """strip-relative row of DP row Q in the last active lane of a register strip (the row whose match score feeds the backtrace)"""
    T = (Q + 31) // 32
    return (Q - 1) - ((Q - 1) // T) * T


def max_fitting_r(Q: int, smem_optin: int) -> int:
    """the longest reference a Q-base query can have and still get a warp-kernel slot"""
    R = smem_optin // (Q + 1)
    while k3_slot_bytes(Q, R) > (smem_optin & ~15):
        R -= 1
    return R


# ---------------------------------------------------------------------------------------------------------------------------------
# score sets
# ---------------------------------------------------------------------------------------------------------------------------------
def ga_scores(match, mismatch, open_, extend, off_edge, ins_del, allow_edge_ins, require_edge_del) -> A.SxGaScores:
    return A.SxGaScores(match, mismatch, open_, extend, off_edge, ins_del, int(allow_edge_ins), int(require_edge_del))


# (match, mismatch, open, extend, offEdge, insertDelete).  The +-4096 / +-4097 pairs sit on both sides of the group kernel's score
# limit: the same shapes run in the group kernel with the first and in the warp kernel's register strips with the second.
BASE_SCORES = {
    "active_region": (1, -4, -5, -1, -100, -5),  # sx_ga_active_region_scores (with both flags set)
    "golden": (2, -4, -5, -1, -4, 0),  # the reference's GlobalAlignerTest cases
    "offedge1": (2, -4, -5, -1, -1, 0),
    "open-4096": (1, -4, -4096, -1, -100, -5),
    "open-4097": (1, -4, -4097, -1, -100, -5),
    "offedge-4096": (1, -4, -5, -1, -4096, -5),
    "offedge-4097": (1, -4, -5, -1, -4097, -5),
    "match+4096": (4096, -4, -5, -1, -100, -5),
    "match+4097": (4097, -4, -5, -1, -100, -5),
}
FLAGS = ((False, False), (True, False), (False, True), (True, True))  # (isAllowEdgeInsertion, isRequireEdgeDeletion)


def score_set_ids():
    return [f"{name}-ins{int(a)}-del{int(d)}" for name in BASE_SCORES for a, d in FLAGS]


def score_set(sid: str) -> A.SxGaScores:
    name, ins, dele = sid.rsplit("-", 2)
    return ga_scores(*BASE_SCORES[name], ins == "ins1", dele == "del1")


# ---------------------------------------------------------------------------------------------------------------------------------
# sequences
# ---------------------------------------------------------------------------------------------------------------------------------
BASES = "ACGT"
KINDS = ("edited", "unrelated", "homopolymer", "tandem", "n10", "copy")


def _rand(rng, n: int) -> str:
    return "".join(BASES[i] for i in rng.integers(0, 4, n))


def _fit(rng, s: str, n: int) -> str:
    """exactly n bases of s: a random window of it, or s with random bases added at both ends"""
    if len(s) >= n:
        o = int(rng.integers(0, len(s) - n + 1))
        return s[o : o + n]
    extra = n - len(s)
    left = int(rng.integers(0, extra + 1))
    return _rand(rng, left) + s + _rand(rng, extra - left)


def _edit(rng, s: str, n_edits: int) -> str:
    q = list(s)
    for _ in range(n_edits):
        if not q:
            break
        p = int(rng.integers(0, len(q)))
        e = rng.random()
        if e < 0.4:
            q[p] = BASES[int(rng.integers(0, 4))]
        elif e < 0.7:
            del q[p : p + int(rng.integers(1, 8))]
        else:
            q[p:p] = list(_rand(rng, int(rng.integers(1, 8))))
    return "".join(q)


def _with_n(rng, s: str, frac: float) -> str:
    a = np.array(list(s))
    a[rng.random(len(s)) < frac] = "N"
    return "".join(a)


def _homopolymer(rng, n: int) -> str:
    if rng.random() < 0.4:
        return BASES[int(rng.integers(0, 4))] * n
    out = ""
    while len(out) < n:
        out += BASES[int(rng.integers(0, 4))] * int(rng.integers(3, 40))
    return out[:n]


def _tandem(rng, n: int, unit: str) -> str:
    reps = unit * (n // len(unit) + 2)
    o = int(rng.integers(0, len(unit)))
    return reps[o : o + n]


def make_pair(rng, kind: str, Q: int, R: int):
    """(query, reference) of exactly Q and R bases"""
    n_edits = int(rng.integers(0, 2 + (Q + R) // 100))
    if kind == "edited":
        r = _rand(rng, R)
        return _fit(rng, _edit(rng, r, n_edits), Q), r
    if kind == "unrelated":
        return _rand(rng, Q), _rand(rng, R)
    if kind == "homopolymer":  # ties between equally good gap placements
        r = _homopolymer(rng, R)
        q = _fit(rng, _edit(rng, r, n_edits), Q) if rng.random() < 0.5 else _homopolymer(rng, Q)
        return q, r
    if kind == "tandem":  # 2-3-base repeats: ties between gap placements one unit apart
        unit = _rand(rng, int(rng.integers(2, 4)))
        r = _tandem(rng, R, unit)
        return _fit(rng, _edit(rng, _tandem(rng, Q + 8, unit), n_edits // 2), Q), r
    if kind == "n10":  # about 10 % N on both sides: an N is a mismatch in the '='/'X' expansion, even against N
        r = _with_n(rng, _rand(rng, R), 0.1)
        return _with_n(rng, _fit(rng, _edit(rng, r, n_edits), Q), 0.1), r
    if kind == "copy":  # the query is the reference, or a window of it, or contains it
        r = _rand(rng, R)
        return _fit(rng, r, Q), r
    raise ValueError(kind)


# ---------------------------------------------------------------------------------------------------------------------------------
# shapes and batches
# ---------------------------------------------------------------------------------------------------------------------------------
GROUP_R = (1, 63, 64, 127, 128, 191, 192, 254, 255)
REG_Q = (1, 2, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128)
REG_R = (256, 300, 511, 1000, 3000)
IDENTITY_N = (1, 8, 63, 64, 128, 129, 200, 255, 256, 300, 450)  # query == reference


def group_shapes():
    return [(Q, R) for T in range(1, 17) for Q in (8 * T - 7, 8 * T) for R in GROUP_R]


def smem_shapes(rng, smem_optin: int):
    """Q at 32k-1, 32k, 32k+1 from 129 to 1023, each with the longest reference that still fits a slot, one base more (status 2),
    and a short one"""
    qs = sorted({q for k in range(4, 33) for q in (32 * k - 1, 32 * k, 32 * k + 1) if KG_MAX_Q < q <= 1023})
    out = []
    for Q in qs:
        rf = max_fitting_r(Q, smem_optin)
        out += [(Q, rf), (Q, rf + 1), (Q, int(rng.integers(1, min(rf, 400) + 1)))]
    return out


def route_batches(smem_optin: int = H100_SMEM_OPTIN, seed: int = 0):
    """{name: [(query, reference), ...]}.  "group" holds every group-kernel bucket; the warp-kernel shapes are split by the warps per
    CTA their launch gets (the largest slot of a batch sets it): "warp4", "warp2", and "warp1", which also holds the status-2
    problems.  Each warp batch carries some group-kernel problems too, so both kernels run in one call."""
    rng = np.random.default_rng(seed)
    grp = [(Q, R, None) for Q, R in group_shapes()]
    ident = [(n, n, "copy") for n in IDENTITY_N]
    warp = [(Q, R, None) for Q in REG_Q for R in REG_R] + [(Q, R, None) for Q, R in smem_shapes(rng, smem_optin)] + [s for s in ident if s[0] > KG_MAX_Q]
    shapes = {"group": grp + [s for s in ident if s[0] <= KG_MAX_Q], "warp4": [], "warp2": [], "warp1": []}
    for s in warp:
        slot = pad16(k3_slot_bytes(s[0], s[1]))
        shapes["warp4" if 4 * slot <= smem_optin else "warp2" if 2 * slot <= smem_optin else "warp1"].append(s)
    for i, name in enumerate(("warp4", "warp2", "warp1")):
        shapes[name] += grp[i::23]
    out = {}
    k = 0
    for name, shp in shapes.items():
        pairs = []
        for Q, R, kind in shp:
            pairs.append(make_pair(rng, kind or KINDS[k % len(KINDS)], Q, R))
            k += kind is None
        out[name] = pairs
    return out


def route_sample(pairs, scores: A.SxGaScores, smem_optin: int, per_route: int, seed: int):
    """a sub-batch with up to per_route problems of every route the scores give (order kept)"""
    rng = np.random.default_rng(seed)
    by = {}
    for i, (q, r) in enumerate(pairs):
        by.setdefault(k3_route(len(q), len(r), scores, smem_optin), []).append(i)
    keep = sorted(int(i) for idx in by.values() for i in rng.permutation(idx)[:per_route])
    return [pairs[i] for i in keep]


def shapes_of(pairs):
    return [(len(q), len(r)) for q, r in pairs]


def cells(pairs) -> int:
    return sum(len(q) * len(r) for q, r in pairs)
