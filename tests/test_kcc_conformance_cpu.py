"""Character-controller collision queries without a GPU: the oracle's serial queries (orc_kcc_case, which the step kernel's warp-parallel
sweep, recovery and controller step equal bit for bit) against the independent float64 reference kcc_ref.py, on the constructed
families of kcc_scenes.py, each of which first proves from the reference that it reaches its case.  Plus the argument checks of the
debug entry mv_debug_kcc (they run before any device call).

Where every margin of a case (kcc_ref: graze, start on the surface, feature region, tie, slope filter, penetration threshold) clears
MARGIN, hit or miss, the winning collider and its feature must match, and |t - t_ref| * |d|, the normal and the recovery push-out must
agree within T_BOUND * 2^-24 * S, S = 1 + the largest coordinate of the winner's frame (its centre and half extents relative to the
start, and |d|): float32 rounding of coordinates of size S is 2^-24 * S per operation.  Normals are q / rho with q carrying that
error, so their error is scaled by rho.  Each family test prints its worst error in these units; the largest, 7.0, is in the features
family (boxes up to 50 units), so the bound is 32."""
import numpy as np
import pytest

import kcc_ref
import kcc_scenes as ks
import orc

T_BOUND = 32.0
MARGIN = 1e-4
EPS32 = 2.0 ** -24


def scale(case, idx):
    col = case.colliders()[idx]
    a = np.array(case.query[0:3], dtype=np.float64)
    d = np.array(case.query[3:6], dtype=np.float64) - a if case.mode == ks.SWEEP else np.zeros(3)
    return 1.0 + max(np.abs(np.array(col["c"]) - a).max() + np.abs(col["h"]).max(), np.linalg.norm(d))


def families():
    """every sweep family (the decode family at a spread of live counts: the reference samples each path, which is slow in Python)"""
    out = {k: f for k, f in ks.SWEEP_FAMILIES.items() if k != "decode"}
    out["decode"] = lambda: ks.family_decode(counts=[1, 2, 7, 16, 23, 31, 32])
    return out


def check_sweeps(name, cases, out_i, out_f):
    """reach (from the reference) and agreement within the bound where robust; returns (robust cases, worst error in 2^-24 * S)"""
    robust, worst = 0, 0.0
    for k, cs in enumerate(cases):
        r = kcc_ref.sweep(cs)
        want = cs.want
        if "index" in want and want["index"] >= 0:
            assert r["hit"] and r["index"] == cs.static_index(want["index"]), "%s case %d: reference winner %d, built for %d" % (name, k, r["index"], want["index"])
        if "feature" in want:
            assert r["feature"] == want["feature"], "%s case %d: reference feature %d, built for %d" % (name, k, r["feature"], want["feature"])
        if want.get("tie") in ("dup", "rot", "cap", "seam"):
            assert r["hit"] and r["margin"] < 1e-9, "%s case %d: not a tie" % (name, k)
        if want.get("tie") == "filtered":
            assert r["t"] == 0.0
        if "boundary" in want or want.get("slope") == "at the threshold":
            assert r["margin"] < 1e-6, "%s case %d: margin %.2g, not on the decision it was built for" % (name, k, r["margin"])
        if want.get("slope") == "filtered first":
            t_wall = kcc_ref.first_contact(cs.colliders()[0], np.array(cs.query[0:3], dtype=np.float64), np.array(cs.query[3:6], dtype=np.float64))[0]
            assert t_wall is not None and t_wall < r["t"], "%s case %d: the filtered wall is not the closest contact" % (name, k)
        if want.get("start") == "inside":
            assert kcc_ref.distance(cs.colliders()[0], np.array(cs.query[0:3], dtype=np.float64))[0] <= 0
        if r["margin"] < MARGIN or ("count" in want and want["count"] > 96):
            continue
        robust += 1
        assert bool(out_i[k, 2]) == r["hit"], "%s case %d: hit %d, reference %d" % (name, k, out_i[k, 2], r["hit"])
        if not r["hit"]:
            continue
        assert out_i[k, 3] == r["index"] and out_i[k, 4] == r["feature"], "%s case %d: collider / feature %s, reference %d / %d" % (
            name, k, out_i[k, 3:5], r["index"], r["feature"])
        S = scale(cs, r["index"])
        et = abs(float(out_f[k, 0]) - r["t"]) * r["L"] / (EPS32 * S)
        en = np.abs(out_f[k, 1:4] - r["normal"]).max() * kcc_ref.RHO_BOX / (EPS32 * S)
        worst = max(worst, et, en)
        assert et <= T_BOUND and en <= T_BOUND, "%s case %d: t off by %.1f, normal by %.1f x 2^-24 x S" % (name, k, et, en)
    return robust, worst


def check_recovers(cases, out_i, out_f):
    robust, worst = 0, 0.0
    for k, cs in enumerate(cases):
        r = kcc_ref.recover(cs)
        if "index" in cs.want:
            assert r["pen"] and r["index"] == cs.static_index(cs.want["index"])
        if cs.want["recover"] == "threshold":
            assert r["margin"] < 1e-6  # within a few float32 steps of -0.041
        if r["margin"] < MARGIN:
            continue
        robust += 1
        assert bool(out_i[k, 2]) == r["pen"] and out_i[k, 3] == r["index"], "recover case %d: %s, reference %s" % (k, out_i[k, 2:4], r)
        if r["pen"]:
            e = np.abs(out_f[k, 0:3] - r["delta"]).max() / (EPS32 * scale(cs, r["index"]))
            worst = max(worst, e)
            assert e <= T_BOUND, "recover case %d: push-out off by %.1f x 2^-24 x S" % (k, e)
    return robust, worst


@pytest.mark.parametrize("family", sorted(families()))
def test_oracle_sweep_against_the_float64_reference(family):
    cases = families()[family]()
    out_i, out_f = orc.kcc_cases(*ks.pack(cases))
    robust, worst = check_sweeps(family, cases, out_i, out_f)
    print("%s: %d of %d cases clear every margin, worst error %.1f x 2^-24 x S (bound %g)" % (family, robust, len(cases), worst, T_BOUND))
    assert robust >= 0.5 * len(cases) or family in ("starts", "ties", "boundaries", "slope"), "%s: only %d of %d cases clear every margin" % (family, robust, len(cases))


def test_oracle_recovery_against_the_float64_reference():
    cases = ks.family_recover()
    out_i, out_f = orc.kcc_cases(*ks.pack(cases))
    robust, worst = check_recovers(cases, out_i, out_f)
    print("recover: %d of %d cases clear every margin, worst error %.1f x 2^-24 x S (bound %g)" % (robust, len(cases), worst, T_BOUND))
    assert robust >= 7  # all but the cases built on a decision: the threshold, the cube's centre, coincident capsules


def test_features_family_covers_every_feature_and_yaw():
    """every one of the 23 features is built as the first contact under every yaw of the family (place_feature may skip a draw)"""
    built = {(cs.want["feature"], cs.want["yaw"]) for cs in ks.family_features()}
    missing = [(f, y) for f in range(23) for y in ks.YAWS if (f, y) not in built]
    assert not missing, missing


def test_counts_family_reaches_the_cap():
    """the counts family puts more candidates than MV_MAX_CAND near the agent, and every one of them in the sweep's path"""
    cases = ks.family_counts()
    counts = sorted({cs.want["count"] for cs in cases})
    assert counts[0] == 0 and counts[-1] > ks.MAX_OBJ - 1 and any(c == 96 for c in counts) and any(c == 97 for c in counts)
    out_i, _ = orc.kcc_cases(*ks.pack(cases))
    assert [int(o[0]) for o in out_i] == [cs.want["count"] for cs in cases]  # the oracle's colliders: all of them, no cap


def test_step_families_are_in_reach():
    """the controller families start where they say: fast states reach 60 u/s, edge walls sit 2.8 to 3.2 from the agent"""
    cases = ks.family_steps()
    kinds = {cs.want["step"] for cs in cases}
    assert kinds >= {"ledge", "corner", "graze", "junction", "ceiling", "fall", "on_agent", "embedded", "edge"}
    sp = max(np.linalg.norm(cs.query[3:6]) for cs in cases)
    assert 59.0 < sp <= 60.001
    emb = [cs for cs in cases if cs.want["step"] == "embedded"]
    for cs in emb:  # the start penetrates the big box
        assert kcc_ref.recover(cs)["pen"]


def test_debug_entry_refuses_bad_arguments():
    from megaverse_b200 import capi

    good = ks.pack([ks.Case(ks.SWEEP).sweep((0, 0, 0), (1, 0, 0))])
    bad = []
    h = good[0].copy(); h[0, 1] = ks.MAX_OBJ + 1; bad.append((h,) + good[1:])
    h = good[0].copy(); h[0, 2] = ks.MAX_OBJ + 1; bad.append((h,) + good[1:])
    h = good[0].copy(); h[0, 3] = ks.MAX_AG + 1; bad.append((h,) + good[1:])
    h = good[0].copy(); h[0, 3] = 0; bad.append((h,) + good[1:])
    h = good[0].copy(); h[0, 4] = 3; bad.append((h,) + good[1:])
    h = good[0].copy(); h[0, 5] = 1; bad.append((h,) + good[1:])
    h = good[0].copy(); h[0, 0] = 1; bad.append((h,) + good[1:])  # n_static_pre above n_static
    q = good[3].copy(); q[0, 4] = np.nan; bad.append(good[:3] + (q,))
    q = good[3].copy(); q[0, 9] = np.inf; bad.append(good[:3] + (q,))
    a = good[2].copy(); a[0, 0, 1] = np.nan; bad.append((good[0], good[1], a, good[3]))
    hb = good[0].copy(); hb[0, 1] = 1
    b = good[1].copy(); b[0, 0, 6] = 0.5; bad.append((hb, b) + good[2:])  # a flag not 0 or 1
    b = good[1].copy(); b[0, 0, 3] = -1.0; b[0, 0, 6] = 1.0; bad.append((hb, b) + good[2:])
    b = good[1].copy(); b[0, 0, 0] = np.inf; bad.append((hb, b) + good[2:])
    hs = good[0].copy(); hs[0, 4] = 2
    q = good[3].copy(); q[0, 15] = 0.0; bad.append((hs, good[1], good[2], q))  # dt 0
    for args in bad:
        with pytest.raises(capi.MegaverseError) as ei:
            capi.kcc_cases(*args)
        assert ei.value.code == capi.MV_ERR_ARG
