"""The step kernel's collision code on constructed contact cases: mv_debug_kcc runs the per-step candidate gather, warpSweep, warpRecover
and kccPlayerStep exactly as stepKernel does, one warp per case.  Every family of kcc_scenes.py must equal the oracle's serial queries
(orc_kcc_case, every collider a candidate) bit for bit -- fractions, normals, winning collider and feature, push-outs, end states --
wherever the device reports no fault, and stay within test_kcc_conformance_cpu's bound of the float64 reference.  MV_FAULT_CAND_OVERFLOW
is set exactly where more than MV_MAX_CAND colliders reach the envelope.  The envelope property: wherever the device's end state of a
controller step differs from the oracle's, MV_FAULT_ENVELOPE or MV_FAULT_CAND_OVERFLOW is set -- over the controller families and a
seeded hunt of fast states around the envelope's edge."""
import numpy as np
import pytest

import kcc_scenes as ks
import orc
from test_kcc_conformance_cpu import check_recovers, check_sweeps

pytestmark = pytest.mark.gpu

FAULTS = 16 | 32  # MV_FAULT_ENVELOPE | MV_FAULT_CAND_OVERFLOW


def run_both(cases):
    from megaverse_b200 import capi

    args = ks.pack(cases)
    return capi.kcc_cases(*args), orc.kcc_cases(*args)


def assert_bits_equal(name, cases, dev, ora):
    (di, df), (oi, of) = dev, ora
    for k in range(len(cases)):
        if di[k, 1] & FAULTS:
            continue
        assert np.array_equal(di[k, 2:6], oi[k, 2:6]), "%s case %d: device %s, oracle %s" % (name, k, di[k, 2:6], oi[k, 2:6])
        assert np.array_equal(df[k].view(np.uint32), of[k].view(np.uint32)), "%s case %d: device %s, oracle %s" % (name, k, df[k], of[k])


@pytest.mark.parametrize("family", sorted(ks.SWEEP_FAMILIES))
def test_sweep_families_equal_the_oracle(family):
    cases = ks.SWEEP_FAMILIES[family]()
    dev, ora = run_both(cases)
    assert_bits_equal(family, cases, dev, ora)
    n_over = 0
    for k, cs in enumerate(cases):
        near = int(ora[0][k, 0])  # every one of these cases keeps all its colliders within the envelope
        over = near > 96
        n_over += over
        assert bool(dev[0][k, 1] & 32) == over, "%s case %d: %d colliders, fault bits %d" % (family, k, near, dev[0][k, 1])
        assert dev[0][k, 0] == min(near, 96)
    assert n_over == (3 * 2 if family == "counts" else 0)
    if family != "decode":  # the reference's sampling is slow: the CPU file checks the decode family at a spread of counts
        check_sweeps(family, cases, *dev)


def test_envelope_extent():
    """the candidate gather keeps exactly the colliders whose grown bounds reach the envelope: 0.01 inside each face, kept; 0.01
    outside, culled (the oracle, with no envelope, sees both)"""
    from megaverse_b200 import capi

    cases = ks.family_envelope()
    out_i, _ = capi.kcc_cases(*ks.pack(cases))
    got = [int(o[0]) for o in out_i]
    want = [cs.want["candidates"] for cs in cases]
    bad = [(cs.want["envelope"], g, w) for cs, g, w in zip(cases, got, want) if g != w]
    assert not bad, bad


def test_recovery_family_equals_the_oracle():
    cases = ks.family_recover()
    dev, ora = run_both(cases)
    assert not (dev[0][:, 1] & FAULTS).any()
    assert_bits_equal("recover", cases, dev, ora)
    check_recovers(cases, *dev)


def check_envelope_property(name, cases):
    dev, ora = run_both(cases)
    di, df = dev
    oi, of = ora
    silent, flagged = [], 0
    for k in range(len(cases)):
        same = np.array_equal(df[k].view(np.uint32), of[k].view(np.uint32)) and np.array_equal(di[k, 2:6], oi[k, 2:6])
        if di[k, 1] & FAULTS:
            flagged += 1
        elif not same:
            silent.append(k)
    assert not silent, "%s: %d silent differences, first case %d: device %s / %s, oracle %s / %s" % (
        name, len(silent), silent[0], di[silent[0]], df[silent[0]], oi[silent[0]], of[silent[0]])
    return flagged


def test_controller_families_equal_the_oracle():
    cases = ks.family_steps()
    flagged = check_envelope_property("steps", cases)
    assert flagged < len(cases) // 2


def test_envelope_hunt():
    """fast states and colliders around the envelope's edge: no silent difference, and the hunt does reach the envelope's fault"""
    cases = ks.hunt_steps(4000, seed=7)
    flagged = check_envelope_property("hunt", cases)
    assert flagged > 0


# ------------------------------------------------------------------------------------------------ the real step kernel in real levels
FWD, LEFT, JUMP = 1 << 3, 1 << 1, 1 << 7
CONTACT_SCENARIOS = [("ObstaclesHard", 1), ("ObstaclesWalls", 1), ("ObstaclesSteps", 1), ("Sokoban", 1), ("HexExplore", 1),
                     ("HexMemory", 1), ("Collect", 4)]


def warp_into_contact(run, e, rng):
    """agent 0 next to a random box of the level (a wall, a step, a seam, a maze junction), facing it; in Collect the other agents
    cluster round it and agent 0 starts on top of agent 1.  Returns the action masks to hold."""
    from test_events_gpu import yaw_towards

    inst = run.o.instances(e)
    boxes = inst[(inst[:, 0] == 0) & (np.abs(inst[:, 2 + 12]) < 400)]
    m = boxes[rng.integers(len(boxes)), 2:]
    th = rng.uniform(0, 2 * np.pi)
    r = rng.uniform(0.4, 1.6)
    x, z = m[12] + r * np.cos(th), m[14] + r * np.sin(th)
    y = m[13] + rng.choice([0.2, 1.2, 2.0])
    run.warp(e, 0, x, y, z, yaw_towards(m[12] - x, m[14] - z))
    if run.A > 1:
        for a in range(1, run.A):
            run.warp(e, a, x + 0.7 * np.cos(th + a), y, z + 0.7 * np.sin(th + a), rng.uniform(0, 2 * np.pi))
        ag1 = run.agent(e, 1)
        run.warp(e, 0, ag1[0] + 0.1, ag1[1] + 1.8, ag1[2], yaw_towards(m[12] - x, m[14] - z))
    hold = [FWD, FWD | JUMP, FWD | LEFT, FWD | LEFT | JUMP]
    return [int(hold[rng.integers(4)]) for _ in range(run.A)]


def test_constructed_contacts_in_real_levels_lockstep():
    """agents warped against walls, seams, steps, ledges, rotated maze-wall junctions and (Collect, four agents) onto another agent hold
    move and jump actions for 30 ticks in bit-for-bit lockstep with the oracle; the step kernel's own candidate count (profile slot 12,
    agent 0) shows that some of these runs take the sweep's multi-chunk path, more than 32 candidates"""
    from test_events_gpu import Run

    rng = np.random.default_rng(11)
    max_nc = {}
    for scenario, A in CONTACT_SCENARIOS:
        E = 4
        run = Run(scenario, E, A, seed=1234, coverage=False, team_spirit=[0.0] * A)
        try:
            run.g.step_profile(True, False)
            for rnd in range(3):
                hold = [warp_into_contact(run, e, rng) for e in range(E)]
                run.checkpoint("%s round %d after warps" % (scenario, rnd), frames=False)
                for t in range(30):
                    acts = np.array([hold[e][a] for e in range(E) for a in range(A)], dtype=np.int32)
                    run.step(acts, "%s round %d t=%d" % (scenario, rnd, t))
                    prof = run.g.step_profile(True, True)
                    max_nc[scenario] = max(max_nc.get(scenario, 0), int(prof[:, 12].max()))
                run.checkpoint("%s round %d end" % (scenario, rnd), frames=False)
            assert run.g.faults() == 0
        finally:
            run.close()
    print("agent 0's candidates, most in one step:", max_nc)
    assert max(max_nc.values()) > 32, max_nc
