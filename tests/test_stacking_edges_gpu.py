"""Object stacking at the edges of the dense voxel grid and of the placement rules, through the CUDA step kernel against the oracle.

The scenes of stacking_scenes.py (void columns and stacks beyond the grid, pick-ups from the void, put-downs from above the grid's top,
the building-zone and pedestal edges, an agent in the target voxel, the pick-up height rule) run on test_events_gpu.Run: engine and
oracle on the same env seeds, warps copied from the oracle.  After every tick the rewards, dones and true objectives, the whole state,
the voxel dump, the instance list, the frames (byte-exact, fast_shading 0) and the depth are compared bit for bit, and the fault word
must stay 0.  Every scene's reach clauses hold on the oracle's record (the scripts assert them), so each comparison covers the branch
the scene is named for."""
import numpy as np
import pytest

import stacking_scenes as ss
import test_events_gpu as ev

pytestmark = pytest.mark.gpu


def full_check(run, tag):
    run.checkpoint(tag)
    for e in range(run.E):
        io, ig = run.o.instances(e), run.g.instances(e)
        assert io.shape == ig.shape and np.array_equal(io.view(np.uint32), ig.view(np.uint32)), "%s env %d: instances" % (tag, e)
    assert run.g.faults() == 0, "%s: fault word %#x" % (tag, run.g.faults())


@pytest.mark.parametrize("name", sorted(ss.SCENES))
def test_scene_matches_the_oracle_every_tick(built, name):
    ctxs, ticks = ss.run_scene(name, lambda scenario, E, A, seed, params: ev.Run(scenario, E, A, seed, params=params), full_check)
    print("%s: %d ticks, reached %s" % (name, ticks, sorted({w for c in ctxs for w, _ in c.log})))


class AsyncRun(ev.Run):
    """the engine stepped through mv_step_device, synchronised and compared after every tick"""

    def step(self, acts, tag, host=True):
        import torch

        d = super().step(acts, tag, host=False)  # the oracle's tick
        masks = torch.from_numpy(np.ascontiguousarray(acts, np.int32)).cuda()
        torch.cuda.synchronize()
        self.g.step_device(masks.data_ptr())
        self.g.sync()
        assert np.array_equal(self.o.rewards().view(np.uint32), np.array(self.g.rewards()).view(np.uint32)), tag
        assert np.array_equal(self.o.dones(), np.array(self.g.dones())), tag
        assert np.array_equal(self.o.true_objectives().view(np.uint32), np.array(self.g.true_objectives()).view(np.uint32)), tag
        self.g.fetch_obs()
        return d


def test_void_stacks_through_the_asynchronous_step(built):
    """the Obstacles void-stack scene through mv_step_device"""
    ss.run_scene("void_stack_obstacles", lambda scenario, E, A, seed, params: AsyncRun(scenario, E, A, seed, params=params), full_check)


def test_pickup_height_at_action_repeat_three(built):
    """the pick-up height scene with the engine at action_repeat 3: Interact acts on each call's first tick only (the oracle mirrors
    three ticks per call, Interact on the first)"""
    import test_action_repeat_gpu as rep

    def check(run, tag):
        run.checkpoint(tag)
        assert run.g.faults() == 0, "%s: fault word %#x" % (tag, run.g.faults())

    runs = []

    def make(scenario, E, A, seed, params):
        runs.append(rep.RepeatRun(scenario, E, A, seed, params, 3))
        return runs[0]

    ctxs, _ = ss.run_scene("pickup_height_collect", make, check)
    assert runs[0].carry_events > 0
    assert {"pickup_height_1", "pickup_height_2", "pickup_height_3"} <= {w for c in ctxs for w, _ in c.log}
