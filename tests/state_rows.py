"""Expected state-tensor rows (option "state_tensors", include/megaverse_b200.h) of one env, built from the oracle's orc_get_state and
orc_get_level dumps.  Test infrastructure only.

Every value a dump determines is given exactly, as float32 bits; `known` marks them.  What neither dump holds is left unknown (NaN, known
False): an env's positive_collected outside HexMemory, n_reward in the hex mazes and Empty, the positions of the hex mazes' reward
objects, and, for Collect and HexMemory, whether a reward object that is still in place is good or bad -- `sign_only` marks those values,
whose magnitude (1 in place, 0 collected) is known."""
import numpy as np

SCENARIO_CODES = {"towerbuilding": 0, "collect": 2, "rearrange": 3, "sokoban": 4, "hexexplore": 5, "hexmemory": 6, "empty": 7}
OBSTACLES = ("obstacleseasy", "obstaclesmedium", "obstacleshard", "obstacleswalls", "obstaclessteps", "obstacleslava", "test")
ROWS = 128
AGENT_WORDS, HEADER_WORDS, OBJECT_WORDS = 26, 8, 9  # orc_get_state: per agent, header, per object


def scenario_code(name):
    n = name.lower()
    return 1 if n in OBSTACLES else SCENARIO_CODES[n]


def parse_level(level, A):
    """the oracle's level dump: object spawn voxels, and outside TowerBuilding the reward-object voxels (the hex mazes list none)"""
    lv = np.asarray(level, dtype=np.int64)
    n_static, n_terrain, n_obj = int(lv[0]), int(lv[1]), int(lv[2])
    p = 9 + 8 * n_static + 7 * n_terrain + 3 * n_obj + 3 * A
    rewards = None
    if p < lv.size:
        n_reward = int(lv[p + 1])
        rewards = lv[p + 2:p + 2 + 3 * n_reward].reshape(n_reward, 3)
    return n_obj, rewards


def expected_rows(name, A, state, level):
    """(rows, known, sign_only): dicts of float32 arrays agents [A,16], envs [16], objects [128,4], rewards [128,4] and bool masks"""
    sc = scenario_code(name)
    st = np.asarray(state, dtype=np.float32)
    f32 = np.float32
    agents = np.full((A, 16), np.nan, dtype=np.float32)
    for a in range(A):
        g = st[HEADER_WORDS + AGENT_WORDS * a:HEADER_WORDS + AGENT_WORDS * (a + 1)]
        # pos, basis 0 2 6 8, cur_x, hvel, vvel, was_on_ground, was_jumping, carrying, total_reward
        agents[a] = [g[0], g[1], g[2], g[3], g[5], g[9], g[11], g[21], g[12], g[13], g[14], g[15], g[18], g[19], g[22], g[23]]
    n_obj = int(st[5])
    _, reward_voxels = parse_level(level, A)
    base = HEADER_WORDS + AGENT_WORDS * A
    objects = np.zeros((ROWS, 4), dtype=np.float32)
    O = st[base:base + OBJECT_WORDS * n_obj].reshape(n_obj, OBJECT_WORDS)
    objects[:n_obj, :3] = O[:, :3]
    objects[:n_obj, 3] = O[:, 6]
    tail = st[base + OBJECT_WORDS * n_obj:]
    solved, reached = (tail[0], tail[1]) if sc != 0 else (f32(0), f32(0))
    alive = np.zeros(96, dtype=bool)
    if sc != 0:
        for w in range(3):
            word = int(tail[2 + 2 * w]) | (int(tail[3 + 2 * w]) << 24)
            alive[32 * w:32 * (w + 1)] = [(word >> b) & 1 for b in range(32)]
    hex_like = sc in (5, 6, 7)
    if sc == 0:
        n_reward = 0
    elif sc == 5:
        n_reward = 1
    elif hex_like:
        n_reward = None
    else:
        n_reward = len(reward_voxels)
    envs = np.full(16, np.nan, dtype=np.float32)
    envs[[0, 1, 2]] = st[[0, 1, 2]]
    envs[3], envs[4] = sc, n_obj
    envs[5] = np.nan if n_reward is None else n_reward
    envs[6] = solved
    # reached_exit: the oracle's word is the agents' exit bits (Rearrange: the best match count); HexMemory reports goodObjectsCollected there
    envs[7] = np.nan if sc == 6 else reached
    envs[8], envs[9] = st[3], st[4]
    envs[10] = reached if sc == 6 else (f32(0) if sc in (0, 1, 3, 5, 7) else np.nan)  # Collect, Sokoban: not in the dumps
    envs[11:] = 0
    rewards = np.zeros((ROWS, 4), dtype=np.float32)
    sign_only = {"rewards": np.zeros((ROWS, 4), dtype=bool)}
    rknown = np.ones((ROWS, 4), dtype=bool)
    nr = ROWS if n_reward is None else n_reward
    if n_reward is None:  # HexMemory / Empty: how many there are is not in the dumps
        rknown[:] = False
        rknown[:96, 3] = True
        sign_only["rewards"][:96, 3] = True
    for r in range(min(nr, 96) if n_reward is not None else 96):
        rewards[r, 3] = 1.0 if alive[r] else 0.0
    if n_reward:
        if sc in (1, 2):  # Obstacles / Collect: addDiamond at the voxel, translate(x + 0.5, y + 0.7 / 0.8, z + 0.5)
            dy = f32(0.8) if sc == 2 else f32(0.7)
            v = reward_voxels.astype(np.float32)
            rewards[:n_reward, 0] = v[:, 0] + f32(0.5)
            rewards[:n_reward, 1] = v[:, 1] + dy
            rewards[:n_reward, 2] = v[:, 2] + f32(0.5)
        else:
            rknown[:n_reward, :3] = False
        if sc in (2, 6):
            sign_only["rewards"][:n_reward, 3] = True
    rknown[96:nr, 3] = False  # the oracle's alive words cover 96 objects
    known = {"agents": ~np.isnan(agents), "envs": ~np.isnan(envs), "objects": np.ones((ROWS, 4), dtype=bool), "rewards": rknown}
    rows = {"agents": np.nan_to_num(agents), "envs": np.nan_to_num(envs), "objects": objects, "rewards": rewards}
    sign_only.update({"agents": np.zeros((A, 16), dtype=bool), "envs": np.zeros(16, dtype=bool), "objects": np.zeros((ROWS, 4), dtype=bool)})
    return rows, known, sign_only


def compare(tag, got, want, known, sign_only):
    """bit-for-bit on the known values (magnitude only where sign_only); got: one env's rows as the engine wrote them"""
    for k in ("agents", "envs", "objects", "rewards"):
        g = np.asarray(got[k], dtype=np.float32)
        w, kn, so = want[k], known[k], sign_only[k]
        exact = kn & ~so
        gb, wb = g.view(np.uint32), w.view(np.uint32)
        bad = exact & (gb != wb)
        if bad.any():
            idx = np.argwhere(bad)[:4]
            raise AssertionError("%s: %s differs at %s: engine %s, oracle %s" % (tag, k, idx.tolist(), g[bad][:4], w[bad][:4]))
        bad = kn & so & (np.abs(g) != w)
        if bad.any():
            raise AssertionError("%s: %s magnitude differs at %s" % (tag, k, np.argwhere(bad)[:4].tolist()))
