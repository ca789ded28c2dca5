"""MegaverseEnv: the reference's Python env class (megaverse/megaverse_env.py:42-201) over the H100 engine.

Same constructor, attributes and methods, so Sample-Factory's Wrapper (megaverse_rl/megaverse_utils.py:48-88) drives it
unchanged.  The per-agent pybind loops of the reference (megaverse_env.py:121-162) are replaced by one batched call each;
the values returned are the same lists."""
import numpy as np

from .cameras import chase_views, overview_views
from .gym_shim import Box, Discrete, Env, Tuple

# the product fails loudly when its native extension is missing
from .extension.megaverse import MegaverseGym, reward_component_keys, set_megaverse_log_level  # noqa: E402

MEGAVERSE8 = ['TowerBuilding', 'ObstaclesEasy', 'ObstaclesHard', 'Collect', 'Sokoban', 'HexMemory', 'HexExplore', 'Rearrange']
OBSTACLES_MULTITASK = ['ObstaclesWalls', 'ObstaclesSteps', 'ObstaclesLava', 'ObstaclesEasy', 'ObstaclesHard']


def _multitask_tasks(multitask_name):
    assert 'multitask' in multitask_name
    if multitask_name.endswith('megaverse8'):
        return MEGAVERSE8
    elif multitask_name.endswith('obstacles'):
        return OBSTACLES_MULTITASK
    else:
        raise NotImplementedError()


def make_env_multitask(multitask_name, task_idx, num_envs, num_agents_per_env, num_simulation_threads, use_vulkan=False, params=None):
    tasks = _multitask_tasks(multitask_name)
    scenario = tasks[task_idx % len(tasks)]
    return MegaverseEnv(scenario, num_envs, num_agents_per_env, num_simulation_threads, use_vulkan, params)


def make_env_mixed(multitask_name, num_envs, num_agents_per_env, num_simulation_threads, use_vulkan=False, params=None):
    """(extension) the whole multi-task set in ONE env: env i runs tasks[i % len(tasks)], all stepped and drawn by one engine"""
    tasks = _multitask_tasks(multitask_name)
    return MegaverseEnv([tasks[i % len(tasks)] for i in range(num_envs)], num_envs, num_agents_per_env, num_simulation_threads, use_vulkan, params)


FAULT_NAMES = {1: "LEVEL_NOT_READY", 2: "TRI_OVERFLOW", 4: "GRID_RANGE", 8: "NAN", 16: "ENVELOPE", 32: "CAND_OVERFLOW"}  # csrc/mv_types.h


class MegaverseFault(RuntimeError):
    """the engine left the envelope in which its results equal the reference's (a capacity of the collision or level code was exceeded,
    a NaN position, a level that arrived late): frames, rewards and dones from here on are not trustworthy"""


class EnvState:
    """(extension) env states saved by MegaverseEnv.save_state: owns one state store of the engine that made it; row i holds env envs[i]"""

    def __init__(self, gym, store, envs):
        self._gym, self._store, self.envs = gym, store, list(envs)

    def close(self):
        if self._store is not None:
            self._gym.states_destroy(self._store)
            self._store = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001  (the engine was closed first: mv_close freed the store)
            pass


class MegaverseEnv(Env):
    # The number of static boxes of a level is unbounded, as in the reference; the remaining fixed capacities (movable objects, reward
    # objects, terrain slabs) were never exceeded on hundreds of thousands of generated levels.  Should one be, the strict default makes
    # step() / reset() fail instead of leaving the reference's level sequence; True takes the env's next level instead and counts it
    # (`levels_skipped()`, also reported in the infos).
    SKIP_UNFIT_LEVELS = False
    AUTORESET_MODES = ("same_step", "next_step", "disabled")  # option "autoreset" 0, 1, 2

    def __init__(self, scenario_name, num_envs, num_agents_per_env, num_simulation_threads, use_vulkan=False, params=None, *, final_observation=False,
                 action_repeat=1, segmentation=False, num_levels=None, start_level=0, state_tensors=False,
                 ray_directions=None, ray_max_distance=120.0, reward_components=False, autoreset_mode="same_step"):
        # (extension) a sequence of num_envs names makes a mixed batch: env i runs scenario_name[i]
        # (extension) final_observation=True: the infos of done agents also carry the frame the episode ended on ('final_observation', CHW
        # like the observations) and whether it ended terminal ('terminated': solved) or was cut off ('truncated': time limit or request)
        # (extension) action_repeat=k (1..4): every step() runs k physics ticks with the same actions (Interact on the first only) and draws
        # once; an episode end stops the ticks, and the rewards returned are each agent's sum over the ticks run (option "action_repeat")
        # (extension) segmentation=True: segmentation() gives, per agent, the class and index of the drawable behind every pixel of its
        # current observation (option "segmentation"); step()'s return values do not change
        # (extension) num_levels=L, start_level=s (Procgen's names): the envs play a fixed set of L levels per scenario, the first levels of
        # the generators seeded s .. s + L - 1, kept on the GPU (option "level_set").  level_ids() tells which level each env is on,
        # set_next_levels() chooses an env's next one, and the infos of done agents carry 'level', the level the finished episode was played on
        # (extension) state_tensors=True: state_tensors() gives the state behind the current frames (agents, envs, objects, rewards; option
        # "state_tensors"), and with final_observation=True the infos of done agents carry 'final_state', the agent's row of the state the
        # episode ended on
        # (extension) ray_directions=float32 [R, 3] (camera space: x right, y up, -z forward; megaverse_b200.rays builds fans and rings):
        # every agent casts these rays against its env's drawn scene, up to ray_max_distance; ray_observations() gives each ray's hit
        # distance and segmentation tag, and with final_observation=True the infos of done agents carry 'final_rays', the agent's rays
        # cast from the scene the episode ended on.  step()'s return values do not change
        # (extension) reward_components=True: reward_components() gives, per agent, what each shaping rule paid in the last step (columns
        # named by reward_component_keys()), and the infos of done agents carry 'reward_components', {key: the agent's total under that key
        # over the finished episode} (option "reward_components").  step()'s return values do not change
        # (extension) autoreset_mode (option "autoreset"): "same_step" is the reference's rule (a done step returns the next episode's first
        # frame).  "next_step" (EnvPool, Gymnasium >= 1.0): a done step returns the frame the episode ended on, and the env's next step runs
        # no physics, starts the next episode and returns its first frame with reward 0 and done False.  "disabled": an env that is done
        # stays on its terminal frame with reward 0 and done False until reset_envs restarts it.  Under both, the infos of done agents carry
        # 'terminated' / 'truncated' and, with num_levels, 'level' (the level the frame shows), and awaiting_reset() tells which envs wait
        if autoreset_mode not in self.AUTORESET_MODES:
            raise ValueError('autoreset_mode must be one of %s, not %r' % (', '.join(self.AUTORESET_MODES), autoreset_mode))
        if final_observation and autoreset_mode != "same_step":
            raise ValueError('final_observation needs autoreset_mode "same_step": under %r the observation of a done step is the terminal frame'
                             % autoreset_mode)
        if isinstance(scenario_name, str):
            scenario_name = scenario_name.casefold()
            self.scenarios = [scenario_name] * num_envs
        else:
            scenario_name = [s.casefold() for s in scenario_name]
            if len(scenario_name) != num_envs:
                raise ValueError('%d scenario names for %d envs' % (len(scenario_name), num_envs))
            self.scenarios = list(scenario_name)
        self.scenario_name = scenario_name
        self.is_multiagent = True
        set_megaverse_log_level(2)
        self.img_w = 128
        self.img_h = 72
        self.channels = 3
        self.use_vulkan = use_vulkan
        self.num_agents = num_envs * num_agents_per_env
        self.num_envs = num_envs
        self.num_agents_per_env = num_agents_per_env

        float_params = {}
        if params is not None:
            for k, v in params.items():
                if isinstance(v, float):
                    float_params[k] = v
                else:
                    raise Exception('Params of type %r not supported', type(v))

        self.env = MegaverseGym(self.scenario_name, self.img_w, self.img_h, num_envs, num_agents_per_env, num_simulation_threads, use_vulkan, float_params)
        if self.SKIP_UNFIT_LEVELS:
            self.env.set_option("skip_unfit_levels", 1)
        self.final_observation = bool(final_observation)
        if self.final_observation:
            self.env.set_option("final_obs", 1)
        self.segmentation_enabled = bool(segmentation)
        if self.segmentation_enabled:
            self.env.set_option("segmentation", 1)
        self.state_tensors_enabled = bool(state_tensors)
        if self.state_tensors_enabled:
            self.env.set_option("state_tensors", 1)
        self.num_rays = 0
        if ray_directions is not None:
            dirs = np.ascontiguousarray(ray_directions, dtype=np.float32).reshape(-1, 3)
            self.env.set_rays(dirs, float(ray_max_distance))
            self.num_rays = len(dirs)
        self.reward_components_enabled = bool(reward_components)
        if self.reward_components_enabled:
            self.env.set_option("reward_components", 1)
        self.autoreset_mode = autoreset_mode
        self.metadata = dict(self.metadata, autoreset_mode=autoreset_mode)
        if autoreset_mode != "same_step":
            self.env.set_option("autoreset", self.AUTORESET_MODES.index(autoreset_mode))
        self.action_repeat = int(action_repeat)
        self.env.set_option("action_repeat", self.action_repeat)
        self.num_levels = None if num_levels is None else int(num_levels)
        self._levels_played = None  # per env: the level of the episode in progress, i.e. level_ids() as of the previous call
        if self.num_levels is not None:
            if self.num_levels < 1:
                raise ValueError('num_levels must be positive')
            self.env.set_option("level_set_seed", int(start_level))
            self.env.set_option("level_set", self.num_levels)
        self.default_shaping_scheme = self.env.get_reward_shaping(0, 0)
        # each scenario's default scheme, read from its first env before anyone could change it
        self._default_shaping = {}
        for env_i, s in enumerate(self.scenarios):
            if s not in self._default_shaping:
                self._default_shaping[s] = self.env.get_reward_shaping(env_i, 0)
        self.action_space = self.generate_action_space(self.env.action_space_sizes())
        self.observation_space = Box(0, 255, (self.channels, self.img_h, self.img_w), dtype=np.uint8)

    @staticmethod
    def generate_action_space(action_space_sizes):
        return Tuple([Discrete(sz) for sz in action_space_sizes])

    def seed(self, seed=None):
        if seed is None:
            return
        assert isinstance(seed, int), 'Expect seed to be an integer'
        self.env.seed(seed)

    def observations(self):
        # one [N,h,w,4] view of engine memory -> per-agent CHW views, exactly what the reference's loop produces
        obs = self.env.get_observations()
        chw = np.transpose(obs[:, :, :, :3], (0, 3, 1, 2))
        return [chw[i] for i in range(self.num_agents)]

    def segmentation(self):
        """(extension, segmentation=True) per-agent uint16 [h, w] views, in the order of observations(): MV_SEG_* class << 8 | index of the
        drawable behind each pixel of the current frame, 0 where nothing was drawn.  Views of engine memory, valid until the next step."""
        seg = self.env.get_segmentation()
        return [seg[i] for i in range(self.num_agents)]

    def state_tensors(self):
        """(extension, state_tensors=True) {"agents": float32[num_agents, 16], "envs": float32[num_envs, 16], "objects": float32[num_envs, 128, 4],
        "rewards": float32[num_envs, 128, 4]}: the state the current observations show, rows as in include/megaverse_b200.h.  Views of engine
        memory, valid until the next step."""
        return self.env.get_state_tensors()

    def ray_observations(self):
        """(extension, ray_directions given) (dist float32[num_agents, R], tag uint16[num_agents, R]) for the current observations: the
        distance along each ray to the first front face it meets (0: none within ray_max_distance) and that drawable's MV_SEG_* class << 8 |
        index (0: none).  Views of engine memory, valid until the next step."""
        return self.env.get_rays()

    def reward_components(self):
        """(extension, reward_components=True) float32 [num_agents, 8]: column k of row i is what shaping slot k paid agent i in the last step
        (reward_component_keys(i) names the columns); the row sums to the agent's reward up to float rounding.  A view of engine memory,
        valid until the next step."""
        return self.env.get_reward_components()

    def reward_component_keys(self, actor_idx):
        """the shaping key of each column of reward_components() for agent actor_idx's scenario: 8 entries, None for column 0 (teamSpirit
        scales the other terms and pays nothing itself) and for columns the scenario does not use"""
        return reward_component_keys(self.scenarios[actor_idx // self.num_agents_per_env])

    def check_faults(self):
        """raise if the engine latched a fault bit (one pinned-memory read, no device round trip)"""
        word = self.env.fault_word()
        if word:
            names = [n for b, n in FAULT_NAMES.items() if word & b]
            raise MegaverseFault("megaverse_b200 engine fault bits 0x%x (%s)" % (word, ", ".join(names)))

    def _note_levels(self):
        if self.num_levels is not None:
            self._levels_played = [int(j) for j in self.env.level_ids()]

    def awaiting_reset(self):
        """(extension, autoreset_mode "next_step" or "disabled") per env, True where its episode is done and the next has not started"""
        return [bool(a) for a in self.env.get_awaiting_reset()]

    def level_ids(self):
        """(extension, num_levels given) per env, the level of the set it is on now (after a done: the new episode's under "same_step",
        the finished one's under the other autoreset modes)"""
        return [int(j) for j in self.env.level_ids()]

    def set_next_levels(self, envs, levels):
        """(extension, num_levels given) env envs[i] plays level levels[i] in its next episode, once; afterwards the engine picks again.
        set_next_levels(envs, levels) followed by reset_envs(envs) starts the listed envs on the listed levels now."""
        self.env.set_next_levels([int(e) for e in envs], [int(j) for j in levels])

    def _level_block(self, scenario):
        """the bank block of `scenario` (the batch's distinct scenarios in order of first appearance); None names the only one"""
        if self.num_levels is None:
            raise ValueError('level replacement needs num_levels')
        blocks = list(dict.fromkeys(self.scenarios))
        if scenario is None:
            if len(blocks) > 1:
                raise ValueError('a mixed batch needs scenario= to name the block of levels')
            return 0
        if scenario.casefold() not in blocks:
            raise ValueError('scenario %r is not in this batch' % scenario)
        return blocks.index(scenario.casefold())

    def replace_levels(self, levels, seeds, scenario=None):
        """(extension, num_levels given) level levels[i] of the set (of `scenario`'s block in a mixed batch) is to become the first level of
        seed seeds[i].  Envs playing it finish their episodes on the old level; no env starts it from the next call on, and it is rewritten
        at the start of the first call after a finished call showed no env on it.  Prioritised Level Replay and other curricula use it to
        add fresh levels to the set and evict others."""
        levels, seeds = [int(j) for j in levels], [int(s) for s in seeds]
        if len(levels) != len(seeds):
            raise ValueError('%d levels and %d seeds' % (len(levels), len(seeds)))
        b = self._level_block(scenario)
        for j in levels:
            if not 0 <= j < self.num_levels:
                raise ValueError('level %d is outside the set of %d' % (j, self.num_levels))
        self.env.replace_levels([b * self.num_levels + j for j in levels], seeds)

    def level_seeds(self, scenario=None):
        """(extension, num_levels given) per level of the set (of `scenario`'s block in a mixed batch), the seed of the level it holds now:
        start_level + j until replace_levels rewrites it.  After step(), level_seeds()[info['level']] is the seed of the level a finished
        episode was played on (its level cannot be rewritten before a later call)."""
        b = self._level_block(scenario)
        seeds, _ = self.env.get_level_rows()
        return [int(s) for s in seeds[b * self.num_levels:(b + 1) * self.num_levels]]

    def reset(self):
        self.env.reset()
        self.check_faults()
        self._note_levels()
        return self.observations()

    def step(self, actions):
        self.env.set_actions_batch(np.asarray(actions, dtype=np.int32).reshape(self.num_agents, 6))
        self.env.step()
        self.check_faults()
        return self._step_results()

    def step_envs(self, envs, actions):
        """(extension) step only the envs listed in `envs` (EnvPool's step(actions, env_id)); the others run nothing and keep their state.
        `actions` covers every agent, as in step(), and the entries of unlisted envs are ignored.  Returns step()'s 4-tuple for every agent:
        the agents of unlisted envs get reward 0, done False, {} and their unchanged observation."""
        self.env.set_actions_batch(np.asarray(actions, dtype=np.int32).reshape(self.num_agents, 6))
        self.env.step_envs([int(e) for e in envs])
        self.check_faults()
        return self._step_results()

    def _step_results(self):
        env_dones = self.env.get_dones()
        # the level a done agent's info names: the finished episode's, which the frame still shows unless the env flipped at once
        levels_shown = self._levels_played if self.autoreset_mode == "same_step" else self.level_ids() if self.num_levels is not None else None
        if self.final_observation or self.autoreset_mode != "same_step":
            reasons = self.env.get_done_reasons()
        if self.final_observation:
            final = self.env.get_final_observations()
            final_state = self.env.get_final_state_tensors()['agents'] if self.state_tensors_enabled else None
            final_rays = self.env.get_final_rays() if self.num_rays else None
        episode_components = self.env.get_episode_reward_components() if self.reward_components_enabled else None
        dones, infos = [], []
        for env_i in range(self.num_envs):
            done = bool(env_dones[env_i])
            dones.extend([done for _ in range(self.num_agents_per_env)])
            if done:
                infos.extend([dict(true_reward=float(self.env.true_objective(env_i, j))) for j in range(self.num_agents_per_env)])
                if self.num_levels is not None:
                    for j in range(self.num_agents_per_env):
                        infos[env_i * self.num_agents_per_env + j]['level'] = levels_shown[env_i]
                if episode_components is not None:
                    keys = reward_component_keys(self.scenarios[env_i])
                    for j in range(self.num_agents_per_env):
                        view = env_i * self.num_agents_per_env + j
                        infos[view]['reward_components'] = {k: float(episode_components[view, c]) for c, k in enumerate(keys) if k is not None}
                if self.autoreset_mode != "same_step":
                    for j in range(self.num_agents_per_env):
                        infos[env_i * self.num_agents_per_env + j]['terminated'] = int(reasons[env_i]) == 2
                        infos[env_i * self.num_agents_per_env + j]['truncated'] = int(reasons[env_i]) in (1, 3)
                if self.final_observation:
                    for j in range(self.num_agents_per_env):
                        view = env_i * self.num_agents_per_env + j
                        # a copy: the engine's buffer row is rewritten at the env's next episode end
                        infos[view]['final_observation'] = np.ascontiguousarray(np.transpose(final[view, :, :, :3], (2, 0, 1)))
                        infos[view]['terminated'] = int(reasons[env_i]) == 2
                        infos[view]['truncated'] = int(reasons[env_i]) in (1, 3)
                        if final_state is not None:
                            infos[view]['final_state'] = final_state[view].copy()
                        if final_rays is not None:
                            infos[view]['final_rays'] = (final_rays[0][view].copy(), final_rays[1][view].copy())
            else:
                infos.extend([{} for _ in range(self.num_agents_per_env)])

        if self.SKIP_UNFIT_LEVELS:
            skipped = self.env.levels_skipped()
            if skipped:
                for info in infos:
                    info['levels_skipped'] = skipped
        self._note_levels()
        rewards = self.env.get_last_rewards()
        obs = self.observations()
        return obs, rewards, dones, infos

    def convert_obs(self, obs):
        return obs[:, :, ::-1]  # RGB -> BGR for display; rows are already top-down (the Vulkan path of the reference)

    def render(self, mode='human'):
        self.env.draw_overview()
        self.env.draw_hires()
        rows = []
        for env_i in range(self.num_envs):
            obs = [self.convert_obs(self.env.get_hires_observation(env_i, i)[:, :, :3]) for i in range(self.num_agents_per_env)]
            rows.append(np.concatenate(obs, axis=1))
        obs_final = np.concatenate(rows, axis=0)
        if mode == 'human':
            try:
                import cv2
                cv2.imshow(f'agent_{id(self)}', obs_final)
                cv2.waitKey(1)
            except Exception:  # noqa: BLE001  (headless boxes)
                pass
        return obs_final

    def render_cameras(self, envs, views, w=768, h=432):
        """(extension) spectator cameras: camera c draws env envs[c] of the current scene through the view matrix views[c] (16 float32,
        column-major, megaverse_b200.cameras) at w x h (multiples of 32 x 4, at most 768 x 4096).  Returns RGB uint8 [len(envs), h, w, 3], a
        copy; render() is unchanged"""
        frames = self.env.draw_cameras([int(e) for e in envs], np.asarray(views, dtype=np.float32).reshape(-1, 16), int(w), int(h))[0]
        return np.ascontiguousarray(frames[:, :, :, :3])

    def overview(self, envs, w=768, h=432):
        """(extension) RGB uint8 [len(envs), h, w, 3]: each listed env's whole level seen from above and in front (cameras.overview_views of
        its bounding box)"""
        envs = [int(e) for e in envs]
        return self.render_cameras(envs, overview_views(self.env.level_bounds()[envs], w, h), w, h)

    def chase(self, agents, w=768, h=432):
        """(extension) RGB uint8 [len(agents), h, w, 3]: a third-person camera behind and above each listed agent (index env *
        num_agents_per_env + agent, as in observations()), cameras.chase_views of its own view matrix"""
        agents = [int(a) for a in agents]
        views = chase_views(self.env.get_views()[agents])
        return self.render_cameras([a // self.num_agents_per_env for a in agents], views, w, h)

    def get_default_reward_shaping(self, actor_idx=None):
        """env 0's default scheme; with actor_idx, the default of that actor's scenario (they differ in a mixed batch)"""
        if actor_idx is None:
            return self.default_shaping_scheme
        return dict(self._default_shaping[self.scenarios[actor_idx // self.num_agents_per_env]])

    def get_current_reward_shaping(self, actor_idx: int):
        env_idx = actor_idx // self.num_agents_per_env
        agent_idx = actor_idx % self.num_agents_per_env
        return self.env.get_reward_shaping(env_idx, agent_idx)

    def set_reward_shaping(self, reward_shaping: dict, actor_idx: int):
        env_idx = actor_idx // self.num_agents_per_env
        agent_idx = actor_idx % self.num_agents_per_env
        return self.env.set_reward_shaping(env_idx, agent_idx, reward_shaping)

    def save_state(self, envs=None):
        """(extension) save the complete state of `envs` (default: all) mid-episode; load_state rewinds to it or clones it"""
        envs = list(range(self.num_envs)) if envs is None else [int(e) for e in envs]
        store = self.env.states_create(len(envs))
        state = EnvState(self.env, store, envs)
        self.env.states_save(store, envs, list(range(len(envs))))
        self.check_faults()
        return state

    def load_state(self, state, envs=None, rows=None):
        """(extension) env envs[i] continues from the env saved in row rows[i] of `state` (row i = state.envs[i]); default: every row back into
        the env it was saved from.  A row may go to several envs (clones).  Returns the observations, which equal the saved step's."""
        if state._gym is not self.env:
            raise ValueError("load_state: the state was saved by another env")
        if rows is None:
            rows = list(range(len(state.envs) if envs is None else len(envs)))
        if envs is None:
            envs = [state.envs[r] for r in rows]
        self.env.states_load(state._store, [int(r) for r in rows], [int(e) for e in envs])
        self.check_faults()
        self._note_levels()
        return self.observations()

    def reset_envs(self, envs, seeds=None):
        """(extension) envs[i] start a new episode now, the other envs keep going; with seeds, env envs[i] first takes seed seeds[i] and
        plays the first level of that stream.  Returns the observations of every agent, like reset().  With num_levels, a seed names a
        pick sequence instead, and set_next_levels(envs, levels) before this call chooses the levels the envs start on.  Under
        autoreset_mode "disabled" this is how an env that is done starts its next episode."""
        self.env.reset_envs([int(e) for e in envs], None if seeds is None else [int(s) for s in seeds])
        self.check_faults()
        self._note_levels()
        return self.observations()

    def levels_skipped(self):
        """(extension) levels replaced because they exceeded an engine capacity, see __init__"""
        return self.env.levels_skipped()

    def close(self):
        if self.env:
            self.env.close()
