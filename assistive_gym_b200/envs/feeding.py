"""`FeedingEnv` (reference envs/feeding.py) on the batched backend.

`step` runs the fused kernels (`ag_feeding_step_host`): action -> PD targets -> 5 substeps -> obs /
reward / done.  With a controllable person (FeedingJacoHuman-v1) `step` goes through the per-call path and `step_fused` through
the fused co-optimisation kernels (`ag_coop_step_host`).  `step_reference_api` performs the same step the way the reference does it —
`take_step` + `_get_obs` + `get_food_rewards` + `human_preferences` through the per-call `Agent`
API — and exists so that tests can show the two paths agree."""
import numpy as np

from .. import capi
from ..feeding_batch import HEAD_LINK, IMPAIRMENTS, FeedingBatch
from ..kinematics import q_rot
from ..sim import BatchSim
from .agents.agent import Agent
from .agents.furniture import Furniture
from .env import AssistiveEnv


def feeding_batch_for(robot):
    """The batched scene of `robot`'s Feeding id: the wheelchair-mounted Jaco, or Sawyer / PR2 placed by TOC."""
    from ..feeding_robots_batch import FeedingPR2Batch, FeedingSawyerBatch
    from .agents.robot import PR2, Jaco, Sawyer
    for cls, batch in ((Jaco, FeedingBatch), (Sawyer, FeedingSawyerBatch), (PR2, FeedingPR2Batch)):
        if type(robot) is cls:
            return batch()
    raise KeyError('Feeding is not built for %s' % type(robot).__name__)


class FeedingEnv(AssistiveEnv):
    def __init__(self, robot, human, n_envs=1, device=0, seed=1001, config=None, human_impairment=None):
        super().__init__(robot=robot, human=human, task='feeding', n_envs=n_envs, device=device, seed=seed, human_impairment=human_impairment,
                         obs_robot_len=(18 + len(robot.controllable_joint_indices) - (len(robot.wheel_joint_indices) if robot.mobile else 0)),
                         obs_human_len=(19 + len(human.controllable_joint_indices)))
        self._fb = feeding_batch_for(robot)
        self.human_impairment = 'random'      # build_assistive_env(human_impairment='random'), env.py:114
        self._cfg = config or self._fb.config()
        self._sim_lib = None
        self.total_food_count = 8

    # ------------------------------------------------------------------ reset (feeding.py:114-182)
    def reset(self):
        super().reset()
        fb = self._fb
        if self.id is None:
            self._attach(fb, fb.wheelchair, BatchSim)
            self.table, self.bowl = Furniture(), Furniture()
            self.table.init(fb.table, self.id, self.np_random, indices=-1)
            self.bowl.init(fb.bowl, self.id, self.np_random, indices=-1)
            self.foods_agents = []
            for f in fb.foods:
                a = Agent()
                a.init(f, self.id, self.np_random, indices=-1)
                self.foods_agents.append(a)
        rng = np.random.default_rng(self.np_random.randint(0, 2 ** 31 - 1))
        self.robot.motor_gains = self.human.motor_gains = 0.025          # feeding.py:122
        self.agents = [self.robot]
        coop = bool(self.human.controllable)
        # co-optimisation: 'no_tremor' unless `human_impairment` is given (AssistiveEnv._person_sample)
        imp = 'no_tremor' if coop else self.human_impairment
        s = fb.reset(self.id, rng, settle_steps=25, sample=self._person_sample(fb, rng, imp), impairment=imp, simulate_head=coop)
        self.male = s['male'].astype(bool)
        self.human.gender = 'male' if self.male[0] else 'female'
        # impairments (human.py:79-92).  The reference appends a tremor human to `agents`
        # (env.py:130-131); here each gender's Human carries a per-env tremor mask.
        tremor = s['impairment'] == 3
        self.impairment = s['impairment']
        self.human.impairment = IMPAIRMENTS[int(s['impairment'][0])]
        self.human.limit_scale, self.human.strength = float(s['limit_scale'][0]), float(s['strength'][0])
        rest = fb.tremor_rest_of(s)
        for g, h in self.humans.items():
            h.tremor_mask = tremor & (self.male if g == 'male' else ~self.male)
            h.impairment = 'tremor' if h.tremor_mask.any() else 'none'
            h.tremors = np.where(h.tremor_mask[:, None], s['tremors'], 0.0)
            h.target_joint_angles = rest
            h.motor_gains = self.human.motor_gains
            if h.tremor_mask.any() and not coop:         # a controllable person is an agent anyway, below
                self.agents.append(h)
        if coop:                                  # both gender instances act; the switched-off one moves nothing (env.py:130)
            for h in self.humans.values():
                h.motor_gains, h.motor_forces = self.human.motor_gains, self.human.motor_forces
                self.agents.append(h)
        self.mouth_pos = np.where(self.male[:, None], fb.mouth['male'], fb.mouth['female'])
        fb.start_fused(self.id, s, seed=self._seed)
        if coop:
            fb.start_coop(self.id, s)
        self.foods = np.ones((self.n_envs, 8), dtype=bool)
        self.foods_active = np.ones((self.n_envs, 8), dtype=bool)
        self.task_success = np.zeros(self.n_envs, dtype=int)
        self.update_targets()
        return self._squeeze(self._get_obs())

    # ------------------------------------------------------------------ fused step (feeding.py:12-43)
    def step(self, action):
        if self.human.controllable:               # feeding.py:13-14,40-43: dict in, dicts out (per-call API path)
            return self._coop_step(action)
        obs, rew, done, info = self._fused_step(self.id.feeding_step_host, action)
        # unlike the other tasks' steps, a list of per-env info dicts of Python scalars
        infos = [self._info(float(info[e, 0]), int(info[e, 1])) for e in range(self.n_envs)]
        return self._unwrap(obs, rew, done, infos if self.n_envs > 1 else infos[0])

    # ------------------------------------------------------------------ the same step through the reference-shaped API
    def update_targets(self):                                            # feeding.py:192-196
        hp, hq = self._person_pose(HEAD_LINK)
        self.target_pos = hp + q_rot(hq, self.mouth_pos)

    def get_total_force(self):                                           # feeding.py:45-48
        r = sum(self.id.contact_force_sum(self.robot.body, h.body) for h in self.humans.values())
        s = sum(self.id.contact_force_sum(self.tool.body, h.body) for h in self.humans.values())
        return r.astype(np.float64), s.astype(np.float64)

    def _get_obs(self, agent=None):                                      # feeding.py:85-112
        sp, sq = (np.atleast_2d(x) for x in self.tool.get_base_pos_orient())
        sp_r, sq_r = (np.atleast_2d(x) for x in self.robot.convert_to_realworld(sp, sq))
        q = np.atleast_2d(self.robot.get_joint_angles(self.robot.controllable_joint_indices))
        q = (q + np.pi) % (2 * np.pi) - np.pi
        hp, hq = self._person_pose(HEAD_LINK)
        hp_r, hq_r = (np.atleast_2d(x) for x in self.robot.convert_to_realworld(hp, hq))
        tg_r = np.atleast_2d(self.robot.convert_to_realworld(self.target_pos)[0])
        self.robot_force_on_human, self.spoon_force_on_human = self.get_total_force()
        self.total_force_on_human = self.robot_force_on_human + self.spoon_force_on_human
        robot_obs = np.concatenate([sp_r, sq_r, sp_r - tg_r, q, hp_r, hq_r, self.spoon_force_on_human[:, None]], axis=1)
        if agent == 'robot' or not self.human.controllable:
            return robot_obs
        # feeding.py:101-111: the same quantities in the person's base frame + the person's joint angles
        qh = self._person_joint_angles()
        sp_h, sq_h = self._person_frame(sp, sq)
        hp_h, hq_h = self._person_frame(hp, hq)
        tg_h = self._person_frame(self.target_pos)[0]
        human_obs = np.concatenate([sp_h, sq_h, sp_h - tg_h, qh, hp_h, hq_h, self.robot_force_on_human[:, None], self.spoon_force_on_human[:, None]], axis=1)
        if agent == 'human':
            return human_obs
        return {'robot': robot_obs, 'human': human_obs}

    def get_food_rewards(self):                                          # feeding.py:50-83
        n = self.n_envs
        food_reward, hit_reward, vel_sum = np.zeros(n), np.zeros(n), np.zeros(n)
        active_entry = self.foods_active.copy()
        for i, f in enumerate(self.foods_agents):
            fp = np.atleast_2d(f.get_base_pos_orient()[0])
            dist = np.linalg.norm(self.target_pos - fp, axis=1)
            near = self.id.closest_points(f.body, self.tool.body, 0.1, max_pts=1)[1] > 0
            eaten = self.foods[:, i] & (dist < 0.03)
            spilled = self.foods[:, i] & ~eaten & ~near
            food_reward += 20.0 * eaten - 5.0 * spilled
            self.task_success += eaten
            vel_sum += eaten * np.linalg.norm(np.atleast_2d(f.get_velocity(f.base)), axis=1)
            self.foods[:, i] &= ~(eaten | spilled)
            self.foods_active[:, i] &= ~eaten
            if eaten.any():   # teleport eaten food far away (feeding.py:69)
                far = self.np_random.uniform(1000, 2000, size=(n, 3))
                self.id.set_base_pose(f.body, np.where(eaten[:, None], far, fp), None, mask=eaten.astype(np.int32))
        for i, f in enumerate(self.foods_agents):
            touching = sum(self.id.get_contacts(f.body, h.body, max_pts=1)[1] for h in self.humans.values()) > 0
            hit = active_entry[:, i] & touching
            hit_reward -= hit
            self.foods_active[:, i] &= ~hit
        return food_reward, vel_sum, hit_reward

    def step_reference_api(self, action):
        a = np.asarray(action, dtype=np.float64).reshape(self.n_envs, -1)
        self.take_step(a)
        obs = self._get_obs()
        reward_food, vel_sum, food_hit = self.get_food_rewards()
        ee_vel = np.linalg.norm(np.atleast_2d(self.robot.get_velocity(self.robot.right_end_effector)), axis=1)
        pref = (self.C_v * (-ee_vel) + self.C_f * (-self.total_force_on_human) +
                self.C_hf * np.where(self.spoon_force_on_human < 10, 0.0, -self.spoon_force_on_human) + self.C_fd * food_hit + self.C_fdv * (-vel_sum))
        spoon_pos = np.atleast_2d(self.tool.get_base_pos_orient()[0])
        reward = (self.config('distance_weight') * (-np.linalg.norm(self.target_pos - spoon_pos, axis=1)) +
                  self.config('action_weight') * (-np.linalg.norm(a, axis=1)) + self.config('food_reward_weight') * reward_food + pref)
        done = np.full(self.n_envs, self.iteration >= 200)
        info = self._info(self.total_force_on_human, (self.task_success >= self.total_food_count * self.config('task_success_threshold')).astype(int))
        # as ScratchItch's, unlike Dressing's, BedBathing's and Drinking's: with n_envs == 1 the reward stays a NumPy value and info is not unwrapped
        return self._squeeze(obs), self._squeeze(reward), self._squeeze(done), info
