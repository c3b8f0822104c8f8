"""`DrinkingEnv` (reference envs/drinking.py) on the batched backend.  `step` is the per-call API path: `take_step` + `_get_obs` +
`get_water_rewards` + `human_preferences` through the `Agent` getters, vectorised over `n_envs` (the per-particle Python loops of
drinking.py:51-82 become masks over [n_envs][64]), checked against the reference's own step code
(tests/test_reference_drinking_semantics.py).  `step_fused` runs the same step on the fused device kernels (ag_drinking.cuh,
`ag_drinking_step_host`), armed by `reset`, and returns exactly what `step` returns; `AssistiveVecEnv` steps those kernels with
device tensors.  The robot is the wheelchair-mounted Jaco or Sawyer / PR2 placed by TOC (`drinking_robots_batch.py`)."""
import numpy as np

from ..drinking_batch import CUP_BOTTOM_CENTER_OFFSET, CUP_TOP_CENTER_OFFSET, N_WATER, DrinkingBatch
from ..feeding_batch import HEAD_LINK, IMPAIRMENTS
from ..kinematics import q_rot
from ..sim import BatchSim
from .agents.agent import Agent
from .env import AssistiveEnv


def points_in_cylinder(pt1, pt2, r, q):
    """util.py:53-56 for [n] cylinders and [n][m] points"""
    vec = pt2 - pt1
    const = r * np.linalg.norm(vec, axis=-1)
    a, b = q - pt1[:, None, :], q - pt2[:, None, :]
    return (np.einsum('nmk,nk->nm', a, vec) >= 0) & (np.einsum('nmk,nk->nm', b, vec) <= 0) & (np.linalg.norm(np.cross(a, vec[:, None, :]), axis=-1) <= const[:, None])


def drinking_batch_for(robot):
    """The batched scene of `robot`'s Drinking id: the wheelchair-mounted Jaco, or Sawyer / PR2 placed by TOC."""
    from ..drinking_robots_batch import DrinkingPR2Batch, DrinkingSawyerBatch
    from .agents.robot import PR2, Jaco, Sawyer
    for cls, batch in ((Jaco, DrinkingBatch), (Sawyer, DrinkingSawyerBatch), (PR2, DrinkingPR2Batch)):
        if type(robot) is cls:
            return batch()
    raise KeyError('Drinking is not built for %s' % type(robot).__name__)


class DrinkingEnv(AssistiveEnv):
    def __init__(self, robot, human, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=robot, human=human, task='drinking', n_envs=n_envs, device=device, seed=seed,
                         obs_robot_len=(18 + len(robot.controllable_joint_indices) - (len(robot.wheel_joint_indices) if robot.mobile else 0)),
                         obs_human_len=(19 + len(human.controllable_joint_indices)))
        self._db = drinking_batch_for(robot)
        self.human_impairment = 'random'
        self._cfg = config or DrinkingBatch.config()
        self._sim_lib = None
        self.total_water_count = N_WATER

    # ------------------------------------------------------------------ reset (drinking.py:119-183)
    def reset(self):
        super().reset()
        db = self._db
        if self.id is None:
            self.id = BatchSim(db.scene, self._cfg, self.n_envs, device=self.device, _lib=self._sim_lib)
            self.attach(self.id)
        rng = np.random.default_rng(self.np_random.randint(0, 2 ** 31 - 1))
        s = db.reset(self.id, rng, settle_steps=50, impairment='no_tremor')
        self.start_episode(s)
        db.start_fused(self.id, s, seed=self._seed)
        return self._squeeze(self._get_obs())

    def attach(self, sim):
        """the Agent objects of the scene on `sim` (any object with the BatchSim getter / setter surface)"""
        db = self._db
        self.id = sim
        self.plane.init(db.plane, sim, self.np_random, indices=-1)
        self.robot.init(db.robot, sim, self.np_random)
        self.tool.init(db.tool, sim, self.np_random, indices=-1)
        self.furniture.init(db.wheelchair, sim, self.np_random, indices=-1)
        self.humans = {}
        for g, hb in db.humans.items():
            h = type(self.human)(self.human.controllable_joint_indices, controllable=False)
            h.init(hb, sim, self.np_random, self.human.controllable_joint_indices)
            self.humans[g] = h
        self.water_agents = []
        for w in db.waters:
            a = Agent()
            a.init(w, sim, self.np_random, indices=-1)
            self.water_agents.append(a)

    def start_episode(self, s):
        self.robot.motor_gains = self.human.motor_gains = 0.005              # drinking.py:126
        self.agents = [self.robot]
        self.male = s['male'].astype(bool)
        self.human.gender = 'male' if self.male[0] else 'female'
        self.impairment = s['impairment']
        self.human.impairment = IMPAIRMENTS[int(s['impairment'][0])]
        self.mouth_pos = np.where(self.male[:, None], self._db.mouth['male'], self._db.mouth['female'])
        self.waters = np.ones((self.n_envs, N_WATER), dtype=bool)
        self.waters_active = np.ones((self.n_envs, N_WATER), dtype=bool)
        self.task_success = np.zeros(self.n_envs, dtype=int)
        self.iteration = 0
        self.update_targets()

    def _squeeze(self, a):
        return a[0] if self.n_envs == 1 else a

    # ------------------------------------------------------------------ step (drinking.py:10-49)
    def step(self, action):
        a = np.asarray(action, dtype=np.float64).reshape(self.n_envs, -1)
        self.take_step(a)
        obs = self._get_obs()
        reward_water, vel_sum, water_hit = self.get_water_rewards()
        ee_vel = np.linalg.norm(np.atleast_2d(self.robot.get_velocity(self.robot.right_end_effector)), axis=1)
        pref = (self.C_v * (-ee_vel) + self.C_f * (-self.total_force_on_human) + self.C_hf * np.where(self.cup_force_on_human < 10, 0.0, -self.cup_force_on_human) +
                self.C_fd * water_hit + self.C_fdv * (-vel_sum))                 # env.py:237-274, task 'drinking'
        top, _bottom, cup_quat = self._cup_centres()
        reward_distance = -np.linalg.norm(self.target_pos - top, axis=1)
        x, y, z, w = cup_quat.T                                             # roll of the cup frame (get_euler(...)[0], XYZ fixed axes)
        reward_tilt = -np.abs(np.arctan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y)) - np.pi / 2)
        reward = (self.config('distance_weight') * reward_distance + self.config('action_weight') * (-np.linalg.norm(a, axis=1)) +
                  self.config('cup_tilt_weight') * reward_tilt + self.config('drinking_reward_weight') * reward_water + pref)
        done = np.full(self.n_envs, self.iteration >= 200)
        info = {'total_force_on_human': self.total_force_on_human, 'task_success': (self.task_success >= self.total_water_count * self.config('task_success_threshold')).astype(int),
                'action_robot_len': self.action_robot_len, 'action_human_len': self.action_human_len, 'obs_robot_len': self.obs_robot_len, 'obs_human_len': self.obs_human_len}
        if self.n_envs == 1:
            return obs[0], float(reward[0]), bool(done[0]), {k_: (v[0] if isinstance(v, np.ndarray) else v) for k_, v in info.items()}
        return obs, reward, done, info

    def step_fused(self, action):
        """`step` on the fused, graph-replayed device path (armed by `reset`): takes and returns exactly what `step` does, and
        leaves `waters`, `waters_active` and `task_success` as `step` would."""
        a = np.asarray(action, dtype=np.float32).reshape(self.n_envs, -1)
        obs, rew, done, info = self.id.drinking_step_host(a)
        self.iteration += 1
        ts, w, wa = self.id.drinking_get_state()
        bits = np.arange(N_WATER, dtype=np.uint64)
        self.waters = ((w[:, None] >> bits) & np.uint64(1)).astype(bool)
        self.waters_active = ((wa[:, None] >> bits) & np.uint64(1)).astype(bool)
        self.task_success = ts.astype(int)
        self.total_force_on_human, self.robot_force_on_human, self.cup_force_on_human = (info[:, k].astype(np.float64) for k in (0, 2, 3))
        obs, reward, done = obs.astype(np.float64), rew.astype(np.float64), done > 0.5
        info = {'total_force_on_human': self.total_force_on_human, 'task_success': info[:, 1].astype(int),
                'action_robot_len': self.action_robot_len, 'action_human_len': self.action_human_len, 'obs_robot_len': self.obs_robot_len, 'obs_human_len': self.obs_human_len}
        if self.n_envs == 1:
            return obs[0], float(reward[0]), bool(done[0]), {k_: (v[0] if isinstance(v, np.ndarray) else v) for k_, v in info.items()}
        return obs, reward, done, info

    def _head_pose(self):
        pm, qm = self.humans['male'].get_pos_orient(HEAD_LINK)
        pf, qf = self.humans['female'].get_pos_orient(HEAD_LINK)
        pm, qm, pf, qf = (np.atleast_2d(x) for x in (pm, qm, pf, qf))
        return np.where(self.male[:, None], pm, pf), np.where(self.male[:, None], qm, qf)

    def update_targets(self):                                            # drinking.py:192-196
        hp, hq = self._head_pose()
        self.target_pos = hp + q_rot(hq, self.mouth_pos)

    def _cup_centres(self):                                              # drinking.py:24-26, 54-57
        cp, cq = (np.atleast_2d(x) for x in self.tool.get_base_pos_orient())
        p, q = self._db.cup_frame(cp.astype(np.float64), cq.astype(np.float64))
        return p + q_rot(q, CUP_TOP_CENTER_OFFSET), p + q_rot(q, CUP_BOTTOM_CENTER_OFFSET), q

    def get_total_force(self):                                           # drinking.py:46-49
        r = sum(self.id.contact_force_sum(self.robot.body, h.body) for h in self.humans.values())
        c = sum(self.id.contact_force_sum(self.tool.body, h.body) for h in self.humans.values())
        return np.asarray(r, dtype=np.float64), np.asarray(c, dtype=np.float64)

    def _get_obs(self, agent=None):                                      # drinking.py:84-117 (the robot's part)
        cp, cq = (np.atleast_2d(x) for x in self.tool.get_base_pos_orient())
        cp_r, cq_r = (np.atleast_2d(x) for x in self.robot.convert_to_realworld(cp, cq))
        q = np.atleast_2d(self.robot.get_joint_angles(self.robot.controllable_joint_indices))
        q = (q + np.pi) % (2 * np.pi) - np.pi
        hp, hq = self._head_pose()
        hp_r, hq_r = (np.atleast_2d(x) for x in self.robot.convert_to_realworld(hp, hq))
        tg_r = np.atleast_2d(self.robot.convert_to_realworld(self.target_pos)[0])
        self.robot_force_on_human, self.cup_force_on_human = self.get_total_force()
        self.total_force_on_human = self.robot_force_on_human + self.cup_force_on_human
        return np.concatenate([cp_r, cq_r, cp_r - tg_r, q, hp_r, hq_r, self.cup_force_on_human[:, None]], axis=1)

    def get_water_rewards(self):                                         # drinking.py:51-82
        n = self.n_envs
        top, bottom, _ = self._cup_centres()
        sc = self.id.scene
        ls = self.id.get_link_states([int(sc['body_link0'][w.body]) for w in self.water_agents])
        wp, wv = ls['pos'].astype(np.float64), ls['lin_vel'].astype(np.float64)
        outside = ~points_in_cylinder(top, bottom, 0.05, wp)
        dist = np.linalg.norm(self.target_pos[:, None, :] - wp, axis=-1)
        near = np.zeros((n, N_WATER), dtype=bool)
        candidates = self.waters & outside & ~(dist < 0.03)
        for i in np.where(candidates.any(axis=0))[0]:                    # only particles that left the cup are asked about
            near[:, i] = self.id.closest_points(self.water_agents[i].body, self.tool.body, 0.1, max_pts=1)[1] > 0
        swallowed = self.waters & outside & (dist < 0.03)
        spilled = candidates & ~near
        reward = 10.0 * swallowed.sum(axis=1) - 1.0 * spilled.sum(axis=1)
        self.task_success = self.task_success + swallowed.sum(axis=1)
        vel_sum = (np.linalg.norm(wv, axis=-1) * swallowed).sum(axis=1)
        active_entry = self.waters_active.copy()
        self.waters &= ~(swallowed | spilled)
        self.waters_active &= ~swallowed
        for i in np.where(swallowed.any(axis=0))[0]:                     # drinking.py:70: a swallowed particle is moved far away
            far = self.np_random.uniform(1000, 2000, size=(n, 3))
            self.id.set_base_pose(self.water_agents[i].body, np.where(swallowed[:, i:i + 1], far, wp[:, i]), None, mask=swallowed[:, i].astype(np.int32))
        hit = np.zeros((n, N_WATER), dtype=bool)
        for h in self.humans.values():                                   # particles that touch the person
            c, k = self.id.get_contacts(h.body, -2, max_pts=256)
            for j in range(int(k.max()) if n else 0):
                on = j < k
                lb = c['link_b'][:, j]
                for i, w in enumerate(self.water_agents):
                    hit[:, i] |= on & (lb == int(sc['body_link0'][w.body]))
        hit &= active_entry
        self.waters_active &= ~hit
        return reward, vel_sum, -hit.sum(axis=1).astype(np.float64)
