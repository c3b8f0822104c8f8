"""`BedBathingEnv` (reference envs/bed_bathing.py) on the batched backend.

`step` runs the fused kernels (`ag_bathing_step_host`): action -> PD targets -> 5 substeps -> obs /
reward / done, wiping targets included.  `step_reference_api` performs the same step the way the
reference does it -- `take_step` + `_get_obs` + `get_total_force` + `human_preferences` through the
per-call `Agent` API, vectorised over `n_envs` (the per-contact Python loop of `get_total_force`,
bed_bathing.py:41-78, becomes one masked distance test of every tool-cloth contact against every
remaining wiping target) -- and exists so that tests can show the two paths agree.

With a controllable person (co-optimisation, `BedBathingSawyerHuman-v1`) `step` takes {'robot': a7, 'human': a10} and goes through
the per-call path (`step_reference_api`): `take_step` drives the person's right arm, keeps it inside its (per-env scaled) limits
and the realistic joint limits (human.py:134-152) after every substep, and the wiping targets follow the arm (`update_targets`).
`step_fused` runs the same co-optimisation step on the device (`ag_coop_step_host`).  Deviations: the person is not settled as a
ragdoll at reset (it is lowered onto the mattress, as for the static person), and `tremor` is not drawn for it."""
import numpy as np

from .. import capi
from ..bed_bathing_batch import R_ELBOW, R_SHOULDER, R_WRIST, WIPER_CLOTH_LINK, BedBathingBatch
from ..sim import BatchSim
from .agents.furniture import Furniture
from .env import AssistiveEnv

MAX_TOOL_CONTACTS = 32


class BedBathingEnv(AssistiveEnv):
    def __init__(self, robot, human, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=robot, human=human, task='bed_bathing', n_envs=n_envs, device=device, seed=seed,
                         obs_robot_len=(17 + len(robot.controllable_joint_indices) - (len(robot.wheel_joint_indices) if robot.mobile else 0)),
                         obs_human_len=(18 + len(human.controllable_joint_indices)))
        self._bb = BedBathingBatch(controllable_person=human.controllable)
        self._cfg = config or capi.default_config()
        self._sim_lib = None

    # ------------------------------------------------------------------ fused step (bed_bathing.py:12-39)
    def step(self, action):
        if self.human.controllable:               # dict in, dicts out (bed_bathing.py:13-14,35-39)
            a = np.concatenate([np.asarray(action['robot'], dtype=np.float64).reshape(self.n_envs, -1),
                                np.asarray(action['human'], dtype=np.float64).reshape(self.n_envs, -1)], axis=1)
            obs, reward, done, info = self.step_reference_api(a)
            d = bool(np.all(done)) if self.n_envs > 1 else bool(done)
            return obs, {'robot': reward, 'human': reward}, {'robot': done, 'human': done, '__all__': d}, {'robot': info, 'human': info}
        a = np.asarray(action, dtype=np.float32).reshape(self.n_envs, -1)
        obs, rew, done, info = self.id.bathing_step_host(a)
        self.iteration += 1
        self.total_force_on_human, self.tool_force_on_human, self.new_contact_points = info[:, 0], info[:, 2], info[:, 3].astype(int)
        self.task_success += self.new_contact_points
        out = {'total_force_on_human': info[:, 0], 'task_success': info[:, 1].astype(int), 'action_robot_len': self.action_robot_len,
               'action_human_len': self.action_human_len, 'obs_robot_len': self.obs_robot_len, 'obs_human_len': self.obs_human_len}
        if self.n_envs == 1:
            return obs[0], float(rew[0]), bool(done[0] > 0.5), {k_: (v[0] if isinstance(v, np.ndarray) else v) for k_, v in out.items()}
        return obs, rew, done > 0.5, out

    def step_fused(self, action):
        """`step` of the co-optimisation env (BedBathingSawyerHuman-v1) on the fused, graph-replayed device path: takes and returns
        exactly what `step` does.  `step` itself stays on the per-call path."""
        return self._coop_step_fused(action)

    # ------------------------------------------------------------------ the same step through the reference-shaped API
    def step_reference_api(self, action):
        a = np.asarray(action, dtype=np.float64).reshape(self.n_envs, -1)
        self.take_step(a)
        obs = self._get_obs()
        ee_vel = np.linalg.norm(np.atleast_2d(self.robot.get_velocity(self.robot.left_end_effector)), axis=1)
        pref = self.human_preferences(end_effector_velocity=ee_vel, total_force_on_human=self.total_force_on_human,
                                      tool_force_at_target=self.tool_force_on_human)
        dmin = np.full(self.n_envs, np.inf)                                                  # bed_bathing.py:23
        for hb in self._bb.humans.values():           # the inactive gender returns no points
            c, k = self.id.closest_points(self.tool.body, hb, 5.0, max_pts=256)        # within 5 m that is every collider pair of wiper x person (~140): all of them, the minimum may be anywhere
            assert int(k.max()) <= 256
            dmin = np.minimum(dmin, np.where(np.arange(256)[None, :] < k[:, None], c['distance'], np.inf).min(axis=1))
        dmin = np.where(np.isfinite(dmin), dmin, 5.0)
        reward = (self.config('distance_weight') * (-dmin) + self.config('action_weight') * (-np.linalg.norm(a, axis=1)) +
                  self.config('wiping_reward_weight') * self.new_contact_points + pref)
        done = np.full(self.n_envs, self.iteration >= 200)
        success = (self.task_success >= self.total_target_count * self.config('task_success_threshold')).astype(int)
        info = {'total_force_on_human': self.total_force_on_human, 'task_success': success, 'action_robot_len': self.action_robot_len,
                'action_human_len': self.action_human_len, 'obs_robot_len': self.obs_robot_len, 'obs_human_len': self.obs_human_len}
        if self.n_envs == 1:
            obs = {k_: v[0] for k_, v in obs.items()} if isinstance(obs, dict) else obs[0]
            return obs, float(reward[0]), bool(done[0]), {k_: (v[0] if isinstance(v, np.ndarray) else v) for k_, v in info.items()}
        return obs, reward, done, info

    # ------------------------------------------------------------------ get_total_force (bed_bathing.py:41-78)
    def get_total_force(self):
        tool_force, tool_on_human, total, new_pts = self._bb.total_force(self.id, self.targets_pos_world, self.targets_alive, MAX_TOOL_CONTACTS)
        self.task_success += new_pts
        return tool_force, tool_on_human, total, new_pts

    def _get_obs(self, agent=None):                                       # bed_bathing.py:80-111
        tp, tq = (np.atleast_2d(x) for x in self.tool.get_pos_orient(WIPER_CLOTH_LINK))
        tp_r, tq_r = (np.atleast_2d(x) for x in self.robot.convert_to_realworld(tp, tq))
        q = np.atleast_2d(self.robot.get_joint_angles(self.robot.controllable_joint_indices))
        q = (q + np.pi) % (2 * np.pi) - np.pi
        arm = [np.atleast_2d(self.robot.convert_to_realworld(p_)[0]) for p_ in self._arm_points()]
        self.tool_force, self.tool_force_on_human, self.total_force_on_human, self.new_contact_points = self.get_total_force()
        robot_obs = np.concatenate([tp_r, tq_r, q] + arm + [self.tool_force[:, None]], axis=1)
        if agent == 'robot' or not self.human.controllable:
            return robot_obs
        # bed_bathing.py:99-105: the wiper, the person's joint angles (not wrapped) and the arm points in the person's base frame
        def human_frame(pos, orient=None):
            outs = []
            for g in ('male', 'female'):
                r = self.humans[g].convert_to_realworld(pos, orient if orient is not None else np.array([0, 0, 0, 1.0]))
                outs.append([np.atleast_2d(x) for x in r])
            return [np.where(self.male[:, None], m, f) for m, f in zip(*outs)]
        ci = self.human.controllable_joint_indices
        qh = np.where(self.male[:, None], np.atleast_2d(self.humans['male'].get_joint_angles(ci)), np.atleast_2d(self.humans['female'].get_joint_angles(ci)))
        tp_h, tq_h = human_frame(tp, tq)
        arm_h = [human_frame(p_)[0] for p_ in self._arm_points()]
        human_obs = np.concatenate([tp_h, tq_h, qh] + arm_h + [np.asarray(self.total_force_on_human, dtype=np.float64)[:, None],
                                                              np.asarray(self.tool_force_on_human, dtype=np.float64)[:, None]], axis=1)
        if agent == 'human':
            return human_obs
        return {'robot': robot_obs, 'human': human_obs}

    def _arm_points(self):
        out = []
        for link in (R_SHOULDER, R_ELBOW, R_WRIST):
            pm = np.atleast_2d(self.humans['male'].get_pos_orient(link)[0])
            pf = np.atleast_2d(self.humans['female'].get_pos_orient(link)[0])
            out.append(np.where(self.male[:, None], pm, pf))
        return out

    # ------------------------------------------------------------------ reset (bed_bathing.py:113-168)
    def reset(self):
        super().reset()
        bb = self._bb
        if self.id is None:
            self.id = BatchSim(bb.scene, self._cfg, self.n_envs, device=self.device, _lib=self._sim_lib)
            sim = self.id
            self.plane.init(bb.plane, sim, self.np_random, indices=-1)
            self.robot.init(bb.robot, sim, self.np_random)
            self.tool.init(bb.tool, sim, self.np_random, indices=-1)
            self.furniture.init(bb.bed, sim, self.np_random, indices=-1)
            self.humans = {}
            for g, hb in bb.humans.items():
                h = type(self.human)(self.human.controllable_joint_indices, controllable=self.human.controllable)
                h.init(hb, sim, self.np_random, self.human.controllable_joint_indices)
                self.humans[g] = h
        rng = np.random.default_rng(self.np_random.randint(0, 2 ** 31 - 1))
        self.agents = [self.robot]
        s = bb.reset(self.id, rng)
        self.male = s['male'].astype(bool)
        self.human.gender = 'male' if self.male[0] else 'female'
        if self.human.controllable:               # both gender instances act; the switched-off one moves nothing (env.py:130)
            for g, h in self.humans.items():
                h.env_mask = self.male if g == 'male' else ~self.male
                h.arm_previous_valid_pose = {True: None, False: None}
                h.set_limit_scale(s['limit_scale'])                               # impairment 'limits': scaled joint limits (human.py:85)
                h.enforce_joint_limits(h.controllable_joint_indices)              # the start pose is clipped to them (human.py:115)
                self.agents.append(h)
            self.id.forward_kinematics()
        self.generate_targets(s)
        if self.human.controllable:
            bb.start_coop(self.id, s)
        self.task_success = np.zeros(self.n_envs, dtype=int)
        obs = self._get_obs()
        if isinstance(obs, dict):
            return {k_: (v[0] if self.n_envs == 1 else v) for k_, v in obs.items()}
        return obs[0] if self.n_envs == 1 else obs

    def generate_targets(self, s):                                         # bed_bathing.py:173-203
        self.targets_pos_world, self.targets_alive = self._bb.start_fused(self.id, s)
        self.total_target_count = self.targets_alive.sum(axis=1)

    def update_targets(self):                                              # bed_bathing.py:190-203
        if not self.human.controllable:
            return     # the person is static after reset: the world positions computed in generate_targets stay valid
        self.targets_pos_world = self._bb.targets_world(self.id, {'male': self.male})[0]
