"""`ScratchItchEnv` (reference envs/scratch_itch.py) on the batched backend: `step` runs the fused path
(`ag_scratch_step_host`); `_get_obs` (used by `reset`) reads the same quantities through the per-call Agent API.
With a controllable person (co-optimisation, `ScratchItchJacoHuman-v1`) `step` takes {'robot': a7, 'human': a10} and goes through
the per-call path (`step_reference_api`): `take_step` drives the person's right arm too and keeps it inside the realistic joint
limits (the MLP classifier of human.py:134-152) after every substep.  `step_fused` runs the same co-optimisation step on the
device (`ag_coop_step_host`)."""
import numpy as np

from .. import capi
from ..kinematics import q_rot
from ..scratch_itch_batch import R_ELBOW, R_SHOULDER, R_WRIST, ScratchItchBatch
from ..sim import BatchSim
from .env import AssistiveEnv


class ScratchItchEnv(AssistiveEnv):
    def __init__(self, robot, human, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=robot, human=human, task='scratch_itch', n_envs=n_envs, device=device, seed=seed,
                         obs_robot_len=(23 + len(robot.controllable_joint_indices) - (len(robot.wheel_joint_indices) if robot.mobile else 0)),
                         obs_human_len=(24 + len(human.controllable_joint_indices)))
        self._sb = ScratchItchBatch()
        self._cfg = config or capi.default_config()
        self._sim_lib = None

    def step(self, action):                                                # scratch_itch.py:10-44
        if self.human.controllable:               # dict in, dicts out (scratch_itch.py:11-12,39-44)
            a = np.concatenate([np.asarray(action['robot'], dtype=np.float64).reshape(self.n_envs, -1),
                                np.asarray(action['human'], dtype=np.float64).reshape(self.n_envs, -1)], axis=1)
            obs, reward, done, info = self.step_reference_api(a)
            d = bool(np.all(done)) if self.n_envs > 1 else bool(done)
            return obs, {'robot': reward, 'human': reward}, {'robot': done, 'human': done, '__all__': d}, {'robot': info, 'human': info}
        a = np.asarray(action, dtype=np.float32).reshape(self.n_envs, -1)
        obs, rew, done, info = self.id.scratch_step_host(a)
        self.iteration += 1
        self.total_force_on_human, self.tool_force_at_target, self.task_success = info[:, 0], info[:, 2], info[:, 3].astype(int)
        out = {'total_force_on_human': info[:, 0], 'task_success': info[:, 1].astype(int), 'action_robot_len': self.action_robot_len,
               'action_human_len': self.action_human_len, 'obs_robot_len': self.obs_robot_len, 'obs_human_len': self.obs_human_len}
        if self.n_envs == 1:
            return obs[0], float(rew[0]), bool(done[0] > 0.5), {k_: (v[0] if isinstance(v, np.ndarray) else v) for k_, v in out.items()}
        return obs, rew, done > 0.5, out

    def step_fused(self, action):
        """`step` of the co-optimisation env (ScratchItchJacoHuman-v1) on the fused, graph-replayed device path: takes and returns
        exactly what `step` does.  `step` itself stays on the per-call path."""
        return self._coop_step_fused(action)

    def update_targets(self):                                              # scratch_itch.py:149-153
        links, col = np.unique(self._limb_links, return_inverse=True)       # a handful of distinct links, whatever the batch size
        ls = self.id.get_link_states(list(links))
        idx = np.arange(self.n_envs)
        self.target_pos = ls['pos'][idx, col].astype(np.float64) + q_rot(ls['quat'][idx, col].astype(np.float64), self._target_local)

    def _get_obs(self, agent=None):                                        # scratch_itch.py:60-91
        self.update_targets()
        tp, tq = (np.atleast_2d(x) for x in self.tool.get_pos_orient(1))
        tp_r, tq_r = (np.atleast_2d(x) for x in self.robot.convert_to_realworld(tp, tq))
        tg_r = np.atleast_2d(self.robot.convert_to_realworld(self.target_pos)[0])
        q = np.atleast_2d(self.robot.get_joint_angles(self.robot.controllable_joint_indices))
        q = (q + np.pi) % (2 * np.pi) - np.pi
        arm = []
        for link in (R_SHOULDER, R_ELBOW, R_WRIST):
            pm = np.atleast_2d(self.humans['male'].get_pos_orient(link)[0]); pf = np.atleast_2d(self.humans['female'].get_pos_orient(link)[0])
            arm.append(np.atleast_2d(self.robot.convert_to_realworld(np.where(self.male[:, None], pm, pf))[0]))
        self.tool_force = self.id.contact_force_sum(self.tool.body).astype(np.float64)
        robot_obs = np.concatenate([tp_r, tq_r, tp_r - tg_r, tg_r, q] + arm + [self.tool_force[:, None]], axis=1)
        if agent == 'robot' or not self.human.controllable:
            return robot_obs
        # scratch_itch.py:75-84: the same quantities in the person's base frame, the person's joint angles, two forces
        self.total_force_on_human, _, self.tool_force_at_target, self.target_contact_pos = self.get_total_force()

        def human_frame(pos, orient=None):
            outs = []
            for g in ('male', 'female'):
                r = self.humans[g].convert_to_realworld(pos, orient if orient is not None else np.array([0, 0, 0, 1.0]))
                outs.append([np.atleast_2d(x) for x in r])
            return [np.where(self.male[:, None], m, f) for m, f in zip(*outs)]
        ci = self.human.controllable_joint_indices
        qh = np.where(self.male[:, None], np.atleast_2d(self.humans['male'].get_joint_angles(ci)), np.atleast_2d(self.humans['female'].get_joint_angles(ci)))
        tp_h, tq_h = human_frame(tp, tq)
        tg_h = human_frame(self.target_pos)[0]
        arm_h = []
        for link in (R_SHOULDER, R_ELBOW, R_WRIST):
            pm = np.atleast_2d(self.humans['male'].get_pos_orient(link)[0]); pf = np.atleast_2d(self.humans['female'].get_pos_orient(link)[0])
            arm_h.append(human_frame(np.where(self.male[:, None], pm, pf))[0])
        human_obs = np.concatenate([tp_h, tq_h, tp_h - tg_h, tg_h, qh] + arm_h + [self.total_force_on_human[:, None], self.tool_force_at_target[:, None]], axis=1)
        if agent == 'human':
            return human_obs
        return {'robot': robot_obs, 'human': human_obs}

    def get_total_force(self):                                             # scratch_itch.py:46-58, every env at once
        n = self.n_envs
        total = sum(self.id.contact_force_sum(self.robot.body, h.body) for h in self.humans.values()).astype(np.float64)
        tool_force = self.id.contact_force_sum(self.tool.body).astype(np.float64)
        at_target, cpos = np.zeros(n), np.full((n, 3), np.nan)
        tool_links = [self.tool.link0, self.tool.link0 + 1]                # linkA in [0, 1]: the handle and the tip
        for h in self.humans.values():
            c, k = self.id.get_contacts(self.tool.body, h.body, max_pts=32)
            for i in range(int(k.max()) if n else 0):
                on = i < k
                f = np.where(on, c['normal_force'][:, i], 0.0).astype(np.float64)
                total += f
                pb = c['pos_b'][:, i].astype(np.float64)
                near = on & np.isin(c['link_a'][:, i], tool_links) & (np.linalg.norm(pb - self.target_pos, axis=1) < 0.025)
                at_target += np.where(near, f, 0.0)
                cpos = np.where(near[:, None], pb, cpos)
        return total, tool_force, at_target, cpos

    def step_reference_api(self, action):                                  # scratch_itch.py:10-44 through the per-call API
        a = np.asarray(action, dtype=np.float64).reshape(self.n_envs, -1)
        self.take_step(a)
        obs = self._get_obs()
        self.total_force_on_human, self.tool_force, self.tool_force_at_target, self.target_contact_pos = self.get_total_force()
        ee_vel = np.linalg.norm(np.atleast_2d(self.robot.get_velocity(self.robot.left_end_effector)), axis=1)
        pref = self.human_preferences(end_effector_velocity=ee_vel, total_force_on_human=self.total_force_on_human, tool_force_at_target=self.tool_force_at_target)
        tool_pos = np.atleast_2d(self.tool.get_pos_orient(1)[0])
        cpos = self.target_contact_pos
        moved = ~np.isnan(cpos[:, 0]) & (np.linalg.norm(np.nan_to_num(cpos) - self.prev_target_contact_pos, axis=1) > 0.01) & (self.tool_force_at_target < 10)
        self.prev_target_contact_pos = np.where(moved[:, None], np.nan_to_num(cpos), self.prev_target_contact_pos)
        self.task_success = self.task_success + moved
        reward = (self.config('distance_weight') * (-np.linalg.norm(self.target_pos - tool_pos, axis=1)) + self.config('action_weight') * (-np.linalg.norm(a, axis=1)) +
                  self.config('scratch_reward_weight') * 5.0 * moved + pref)
        done = np.full(self.n_envs, self.iteration >= 200)
        info = {'total_force_on_human': self.total_force_on_human, 'task_success': (self.task_success >= self.config('task_success_threshold')).astype(int),
                'action_robot_len': self.action_robot_len, 'action_human_len': self.action_human_len, 'obs_robot_len': self.obs_robot_len, 'obs_human_len': self.obs_human_len}
        sq = (lambda v: {k_: sq(x) for k_, x in v.items()} if isinstance(v, dict) else (v[0] if self.n_envs == 1 else v))
        return sq(obs), sq(reward), sq(done), info

    def reset(self):                                                       # scratch_itch.py:93-132
        super().reset()
        sb = self._sb
        if self.id is None:
            self.id = BatchSim(sb.scene, self._cfg, self.n_envs, device=self.device, _lib=self._sim_lib)
            sim = self.id
            self.plane.init(sb.plane, sim, self.np_random, indices=-1)
            self.robot.init(sb.robot, sim, self.np_random)
            self.tool.init(sb.tool, sim, self.np_random, indices=-1)
            self.furniture.init(sb.wheelchair, sim, self.np_random, indices=-1)
            self.humans = {}
            for g, hb in sb.humans.items():
                h = type(self.human)(self.human.controllable_joint_indices, controllable=self.human.controllable)
                h.init(hb, sim, self.np_random, self.human.controllable_joint_indices)
                self.humans[g] = h
        rng = np.random.default_rng(self.np_random.randint(0, 2 ** 31 - 1))
        self.agents = [self.robot]
        s = sb.reset(self.id, rng)
        self.male = s['male'].astype(bool)
        self.human.gender = 'male' if self.male[0] else 'female'
        self.prev_target_contact_pos = np.zeros((self.n_envs, 3))         # scratch_itch.py:96
        if self.human.controllable:               # both gender instances act; the switched-off one moves nothing (env.py:130)
            for g, h in self.humans.items():
                h.env_mask = self.male if g == 'male' else ~self.male
                h.arm_previous_valid_pose = {True: None, False: None}
                h.set_limit_scale(s.get('limit_scale', np.ones(self.n_envs)))     # impairment 'limits': scaled joint limits (human.py:85)
                h.enforce_joint_limits(h.controllable_joint_indices)              # the start pose is clipped to them (human.py:115 set_joint_angles)
                self.agents.append(h)
            self.id.forward_kinematics()
        self._limb_links, self._target_local = sb.limb_links(s), s['target_local']
        sb.start_fused(self.id, s)
        if self.human.controllable:
            sb.start_coop(self.id, s)
        self.task_success = np.zeros(self.n_envs, dtype=int)
        obs = self._get_obs()
        if isinstance(obs, dict):
            return {k_: (v[0] if self.n_envs == 1 else v) for k_, v in obs.items()}
        return obs[0] if self.n_envs == 1 else obs
