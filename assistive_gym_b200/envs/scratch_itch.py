"""`ScratchItchEnv` (reference envs/scratch_itch.py) on the batched backend: `step` runs the fused path
(`ag_scratch_step_host`); `_get_obs` (used by `reset`) reads the same quantities through the per-call Agent API.  The robot is the
wheelchair-mounted Jaco or Sawyer / PR2 placed by TOC (`scratch_itch_robots_batch.py`).
With a controllable person (co-optimisation, `ScratchItchJacoHuman-v1`, `ScratchItchSawyerHuman-v1`, `ScratchItchPR2Human-v1`) `step` takes {'robot': a7, 'human': a10} and goes through
the per-call path (`step_reference_api`): `take_step` drives the person's right arm too and keeps it inside the realistic joint
limits (the MLP classifier of human.py:134-152) after every substep.  `step_fused` runs the same co-optimisation step on the
device (`ag_coop_step_host`)."""
import numpy as np

from .. import capi
from ..kinematics import q_rot
from ..scratch_itch_batch import R_ELBOW, R_SHOULDER, R_WRIST, ScratchItchBatch
from ..sim import BatchSim
from .env import AssistiveEnv


def scratch_batch_for(robot):
    """The batched scene of `robot`'s ScratchItch id: the wheelchair-mounted Jaco, or Sawyer / PR2 placed by TOC."""
    from ..scratch_itch_robots_batch import ScratchItchPR2Batch, ScratchItchSawyerBatch
    from .agents.robot import PR2, Jaco, Sawyer
    for cls, batch in ((Jaco, ScratchItchBatch), (Sawyer, ScratchItchSawyerBatch), (PR2, ScratchItchPR2Batch)):
        if type(robot) is cls:
            return batch()
    raise KeyError('ScratchItch is not built for %s' % type(robot).__name__)


class ScratchItchEnv(AssistiveEnv):
    def __init__(self, robot, human, n_envs=1, device=0, seed=1001, config=None, human_impairment=None):
        super().__init__(robot=robot, human=human, task='scratch_itch', n_envs=n_envs, device=device, seed=seed, human_impairment=human_impairment,
                         obs_robot_len=(23 + len(robot.controllable_joint_indices) - (len(robot.wheel_joint_indices) if robot.mobile else 0)),
                         obs_human_len=(24 + len(human.controllable_joint_indices)))
        self._sb = scratch_batch_for(robot)
        self._cfg = config or capi.default_config()
        self._sim_lib = None

    def step(self, action):                                                # scratch_itch.py:10-44
        if self.human.controllable:               # dict in, dicts out (scratch_itch.py:11-12,39-44)
            return self._coop_step(action)
        obs, rew, done, info = self._fused_step(self.id.scratch_step_host, action)
        self.tool_force_at_target, self.task_success = info[:, 2], info[:, 3].astype(int)
        return self._unwrap(obs, rew, done, self._info(info[:, 0], info[:, 1].astype(int)))

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
        arm = [np.atleast_2d(self.robot.convert_to_realworld(self._person_pose(link)[0])[0]) for link in (R_SHOULDER, R_ELBOW, R_WRIST)]
        self.tool_force = self.id.contact_force_sum(self.tool.body).astype(np.float64)
        robot_obs = np.concatenate([tp_r, tq_r, tp_r - tg_r, tg_r, q] + arm + [self.tool_force[:, None]], axis=1)
        if agent == 'robot' or not self.human.controllable:
            return robot_obs
        # scratch_itch.py:75-84: the same quantities in the person's base frame, the person's joint angles, two forces
        self.total_force_on_human, _, self.tool_force_at_target, self.target_contact_pos = self.get_total_force()
        qh = self._person_joint_angles()
        tp_h, tq_h = self._person_frame(tp, tq)
        tg_h = self._person_frame(self.target_pos)[0]
        arm_h = [self._person_frame(self._person_pose(link)[0])[0] for link in (R_SHOULDER, R_ELBOW, R_WRIST)]
        human_obs = np.concatenate([tp_h, tq_h, tp_h - tg_h, tg_h, qh] + arm_h + [self.total_force_on_human[:, None], self.tool_force_at_target[:, None]], axis=1)
        if agent == 'human':
            return human_obs
        return {'robot': robot_obs, 'human': human_obs}

    def get_total_force(self):                                             # scratch_itch.py:46-58, every env at once
        n = self.n_envs
        total = sum(self.id.contact_force_sum(self.robot.body, h.body) for h in self.humans.values()).astype(np.float64)
        tool_force = self.id.contact_force_sum(self.tool.body).astype(np.float64)
        at_target, cpos = np.zeros(n), np.full((n, 3), np.nan)
        tool_links = [self.tool._gl(0), self.tool._gl(1)]                  # linkA in [0, 1]: the scratcher's links 0 and 1 (not its base)
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
        info = self._info(self.total_force_on_human, (self.task_success >= self.config('task_success_threshold')).astype(int))
        # as Feeding's, unlike Dressing's, BedBathing's and Drinking's: with n_envs == 1 the reward stays a NumPy value and info is not unwrapped
        return self._squeeze(obs), self._squeeze(reward), self._squeeze(done), info

    def reset(self):                                                       # scratch_itch.py:93-132
        super().reset()
        sb = self._sb
        if self.id is None:
            self._attach(sb, sb.wheelchair, BatchSim)
        rng = np.random.default_rng(self.np_random.randint(0, 2 ** 31 - 1))
        self.agents = [self.robot]
        s = sb.reset(self.id, rng, sample=self._person_sample(sb, rng))
        self.male = s['male'].astype(bool)
        self.human.gender = 'male' if self.male[0] else 'female'
        self.prev_target_contact_pos = np.zeros((self.n_envs, 3))         # scratch_itch.py:96
        if self.human.controllable:
            self._controllable_person(s.get('limit_scale', np.ones(self.n_envs)))
            for h in self.humans.values():
                h.enforce_joint_limits(h.controllable_joint_indices)              # the start pose is clipped to them (human.py:115 set_joint_angles)
            self.id.forward_kinematics()
            if self.human_impairment_coop is not None:
                self._person_tremor(s, sb.coop_tremor_target(s))
        self._limb_links, self._target_local = sb.limb_links(s), s['target_local']
        sb.start_fused(self.id, s)
        if self.human.controllable:
            sb.start_coop(self.id, s)
        self.task_success = np.zeros(self.n_envs, dtype=int)
        return self._squeeze(self._get_obs())
