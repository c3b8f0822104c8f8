"""`DressingEnv` (reference envs/dressing.py) on the batched backend.

`step` runs the fused path (`ag_dressing_step_host`): action -> PD targets -> 5 x (8 rigid substeps + one cloth launch, the
cloth's anchor follows the end effector) -> sleeve-on-arm reward, cloth forces, obs[24] / reward / done.  `_get_obs` (used
by `reset`) reads the same quantities through the per-call Agent API.

The robot is PR2 or Sawyer placed by TOC, or the wheelchair-mounted Jaco (`dressing_batch_for`).

With a controllable person (co-optimisation, `Dressing{PR2,Sawyer,Jaco}Human-v1`) `step` takes {'robot': a7, 'human': a10} and goes through the
per-call path (`step_reference_api`): `take_step` drives the person's left arm and, after every stepSimulation, keeps it inside its
(per-env scaled) limits and the realistic joint limits (human.py:134-152), then moves the gown's anchor to the end effector
(`update_targets`); the observation, the sleeve-on-arm reward and the cloth forces are computed on the host.  `step_fused` runs
the same co-optimisation step on the device (`ag_coop_step_host`).  `tremor` is drawn for a controllable person only with `human_impairment` (AssistiveEnv)."""
import numpy as np

from .. import capi
from ..dressing_batch import L_ELBOW, L_SHOULDER, L_WRIST, RADII, TRIANGLE1, TRIANGLE2, DressingBatch, sleeve_on_arm_reward
from ..sim import BatchSim
from .env import AssistiveEnv

ARM_LINKS = (L_SHOULDER, L_ELBOW, L_WRIST)


def dressing_batch_for(robot, controllable_person=False):
    """The batched scene of `robot`'s Dressing id: PR2 or Sawyer placed by TOC, or the wheelchair-mounted Jaco."""
    from ..dressing_robots_batch import DressingJacoBatch, DressingSawyerBatch
    from .agents.robot import PR2, Jaco, Sawyer
    for cls, batch in ((PR2, DressingBatch), (Sawyer, DressingSawyerBatch), (Jaco, DressingJacoBatch)):
        if type(robot) is cls:
            return batch(controllable_person=controllable_person)
    raise KeyError('Dressing is not built for %s' % type(robot).__name__)


class DressingEnv(AssistiveEnv):
    def __init__(self, robot, human, n_envs=1, device=0, seed=1001, config=None, toc_attempts=50, human_impairment=None):
        super().__init__(robot=robot, human=human, task='dressing', n_envs=n_envs, device=device, seed=seed, human_impairment=human_impairment,
                         obs_robot_len=(17 + len(robot.controllable_joint_indices) - (len(robot.wheel_joint_indices) if robot.mobile else 0)),
                         obs_human_len=(18 + len(human.controllable_joint_indices)))
        self._db = dressing_batch_for(robot, controllable_person=human.controllable)
        self._cfg = config or DressingBatch.config()                       # numSubSteps = 8 (dressing.py:184)
        self._toc_attempts = toc_attempts
        self._sim_lib = None

    def step(self, action):                                                # dressing.py:12-77
        if self.human.controllable:               # dict in, dicts out (dressing.py:16-17,73-77)
            return self._coop_step(action)
        obs, rew, done, info = self._fused_step(self.id.dressing_step_host, action)
        self.cloth_force_sum = obs[:, 23]
        self.task_success = np.maximum(self.task_success, info[:, 2])
        self.forearm_in_sleeve, self.upperarm_in_sleeve = (info[:, 3].astype(int) & 1) > 0, (info[:, 3].astype(int) & 2) > 0
        return self._unwrap(obs, rew, done, self._info(info[:, 0], info[:, 1].astype(int)))

    # ------------------------------------------------------------------ the same step through the reference-shaped API
    def step_reference_api(self, action):
        """dressing.py:12-77 through the per-call API: take_step (with the person's limits and the anchor update after every
        stepSimulation), then the sleeve-on-arm reward, the cloth forces on the person and the observation, on the host."""
        a = np.asarray(action, dtype=np.float64).reshape(self.n_envs, -1)
        self.take_step(a)
        n = self.n_envs
        x, _ = self.id.cloth_get_state()
        limb = [self._person_pose(link)[0].astype(np.float64) for link in ARM_LINKS]
        forearm, upperarm, reward_dressing = np.zeros(n, dtype=bool), np.zeros(n, dtype=bool), np.zeros(n)
        for e in range(n):
            radii = RADII['male' if self.male[e] else 'female']
            fin, uin, d_fore, d_upper, d_hand, _d_elbow, _d_shoulder, fore_len, upper_len = sleeve_on_arm_reward(
                x[e, TRIANGLE1], x[e, TRIANGLE2], limb[0][e], limb[1][e], limb[2][e], *radii)
            if uin:
                reward_dressing[e] = fore_len + (d_upper if d_upper < upper_len else 0.0)
            elif fin and d_fore < fore_len:
                reward_dressing[e] = d_fore
            else:
                reward_dressing[e] = -d_hand
            forearm[e], upperarm[e] = fin, uin
        self.forearm_in_sleeve, self.upperarm_in_sleeve = forearm, upperarm
        obs = self._get_obs()
        ee_vel = np.linalg.norm(np.atleast_2d(self.robot.get_velocity(self.robot.left_end_effector)), axis=1)
        pref = self.C_v * (-ee_vel) + self.C_d * (-self.cloth_force_sum)          # human_preferences with the dressing forces
        reward = self.config('dressing_reward_weight') * reward_dressing + self.config('action_weight') * (-np.linalg.norm(a, axis=1)) + pref
        self.task_success = np.maximum(self.task_success, reward_dressing)
        done = np.full(n, self.iteration >= 200)
        return self._unwrap(obs, reward, done, self._info(self.total_force_on_human, (self.task_success >= self.config('task_success_threshold')).astype(int)))

    def _get_obs(self, agent=None):                                        # dressing.py:79-106
        ep, eq = (np.atleast_2d(x) for x in self.robot.get_pos_orient(self.robot.left_end_effector))
        ep_r, eq_r = (np.atleast_2d(x) for x in self.robot.convert_to_realworld(ep, eq))
        q = np.atleast_2d(self.robot.get_joint_angles(self.robot.controllable_joint_indices))
        q = (q + np.pi) % (2 * np.pi) - np.pi
        arm = [np.atleast_2d(self.robot.convert_to_realworld(self._person_pose(link)[0])[0]) for link in ARM_LINKS]
        cnt, _node, pos, force, _link = self.id.cloth_get_contacts(1024)
        f = np.linalg.norm(force * 10.0, axis=2)
        keep = (np.arange(f.shape[1])[None, :] < cnt[:, None]) & (pos[:, :, 2] < ep[:, 2:3] - 0.05) & (f < 20)
        self.cloth_force_sum = np.where(keep, f, 0.0).sum(axis=1)
        self.robot_force_on_human = sum(self.id.contact_force_sum(self.robot.body, h.body) for h in self.humans.values()).astype(np.float64)
        self.total_force_on_human = self.robot_force_on_human + self.cloth_force_sum
        robot_obs = np.concatenate([ep_r, eq_r, q] + arm + [self.cloth_force_sum[:, None]], axis=1)
        if agent == 'robot' or not self.human.controllable:
            return robot_obs
        # dressing.py:96-105: the end effector, the person's joint angles (not wrapped) and the arm points in the person's base frame
        qh = self._person_joint_angles()
        ep_h, eq_h = self._person_frame(ep, eq)
        arm_h = [self._person_frame(self._person_pose(link)[0])[0] for link in ARM_LINKS]
        human_obs = np.concatenate([ep_h, eq_h, qh] + arm_h + [self.cloth_force_sum[:, None], self.robot_force_on_human[:, None]], axis=1)
        if agent == 'human':
            return human_obs
        return {'robot': robot_obs, 'human': human_obs}

    def reset(self):                                                       # dressing.py:108-198
        super().reset()
        db = self._db
        if self.id is None:
            self._attach(db, db.wheelchair, BatchSim)
        rng = np.random.default_rng(self.np_random.randint(0, 2 ** 31 - 1))
        self.agents = [self.robot]
        self.robot.motor_gains = self.human.motor_gains = 0.01             # dressing.py:117
        s = db.reset(self.id, rng, sample=self._person_sample(db, rng), attempts=self._toc_attempts)
        self.male = s['male'].astype(bool)
        self.human.gender = 'male' if self.male[0] else 'female'
        self.start_ee_pos = db.start_ee_pos
        if self.human.controllable:               # the start pose is not clipped to the scaled limits here, unlike ScratchItch's and BedBathing's
            self._controllable_person(s['limit_scale'])
            for h in self.humans.values():
                h.motor_gains, h.motor_forces = 0.01, 1.0                         # dressing.py:121; Human.motor_forces
            if self.human_impairment_coop is not None:
                self._person_tremor(s, db.coop_tremor_target(s))
        db.start_fused(self.id, s)
        if self.human.controllable:
            db.start_coop(self.id, s)
        self.task_success = np.zeros(self.n_envs)
        return self._squeeze(self._get_obs())

    def update_targets(self):                                              # dressing.py:200-210
        if self.human.controllable:
            # the person's joint-limit clamps of this stepSimulation move its links (PyBullet's resetJointState does so at once):
            # the observation and the next stepSimulation's cloth see the clamped poses, as k_fk after k_coop_limits gives them
            self.id.forward_kinematics()
        self.id.cloth_anchor_follow(self._db.ee_link)
