"""`BedBathingEnv` (reference envs/bed_bathing.py) on the batched backend.

`step` runs the fused kernels (`ag_bathing_step_host`): action -> PD targets -> 5 substeps -> obs /
reward / done, wiping targets included.  `step_reference_api` performs the same step the way the
reference does it -- `take_step` + `_get_obs` + `get_total_force` + `human_preferences` through the
per-call `Agent` API, vectorised over `n_envs` (the per-contact Python loop of `get_total_force`,
bed_bathing.py:41-78, becomes one masked distance test of every tool-cloth contact against every
remaining wiping target) -- and exists so that tests can show the two paths agree.

The robot is Sawyer or PR2's left arm, placed by TOC (`bed_bathing_robots_batch.py`).
With a controllable person (co-optimisation, `BedBathingSawyerHuman-v1`, `BedBathingPR2Human-v1`) `step` takes {'robot': a7, 'human': a10} and goes through
the per-call path (`step_reference_api`): `take_step` drives the person's right arm, keeps it inside its (per-env scaled) limits
and the realistic joint limits (human.py:134-152) after every substep, and the wiping targets follow the arm (`update_targets`).
`step_fused` runs the same co-optimisation step on the device (`ag_coop_step_host`).  Deviations: the person is not settled as a
ragdoll at reset (it is lowered onto the mattress, as for the static person), and `tremor` is not drawn for it."""
import numpy as np

from .. import capi
from ..bed_bathing_batch import R_ELBOW, R_SHOULDER, R_WRIST, WIPER_CLOTH_LINK, BedBathingBatch
from ..sim import BatchSim
from .env import AssistiveEnv

MAX_TOOL_CONTACTS = 32
ARM_LINKS = (R_SHOULDER, R_ELBOW, R_WRIST)


def bathing_batch_for(robot, controllable_person):
    """The batched scene of `robot`'s BedBathing id: Sawyer, or PR2 placed by TOC.  BedBathingJaco is not built: the reference
    puts a wheelchair-mounted robot on a nightstand (bed_bathing.py:150-154), a model this backend does not have."""
    from ..bed_bathing_robots_batch import BedBathingPR2Batch
    from .agents.robot import PR2, Sawyer
    for cls, batch in ((Sawyer, BedBathingBatch), (PR2, BedBathingPR2Batch)):
        if type(robot) is cls:
            return batch(controllable_person=controllable_person)
    raise KeyError('BedBathing is not built for %s' % type(robot).__name__)


class BedBathingEnv(AssistiveEnv):
    def __init__(self, robot, human, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=robot, human=human, task='bed_bathing', n_envs=n_envs, device=device, seed=seed,
                         obs_robot_len=(17 + len(robot.controllable_joint_indices) - (len(robot.wheel_joint_indices) if robot.mobile else 0)),
                         obs_human_len=(18 + len(human.controllable_joint_indices)))
        self._bb = bathing_batch_for(robot, human.controllable)
        self._cfg = config or capi.default_config()
        self._sim_lib = None

    # ------------------------------------------------------------------ fused step (bed_bathing.py:12-39)
    def step(self, action):
        if self.human.controllable:               # dict in, dicts out (bed_bathing.py:13-14,35-39)
            return self._coop_step(action)
        obs, rew, done, info = self._fused_step(self.id.bathing_step_host, action)
        self.tool_force_on_human, self.new_contact_points = info[:, 2], info[:, 3].astype(int)
        self.task_success += self.new_contact_points
        return self._unwrap(obs, rew, done, self._info(info[:, 0], info[:, 1].astype(int)))

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
        return self._unwrap(obs, reward, done, self._info(self.total_force_on_human, success))

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
        arm = [np.atleast_2d(self.robot.convert_to_realworld(self._person_pose(link)[0])[0]) for link in ARM_LINKS]
        self.tool_force, self.tool_force_on_human, self.total_force_on_human, self.new_contact_points = self.get_total_force()
        robot_obs = np.concatenate([tp_r, tq_r, q] + arm + [self.tool_force[:, None]], axis=1)
        if agent == 'robot' or not self.human.controllable:
            return robot_obs
        # bed_bathing.py:99-105: the wiper, the person's joint angles (not wrapped) and the arm points in the person's base frame
        qh = self._person_joint_angles()
        tp_h, tq_h = self._person_frame(tp, tq)
        arm_h = [self._person_frame(self._person_pose(link)[0])[0] for link in ARM_LINKS]
        human_obs = np.concatenate([tp_h, tq_h, qh] + arm_h + [np.asarray(self.total_force_on_human, dtype=np.float64)[:, None],
                                                              np.asarray(self.tool_force_on_human, dtype=np.float64)[:, None]], axis=1)
        if agent == 'human':
            return human_obs
        return {'robot': robot_obs, 'human': human_obs}

    # ------------------------------------------------------------------ reset (bed_bathing.py:113-168)
    def reset(self):
        super().reset()
        bb = self._bb
        if self.id is None:
            self._attach(bb, bb.bed, BatchSim)
        rng = np.random.default_rng(self.np_random.randint(0, 2 ** 31 - 1))
        self.agents = [self.robot]
        s = bb.reset(self.id, rng)
        self.male = s['male'].astype(bool)
        self.human.gender = 'male' if self.male[0] else 'female'
        if self.human.controllable:
            self._controllable_person(s['limit_scale'])
            for h in self.humans.values():
                h.enforce_joint_limits(h.controllable_joint_indices)              # the start pose is clipped to them (human.py:115)
            self.id.forward_kinematics()
        self.generate_targets(s)
        if self.human.controllable:
            bb.start_coop(self.id, s)
        self.task_success = np.zeros(self.n_envs, dtype=int)
        return self._squeeze(self._get_obs())

    def generate_targets(self, s):                                         # bed_bathing.py:173-203
        self.targets_pos_world, self.targets_alive = self._bb.start_fused(self.id, s)
        self.total_target_count = self.targets_alive.sum(axis=1)

    def update_targets(self):                                              # bed_bathing.py:190-203
        if not self.human.controllable:
            return     # the person is static after reset: the world positions computed in generate_targets stay valid
        self.targets_pos_world = self._bb.targets_world(self.id, {'male': self.male})[0]
