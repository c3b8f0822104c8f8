"""`AssistiveEnv` — the reference's gym.Env base class (envs/env.py:20-389) on the batched backend.

Constructor signature, spaces, `seed`, `reset`, `take_step`, `human_preferences`, `config`,
`get_euler/get_quaternion`, `create_sphere(s)` names are kept.  `n_envs` is the one addition:
with n_envs == 1 every method has the reference's shapes; with n_envs > 1 arrays gain a leading
env axis.  The physics client (`p.connect`, env.py:34) is replaced by a `BatchSim` created at the
first `reset` (the scene template is immutable, so `reset` re-randomises state instead of
re-building the world as env.py:92-97 does)."""
import configparser
import os

import numpy as np

from .. import scene as sc_util
from ..gym_compat import gym, seeding, spaces
from .agents.agent import Agent
from .agents.furniture import Furniture
from .agents.human import Human
from .agents.robot import Robot
from .agents.tool import Tool

CONFIG_INI = """
[feeding]
distance_weight = 1.0
action_weight = 0.01
food_reward_weight = 1.0
task_success_threshold = 0.75
[drinking]
distance_weight = 1.0
action_weight = 0.01
cup_tilt_weight = 0.1
drinking_reward_weight = 1.0
task_success_threshold = 0.75
[scratch_itch]
distance_weight = 1.0
action_weight = 0.01
scratch_reward_weight = 1.0
task_success_threshold = 25.0
[bed_bathing]
distance_weight = 1.0
action_weight = 0.01
wiping_reward_weight = 5.0
task_success_threshold = 0.3
[dressing]
dressing_reward_weight = 1.0
action_weight = 0.01
task_success_threshold = 0.4
[human_preferences]
velocity_weight = 0.25
force_nontarget_weight = 0.01
high_forces_weight = 0.05
food_hit_weight = 1.0
food_velocities_weight = 1.0
dressing_force_weight = 0.01
high_pressures_weight = 0.01
[human_male]
mass = 78.4
radius_scale = 1.0
height_scale = 1.0
[human_female]
mass = 62.5
radius_scale = 1.0
height_scale = 1.0
"""

IMPAIRMENTS = ('none', 'limits', 'weakness', 'tremor')      # human.py:80-81, in the order of the reference's np_random.choice


class AssistiveEnv(gym.Env):
    def __init__(self, robot=None, human=None, task='', obs_robot_len=0, obs_human_len=0, time_step=0.02, frame_skip=5,
                 render=False, gravity=-9.81, seed=1001, n_envs=1, device=0, human_impairment=None):
        if human_impairment is not None:
            if not (human is not None and human.controllable):
                raise ValueError('human_impairment selects the impairment of a controllable person (the co-optimisation ids)')
            if human_impairment not in ('random',) + IMPAIRMENTS:
                raise ValueError("human_impairment must be None, 'random' or one of %s" % (IMPAIRMENTS,))
        # None: the person's impairment as each task draws it without the keyword (never 'tremor'); 'random': the reference's
        # four-way draw (human.py:80-81); a name forces that impairment in every env
        self.human_impairment_coop = human_impairment
        self.task = task
        self.time_step, self.frame_skip, self.gravity = time_step, frame_skip, gravity
        self.n_envs, self.device = int(n_envs), device
        self.id = None                 # the BatchSim, created at first reset
        self.gui = False
        self.seed(seed)
        self.action_robot_len = len(robot.controllable_joint_indices) if robot is not None else 0
        self.action_human_len = len(human.controllable_joint_indices) if human is not None and human.controllable else 0
        n_act = self.action_robot_len + self.action_human_len
        self.action_space = spaces.Box(low=np.array([-1.0] * n_act, dtype=np.float32), high=np.array([1.0] * n_act, dtype=np.float32), dtype=np.float32)
        self.obs_robot_len = obs_robot_len
        self.obs_human_len = obs_human_len if human is not None and human.controllable else 0
        n_obs = self.obs_robot_len + self.obs_human_len
        self.observation_space = spaces.Box(low=np.array([-1e9] * n_obs, dtype=np.float32), high=np.array([1e9] * n_obs, dtype=np.float32), dtype=np.float32)
        self.action_space_robot, self.observation_space_robot = self.action_space, self.observation_space
        self.agents = []
        self.plane, self.robot, self.human = Agent(), robot, human
        self.tool, self.furniture = Tool(), Furniture()
        self.configp = configparser.ConfigParser()
        self.configp.read_string(CONFIG_INI)
        hp = 'human_preferences'
        self.C_v, self.C_f, self.C_hf = self.config('velocity_weight', hp), self.config('force_nontarget_weight', hp), self.config('high_forces_weight', hp)
        self.C_fd, self.C_fdv = self.config('food_hit_weight', hp), self.config('food_velocities_weight', hp)
        self.C_d, self.C_p = self.config('dressing_force_weight', hp), self.config('high_pressures_weight', hp)
        self.iteration = 0

    # ---- gym plumbing (env.py:69-89)
    def step(self, action):
        raise NotImplementedError('Implement observations')

    def _get_obs(self, agent=None):
        raise NotImplementedError('Implement observations')

    def config(self, tag, section=None):
        return float(self.configp[self.task if section is None else section][tag])

    def seed(self, seed=None):
        self.np_random, seed = seeding.np_random(seed)
        self._seed = seed
        return [seed]

    def set_seed(self, seed=1000):
        self.np_random.seed(seed)

    def disconnect(self):
        if self.id is not None:
            self.id.close()
            self.id = None

    def close(self):
        self.disconnect()

    def render(self, mode='human'):
        """There is no GUI on this backend (env.py:318-340 opens PyBullet's viewer); with mode='rgb_array' the first env's camera
        image is returned (the collision geometry, ray-cast on the device)."""
        if mode != 'rgb_array' or self.id is None:
            return None
        if getattr(self, 'view', None) is None:
            self.setup_camera()
        return self.get_camera_image_depth()[0]

    def setup_camera(self, camera_eye=(0.5, -0.75, 1.5), camera_target=(-0.2, 0, 0.75), fov=60, camera_width=1920 // 4, camera_height=1080 // 4):
        """env.py:342-346"""
        self.camera_width, self.camera_height = camera_width, camera_height
        self.view = dict(eye=tuple(camera_eye), target=tuple(camera_target), fov=float(fov))

    def setup_camera_rpy(self, camera_target=(-0.2, 0, 0.75), distance=1.5, rpy=(0, -35, 40), fov=60, camera_width=1920 // 4, camera_height=1080 // 4):
        """env.py:348-352 (computeViewMatrixFromYawPitchRoll, up axis z; convention recalled: the eye starts `distance` behind the
        target on -y, is pitched about x and yawed about z; roll is ignored)"""
        pitch, yaw = np.deg2rad(rpy[1]), np.deg2rad(rpy[2])
        off = np.array([0.0, -distance * np.cos(pitch), -distance * np.sin(pitch)])
        off = np.array([np.cos(yaw) * off[0] - np.sin(yaw) * off[1], np.sin(yaw) * off[0] + np.cos(yaw) * off[1], off[2]])
        self.setup_camera(tuple(np.asarray(camera_target) + off), camera_target, fov, camera_width, camera_height)

    def get_camera_image_depth(self, light_pos=(0, -3, 1), shadow=False, ambient=0.8, diffuse=0.3, specular=0.1, env_ids=None):
        """env.py:354-359: (h, w, 4) uint8 image and (h, w) depth buffer; with `env_ids` a leading axis over the requested envs."""
        assert getattr(self, 'view', None) is not None, 'You must call env.setup_camera() or env.setup_camera_rpy() before getting a camera image'
        ids = [0] if env_ids is None else list(env_ids)
        img, depth = self.id.render(self.view['eye'], self.view['target'], fov=self.view['fov'], width=self.camera_width, height=self.camera_height,
                                    env_ids=ids, light_dir=light_pos, ambient=ambient, diffuse=diffuse)
        return (img[0], depth[0]) if env_ids is None else (img, depth)

    def reset(self):
        self.agents = []
        self.iteration = 0
        self.forces = []
        self.task_success = 0

    def get_euler(self, quaternion):
        return sc_util.euler_from_quat(np.asarray(quaternion, dtype=np.float64))

    def get_quaternion(self, euler):
        return sc_util.quat_from_rpy(np.asarray(euler, dtype=np.float64))

    # ---- env.py:174-235
    def take_step(self, actions, gains=None, forces=None, action_multiplier=0.05, step_sim=True):
        """Action -> accumulated PD targets -> frame_skip x stepSimulation, through the per-call API
        (the fused kernels do the same in `FeedingEnv.step`)."""
        if gains is None:
            gains = [a.motor_gains for a in self.agents]
        if forces is None:
            forces = [a.motor_forces for a in self.agents]
        self.iteration += 1
        actions = np.clip(np.asarray(actions, dtype=np.float64).reshape(self.n_envs, -1), self.action_space.low, self.action_space.high) * action_multiplier
        idx = 0
        for i, agent in enumerate(self.agents):
            needs_action = not isinstance(agent, Human) or agent.controllable
            if not needs_action:
                if isinstance(agent, Human) and agent.impairment == 'tremor':     # env.py:212-215
                    sgn = 1.0 if self.iteration % 2 == 0 else -1.0
                    agent.control(agent.controllable_joint_indices, agent.target_joint_angles + agent.tremors * sgn, gains[i], forces[i])
                continue
            k = len(agent.controllable_joint_indices)
            if isinstance(agent, Human):          # the two gender instances of the person share the human part of the action
                action = actions[:, self.action_robot_len:self.action_robot_len + k].copy()
            else:
                action = actions[:, idx:idx + k].copy()
                idx += k
            if isinstance(agent, Robot):
                action *= agent.action_multiplier
            q = np.atleast_2d(agent.get_joint_angles(agent.controllable_joint_indices)).copy()
            lo, hi = agent.controllable_joint_lower_limits, agent.controllable_joint_upper_limits
            # a controllable tremor person (env.py:205-215): per env, the action accumulates into target_joint_angles and the
            # joints are driven to target + tremors x (+-1); the limit checks run against the previous pass's angles
            trem = agent.tremor_mask[:, None] if isinstance(agent, Human) and agent.impairment == 'tremor' else None
            if trem is not None:
                target, wobble = agent.target_joint_angles, agent.tremors * (1.0 if self.iteration % 2 == 0 else -1.0)
            for _ in range(self.frame_skip):
                below, above = q + action < lo, q + action > hi
                action[below | above] = 0
                q = np.where(below, lo, np.where(above, hi, q))
                if trem is None:
                    q = q + action
                else:
                    target = np.where(trem, target + action, target)
                    q = np.where(trem, target + wobble, q + action)
            if trem is not None:
                agent.target_joint_angles = target
            agent.control(agent.controllable_joint_indices, q, gains[i], forces[i])
        if step_sim:
            for _ in range(self.frame_skip):
                self.id.step(1)
                for agent in self.agents:
                    if isinstance(agent, Human):
                        agent.enforce_joint_limits()
                        if agent.controllable:                   # env.py:230-231
                            if agent.impairment == 'tremor':     # its motors drive past the limits: the clamp moves links, at
                                self.id.forward_kinematics()     # once as PyBullet's resetJointState does, before they are read
                            agent.enforce_realistic_joint_limits(getattr(agent, 'env_mask', None))
                self.update_targets()

    def update_targets(self):
        pass

    # ---- what every task env shares around its own observation and reward code
    def _attach(self, batch, furniture, sim_type, sim=None):
        """The Agent objects of `batch`'s scene on `sim` (any object with the BatchSim getter / setter surface; by default a new
        `sim_type` of the scene): the plane, the robot, the tool when the scene has one, `furniture` and both genders' `Human`.
        `sim_type` is the `BatchSim` of the task's module, looked up when the env is reset, so that a test can put the CPU oracle
        in its place."""
        self.id = sim if sim is not None else sim_type(batch.scene, self._cfg, self.n_envs, device=self.device, _lib=self._sim_lib)
        self.plane.init(batch.plane, self.id, self.np_random, indices=-1)
        self.robot.init(batch.robot, self.id, self.np_random)
        if batch.tool is not None:
            self.tool.init(batch.tool, self.id, self.np_random, indices=-1)
        self.furniture.init(furniture, self.id, self.np_random, indices=-1)
        self.humans = {}
        for g, hb in batch.humans.items():
            h = type(self.human)(self.human.controllable_joint_indices, controllable=self.human.controllable)
            h.init(hb, self.id, self.np_random, self.human.controllable_joint_indices)
            self.humans[g] = h

    def _person_sample(self, batch, rng, *args):
        """The reset's sample with `human_impairment` given, else None (the batch's reset draws it, as it always has).  The batch
        draws its sample as without the keyword; then each env's impairment is drawn anew as human.py:80-92 does, and with it the
        `limits` scale, the `weakness` strength and the tremor amplitudes (+-20 deg with the head controllable, +-10 deg for an
        arm, stored at fp32, the precision the device keeps).  Those draws come from a stream jumped ahead of the reset's
        generator, which they leave untouched: for a seed, gender, poses and robot placement are those of the default draw."""
        mode = self.human_impairment_coop
        if mode is None:
            return None
        s = batch.sample(self.n_envs, rng, *args)
        g = np.random.Generator(rng.bit_generator.jumped())
        n, k = self.n_envs, len(self.human.controllable_joint_indices)
        amp = np.deg2rad(20 if Human.head in self.human.controllable_joint_indices else 10)
        imp = g.integers(0, 4, size=n) if mode == 'random' else np.full(n, IMPAIRMENTS.index(mode))
        return dict(s, impairment=imp.astype(np.int32), limit_scale=np.where(imp == 1, g.uniform(0.5, 1.0, size=n), 1.0),
                    strength=np.where(imp == 2, g.uniform(0.25, 1.0, size=n), 1.0),
                    tremors=np.where((imp == 3)[:, None], g.uniform(-amp, amp, size=(n, k)).astype(np.float32).astype(np.float64), 0.0))

    def _person_tremor(self, s, target):
        """The per-call side of a controllable tremor person: each gender instance's tremor mask and amplitudes, and
        target_joint_angles [n, k] as setup_joints takes them at reset (human.py:123)."""
        tremor = np.asarray(s['impairment']) == 3
        for g, h in self.humans.items():
            h.tremor_mask = tremor & (self.male if g == 'male' else ~self.male)
            h.impairment = 'tremor' if h.tremor_mask.any() else 'none'
            h.tremors = np.where(h.tremor_mask[:, None], s['tremors'], 0.0)
            h.target_joint_angles = np.array(target, dtype=np.float64)

    def _controllable_person(self, limit_scale):
        """Both gender instances of the person act; the switched-off one moves nothing (env.py:130).  `limit_scale`: the per-env
        joint-limit scale of impairment 'limits' (human.py:85)."""
        for g, h in self.humans.items():
            h.env_mask = self.male if g == 'male' else ~self.male
            h.arm_previous_valid_pose = {True: None, False: None}
            h.set_limit_scale(limit_scale)
            self.agents.append(h)

    def _person_pose(self, link):
        """world position [n, 3] and orientation [n, 4] of `link` of each env's person (the gender instance `self.male` selects)"""
        pm, qm = (np.atleast_2d(x) for x in self.humans['male'].get_pos_orient(link))
        pf, qf = (np.atleast_2d(x) for x in self.humans['female'].get_pos_orient(link))
        return np.where(self.male[:, None], pm, pf), np.where(self.male[:, None], qm, qf)

    def _person_frame(self, pos, orient=None):
        """[pos, orient] in each env's person's base frame"""
        outs = []
        for g in ('male', 'female'):
            r = self.humans[g].convert_to_realworld(pos, orient if orient is not None else np.array([0, 0, 0, 1.0]))
            outs.append([np.atleast_2d(x) for x in r])
        return [np.where(self.male[:, None], m, f) for m, f in zip(*outs)]

    def _person_joint_angles(self):
        """the controllable joint angles of each env's person, [n, k]"""
        ci = self.human.controllable_joint_indices
        return np.where(self.male[:, None], np.atleast_2d(self.humans['male'].get_joint_angles(ci)), np.atleast_2d(self.humans['female'].get_joint_angles(ci)))

    def _info(self, total_force_on_human, task_success):
        return {'total_force_on_human': total_force_on_human, 'task_success': task_success, 'action_robot_len': self.action_robot_len,
                'action_human_len': self.action_human_len, 'obs_robot_len': self.obs_robot_len, 'obs_human_len': self.obs_human_len}

    def _squeeze(self, a):
        """env 0's value (of every entry of a dict) when n_envs == 1"""
        if isinstance(a, dict):
            return {k: self._squeeze(v) for k, v in a.items()}
        return a[0] if self.n_envs == 1 else a

    def _unwrap(self, obs, reward, done, info):
        """`step`'s return with n_envs == 1: env 0's observation, a float reward, a bool done and env 0's info values"""
        if self.n_envs > 1:
            return obs, reward, done, info
        return self._squeeze(obs), float(reward[0]), bool(done[0]), {k: (v[0] if isinstance(v, np.ndarray) else v) for k, v in info.items()}

    def _by_agent(self, obs, reward, done, info):
        """the co-optimisation `step`'s return: the step's reward, done and info for both agents, and '__all__'"""
        d = bool(np.all(done)) if self.n_envs > 1 else bool(done)
        return obs, {'robot': reward, 'human': reward}, {'robot': done, 'human': done, '__all__': d}, {'robot': info, 'human': info}

    def _coop_step(self, action):
        """`step` with a controllable person, on the per-call path: {'robot': a, 'human': a_h} through `step_reference_api`"""
        n = self.n_envs
        a = np.concatenate([np.asarray(action['robot'], dtype=np.float64).reshape(n, -1), np.asarray(action['human'], dtype=np.float64).reshape(n, -1)], axis=1)
        return self._by_agent(*self.step_reference_api(a))

    def _fused_step(self, step_host, action):
        """One single-agent step on the fused device path (`step_host`, e.g. `self.id.feeding_step_host`): obs [n, obs_robot_len]
        float32, reward [n] float32, done [n] bool and the raw info [n, 4] (force on the person, task success, two task columns)."""
        obs, rew, done, info = step_host(np.asarray(action, dtype=np.float32).reshape(self.n_envs, -1))
        self.iteration += 1
        self.total_force_on_human = info[:, 0]
        return obs, rew, done > 0.5, info

    def step_fused(self, action):
        """The co-optimisation step (dict action in, dict observations / rewards / dones / infos out, as `step` returns them with a
        controllable person) on the fused device path: robot and person act, the person's limits and the realistic-arm-limit
        classifier run on the device after every substep (ag_coop_step_host).  Armed by `reset` (`start_coop`).  `step` itself
        stays on the per-call path."""
        if not (self.human is not None and self.human.controllable):
            raise RuntimeError('step_fused is the co-optimisation step: this env has no controllable person')
        n = self.n_envs
        a = np.concatenate([np.asarray(action['robot'], dtype=np.float32).reshape(n, -1), np.asarray(action['human'], dtype=np.float32).reshape(n, -1)], axis=1)
        obs_r, obs_h, rew, done, info = self.id.coop_step_host(a)
        self.iteration += 1
        self.total_force_on_human = info[:, 0].astype(np.float64)
        obs = self._squeeze({'robot': obs_r.astype(np.float64), 'human': obs_h.astype(np.float64)})
        return self._by_agent(obs, self._squeeze(rew.astype(np.float64)), self._squeeze(done > 0.5), self._info(self.total_force_on_human, info[:, 1].astype(int)))

    # ---- env.py:237-274
    def human_preferences(self, end_effector_velocity=0, total_force_on_human=0, tool_force_at_target=0, food_hit_human_reward=0,
                          food_mouth_velocities=(), dressing_forces=((),), arm_manipulation_tool_forces_on_human=(0, 0),
                          arm_manipulation_total_force_on_human=0):
        reward_velocity = -end_effector_velocity
        reward_high_target_forces = np.where(np.asarray(tool_force_at_target) < 10, 0.0, -np.asarray(tool_force_at_target))
        reward_force_nontarget = -(total_force_on_human - tool_force_at_target)
        if self.task in ['feeding', 'drinking']:
            reward_force_nontarget = -total_force_on_human
        reward_food_hit_human = food_hit_human_reward
        reward_food_velocities = 0 if len(food_mouth_velocities) == 0 else -np.sum(food_mouth_velocities)
        reward_dressing_force = -np.sum(np.linalg.norm(np.asarray(dressing_forces, dtype=np.float64).reshape(-1, 3), axis=-1)) if np.size(dressing_forces) else 0.0
        return (self.C_v * reward_velocity + self.C_f * reward_force_nontarget + self.C_hf * reward_high_target_forces +
                self.C_fd * reward_food_hit_human + self.C_fdv * reward_food_velocities + self.C_d * reward_dressing_force)
