"""DrinkingJaco-v1 as a batched scene: template construction and batched reset.

Restates `DrinkingEnv.reset` (reference envs/drinking.py:119-183) and what it calls (the same helpers as Feeding: `build_assistive_env`
env.py:114-134, `Human.init/setup_joints` human.py:72-127, `Tool.init` tool.py:10-54 with the coffee cup at scale 0.045,
`init_robot_pose` env.py:276-310).  The scene is Feeding's without table and bowl, with the cup instead of the spoon and 64 water
particles (4 x 4 x 4 spheres of radius 5 mm, 1 g) instead of 8 food particles; `numSubSteps = 4`, `numSolverIterations = 10`
(drinking.py:157) are `config()`.

Status: per-call API path (`DrinkingEnv.step`) and the fused device step (`start_fused`, `ag_drinking_step_*`, ag_drinking.cuh,
`DrinkingEnv.step_fused`, `AssistiveVecEnv`); both replay the reference's own rollout (tests/test_reference_drinking_semantics.py,
tests/test_drinking_fused.py), the fused step on the H100 too; its rate is tools/gpu_drinking_bench.py's."""
import numpy as np

from . import capi
from .feeding_batch import HEAD_JOINTS, HEAD_LINK, HUMAN_PRESET, IMPAIRMENTS, TREMOR_JOINTS, FeedingBatch
from .human_model import create_human
from .kinematics import BodyKinematics, q_from_rpy, q_mul, q_rot
from .scene import SceneBuilder, quat_from_rpy

MOTOR_POSITION = 1
JACO = dict(arm=[1, 2, 3, 4, 5, 6, 7], ee=8, gripper=[9, 11, 13], tool_joint=8, gripper_collision=list(range(7, 15)),
            gripper_pos=0.63, tool_pos_offset=[0.05, -0.005, 0], tool_orient_offset=[0, -np.pi / 2.0, np.pi / 2.0],
            base_offset=[-0.35, -0.3, 0.3], ee_orient_rpy=[0, np.pi / 2.0, 0])          # jaco.py:19-47, task 'drinking'
WATER_RADIUS, WATER_MASS, N_WATER = 0.005, 0.001, 64                                     # drinking.py:160-168
CUP_TOP_CENTER_OFFSET, CUP_BOTTOM_CENTER_OFFSET = np.array([0, 0, -0.055]), np.array([0, 0, 0.07])      # drinking.py:137-138


class DrinkingBatch(FeedingBatch):
    """Shares `sample`, `solve_ik` and the tremor helpers with `FeedingBatch` (the person, the robot and the wheelchair are the same)."""

    def __init__(self):
        b = SceneBuilder()
        self.builder = b
        b.set_gravity([0, 0, -9.81])
        self.plane = b.load_urdf('plane')
        wheelchair_pos = np.array([0, 0, 0.06])
        self.robot_base_pos = wheelchair_pos + np.array(JACO['base_offset'])
        self.robot_base_quat = quat_from_rpy([0, 0, -np.pi / 2.0])
        self.robot = b.load_urdf('jaco', base_pos=self.robot_base_pos, base_quat=self.robot_base_quat, fixed_base=True, self_collision=True)
        self.humans = {}
        for gender, z in (('male', 0.89), ('female', 0.86)):
            hb, info = create_human(b, gender=gender, static=True)
            b.bodies[hb].base_pos = np.array([0, 0.03, z])
            for j in range(b.num_joints(hb)):
                if j not in TREMOR_JOINTS:
                    b.change_dynamics(hb, j, mass=0)
            self.humans[gender] = hb
        self.wheelchair = b.load_urdf('wheelchair_jaco', base_pos=wheelchair_pos, fixed_base=False)
        cup_shape = b.create_collision_shape('mesh', mesh_asset='cup_vhacd', mesh_scale=[0.045] * 3)          # tool.py:23-34, drinking.py:136
        self.tool = b.create_multibody(base_mass=1.0, base_shape=cup_shape, name='cup')
        for j in JACO['gripper_collision']:
            b.set_collision_filter_pair(self.robot, self.tool, j, -1, False)
        self.tool_pos_offset = np.array(JACO['tool_pos_offset'], dtype=np.float64)
        self.tool_quat_offset = quat_from_rpy(JACO['tool_orient_offset'])
        b.create_fixed_constraint(self.robot, JACO['tool_joint'], self.tool, -1, self.tool_pos_offset, [0, 0, 0], self.tool_quat_offset, [0, 0, 0, 1], max_force=500)
        ws = b.create_collision_shape('sphere', radius=WATER_RADIUS)
        self.waters = [b.create_multibody(base_mass=WATER_MASS, base_shape=ws, name='water%d' % i) for i in range(N_WATER)]
        self.foods = self.waters                                                # (FeedingBatch helpers iterate `foods`)
        b.set_gravity([0, 0, 0], body=self.robot)
        for hb in self.humans.values():
            b.set_gravity([0, 0, 0], body=hb)
        b.set_gravity([0, 0, 0], body=self.tool)
        self.scene = b.finalize()
        sc = self.scene
        self.gl = lambda body, link: int(sc['body_link0'][body]) + 1 + link
        self.arm_links = [self.gl(self.robot, j) for j in JACO['arm']]
        self.gripper_links = [self.gl(self.robot, j) for j in JACO['gripper']]
        self.ee_link = self.gl(self.robot, JACO['ee'])
        self.kin = BodyKinematics(sc, self.robot)
        self.arm_lower = sc['link_lower'][self.arm_links].copy()
        self.arm_upper = sc['link_upper'][self.arm_links].copy()
        self.hkin = {g: BodyKinematics(sc, hb) for g, hb in self.humans.items()}
        self.mouth = {'male': np.array([0, -0.11, 0.03]), 'female': np.array([0, -0.1, 0.03])}          # drinking.py:187

    @staticmethod
    def config(**kw):
        """drinking.py:157: four substeps per stepSimulation, ten solver iterations; a contact budget for 64 particles in a cup."""
        return capi.default_config(**dict(dict(num_substeps=4, num_solver_iters=10, max_contacts=512), **kw))

    def drinking_params(self, seed=1001):
        """AgDrinkingParams of the fused step; the weights are the per-call env's (config.ini [drinking], [human_preferences])."""
        import configparser
        from .envs.env import CONFIG_INI
        cfg = configparser.ConfigParser()
        cfg.read_string(CONFIG_INI)
        d, hp = cfg['drinking'], cfg['human_preferences']
        P = capi.AgDrinkingParams()
        P.robot_body, P.tool_body = self.robot, self.tool
        P.human_body_m, P.human_body_f = self.humans['male'], self.humans['female']
        for i, l in enumerate(self.arm_links):
            P.arm_links[i], P.arm_lower[i], P.arm_upper[i] = l, self.arm_lower[i], self.arm_upper[i]
        P.ee_link = self.ee_link
        P.head_link_m, P.head_link_f = self.gl(self.humans['male'], HEAD_LINK), self.gl(self.humans['female'], HEAD_LINK)
        P.water_body0, P.n_water = self.waters[0], len(self.waters)
        if list(self.waters) != list(range(self.waters[0], self.waters[0] + len(self.waters))):
            raise ValueError('the water particles must be consecutive bodies')
        fp, fq = self.cup_frame(np.zeros((1, 3)), np.array([[0, 0, 0, 1.0]]))
        for i in range(3):
            P.mouth_m[i], P.mouth_f[i] = self.mouth['male'][i], self.mouth['female'][i]
            P.cup_frame_pos[i] = fp[0, i]
            P.cup_top[i], P.cup_bottom[i] = CUP_TOP_CENTER_OFFSET[i], CUP_BOTTOM_CENTER_OFFSET[i]
        for i in range(4):
            P.cup_frame_quat[i] = fq[0, i]
        P.action_multiplier, P.frame_skip = 0.05, 5
        P.w_distance, P.w_action = float(d['distance_weight']), float(d['action_weight'])
        P.w_cup_tilt, P.w_drinking = float(d['cup_tilt_weight']), float(d['drinking_reward_weight'])
        P.c_v, P.c_f, P.c_hf = float(hp['velocity_weight']), float(hp['force_nontarget_weight']), float(hp['high_forces_weight'])
        P.c_fd, P.c_fdv = float(hp['food_hit_weight']), float(hp['food_velocities_weight'])
        P.task_success_threshold = float(d['task_success_threshold'])
        P.seed = seed
        return P

    def start_fused(self, sim, sample=None, seed=1001):
        """Arm the fused step (`sim.drinking_step_*`) for the envs last put in place by `reset` (or `sample`): a new episode with
        every particle in play.  Draws nothing from the reset's generator."""
        s = sample or self.last_sample
        sim.drinking_init(self.drinking_params(seed), s['male'])

    def cup_frame(self, cup_pos, cup_quat):
        """drinking.py:25-26: the cup's frame used for its top / bottom centres: shifted by (0, 0.06, 0) and turned by 90 degrees about x."""
        p = cup_pos + q_rot(cup_quat, np.array([0, 0.06, 0.0]))
        q = q_mul(cup_quat, np.broadcast_to(q_from_rpy([np.pi / 2.0, 0, 0]), cup_quat.shape))
        return p, q

    def reset(self, sim, rng, settle_steps=50, sample=None, impairment='random', simulate_head=False):
        n = sim.n
        s = sample or self.sample(n, rng, impairment)
        self.last_sample = s
        self._reset_person(sim, s, simulate_head)
        self._reset_mounted_arm(sim, s, rng)
        self._reset_water(sim, settle_steps)
        return s

    def _reset_person(self, sim, s, simulate_head):
        """Floor friction, both genders at Feeding's presets with the sampled head pose (one active per env), the head joints held by
        weak motors."""
        n = sim.n
        sc = self.scene
        male = s['male'].astype(bool)
        tremor = s['impairment'] == 3
        sim.set_link_friction(int(sc['body_link0'][self.plane]), s['plane_friction'])
        for gender, hb in self.humans.items():
            nl = int(sc['body_nlinks'][hb])
            q = np.zeros((n, nl - 1))
            for j, deg in HUMAN_PRESET.items():                                  # drinking.py:128: the same presets as Feeding
                q[:, j] = np.deg2rad(deg)
            for c, j in enumerate(HEAD_JOINTS):
                q[:, j] = np.deg2rad(s['head_deg'][:, c])
            links = [self.gl(hb, j) for j in range(nl - 1)]
            q = np.clip(q, sc['link_lower'][links], sc['link_upper'][links])
            sim.set_joint_state(links, q=q, qd=np.zeros_like(q))
            on = male if gender == 'male' else ~male
            sim.set_body_active(hb, np.where(on, np.where(tremor | simulate_head, 1, 2), 0).astype(np.int32))
            hl = [self.gl(hb, j) for j in TREMOR_JOINTS]
            sim.set_motor(hl, MOTOR_POSITION, target=q[:, list(TREMOR_JOINTS)], kp=[0.005] * 4, kd=[1.0] * 4, max_force=[1.0] * 4)     # drinking.py:126
            sim.set_hard_limits(hl, True)

    def _reset_mounted_arm(self, sim, s, rng):
        n = sim.n
        gq0 = np.full((n, 3), JACO['gripper_pos'])
        sim.set_joint_state(self.gripper_links, q=gq0, qd=np.zeros_like(gq0))
        if 'q7' in s:
            arm_q = s['q7'].copy()
            self.ik_colliding = 0
        else:
            # start pose of the arm: IK to the randomised goal, resampled while the arm or the cup touch the person or the wheelchair
            # (ik_random_restarts with collision_objects, robot.py:107-112; env.py:300-309)
            target = np.array([-0.2, -0.5, 1.1]) + s['ee_offset']              # drinking.py:140
            arm_q, self.ik_err = self._solve_ik_drinking(n, target, rng, sim, None)
            obstacles = [self.humans['male'], self.humans['female'], self.wheelchair]
            hit = np.zeros(n, dtype=bool)
            for attempt in range(30):
                sim.set_joint_state(self.arm_links, q=arm_q, qd=np.zeros_like(arm_q))
                self._place_cup(sim, arm_q)
                sim.forward_kinematics()
                hit = np.zeros(n, dtype=bool)
                for ob in obstacles:
                    hit |= sim.closest_points(self.robot, ob, 0.0, max_pts=1)[1] > 0
                    hit |= sim.closest_points(self.tool, ob, 0.0, max_pts=1)[1] > 0
                if not hit.any():
                    break
                q2, e2 = self._solve_ik_drinking(n, target, rng, sim, hit)
                arm_q[hit], self.ik_err[hit] = q2[hit], e2[hit]
            self.ik_colliding = int(hit.sum())
            s['q7'] = arm_q.copy()
        gq = np.full((n, 3), JACO['gripper_pos'])
        sim.set_joint_state(self.gripper_links, q=gq, qd=np.zeros_like(gq))
        sim.set_joint_state(self.arm_links, q=arm_q, qd=np.zeros_like(arm_q))
        sim.set_motor(self.arm_links, MOTOR_POSITION, target=arm_q, kp=[0.005] * 7, kd=[1.0] * 7, max_force=[1.0] * 7)              # drinking.py:126
        sim.set_motor(self.gripper_links, MOTOR_POSITION, target=gq, kp=[0.05] * 3, kd=[1.0] * 3, max_force=[500.0] * 3)
        self._place_cup(sim, arm_q)

    def _reset_water(self, sim, settle_steps):
        """The 4 x 4 x 4 water grid over the cup's centre of mass, then the settle."""
        n = sim.n
        sc = self.scene
        zero3 = np.zeros((n, 3))
        # water above the cup (drinking.py:159-168): the cup's base position is its centre of mass frame, as PyBullet reports it
        sim.forward_kinematics()
        cup_com = sim.get_link_states([int(sc['body_link0'][self.tool])])['com_pos'][:, 0].astype(np.float64)
        k = 0
        for i in range(4):
            for j in range(4):
                for l in range(4):
                    wp = cup_com + np.array([i * 2 * WATER_RADIUS - 0.02, j * 2 * WATER_RADIUS - 0.02, l * 2 * WATER_RADIUS + 0.075])
                    sim.set_base_pose(self.waters[k], wp, np.array([0, 0, 0, 1.0]))
                    sim.set_base_velocity(self.waters[k], zero3, zero3)
                    k += 1
        sim.forward_kinematics()
        if settle_steps:
            sim.step(settle_steps)                                              # "drop water in the cup" (drinking.py:175-176)

    def _place_cup(self, sim, arm_q):
        """the cup at the tool joint's COM frame composed with the offsets (tool.py:49-54)"""
        n = sim.n
        qfull = np.zeros((n, self.kin.nl)); qfull[:, np.array(JACO['arm']) + 1] = arm_q; qfull[:, np.array(JACO['gripper']) + 1] = JACO['gripper_pos']
        pos, quat = self.kin.fk(np.broadcast_to(self.robot_base_pos, (n, 3)), np.broadcast_to(self.robot_base_quat, (n, 4)), qfull)
        cp, cq = self.kin.link_com_pose(pos, quat, JACO['tool_joint'] + 1)
        sp = cp + q_rot(cq, self.tool_pos_offset)
        sq = q_mul(cq, np.broadcast_to(self.tool_quat_offset, (n, 4)))
        sim.set_base_pose(self.tool, sp, sq)
        sim.set_base_velocity(self.tool, np.zeros((n, 3)), np.zeros((n, 3)))
        return sp, sq

    def _solve_ik_drinking(self, n, target, rng, sim, mask=None):
        """start pose of the arm: the task's end-effector orientation at the randomised position (env.py:296, robot.py:84-121)"""
        tq = q_from_rpy(JACO['ee_orient_rpy'])
        if hasattr(sim, 'ik_solve'):
            q7, err = sim.ik_solve(self.arm_links, self.ee_link, target, tq, max_restarts=20, iters=120, threshold=0.01, seed=int(rng.integers(1, 2 ** 31 - 1)),
                                   mask=None if mask is None else mask.astype(np.int32))
            return q7.astype(np.float64), err.astype(np.float64)
        from .kinematics import ik_dls
        joints = np.array(JACO['arm']) + 1
        best_q, best_e = np.zeros((n, 7)), np.full(n, np.inf)
        bp, bq = np.broadcast_to(self.robot_base_pos, (n, 3)), np.broadcast_to(self.robot_base_quat, (n, 4))
        for r in range(100):                                                    # (the reference allows up to 1000 restarts, robot.py:84-121)
            q0 = np.zeros((n, self.kin.nl)); q0[:, joints] = rng.uniform(self.arm_lower, self.arm_upper, size=(n, 7))
            q, pe, oe = ik_dls(self.kin, bp, bq, q0, joints, JACO['ee'] + 1, target, np.broadcast_to(tq, (n, 4)).copy(), self.arm_lower, self.arm_upper, iters=120)
            e = np.maximum(pe, oe)
            better = e < best_e
            best_q[better], best_e[better] = q[better][:, joints], e[better]
            if np.all(best_e < 0.01):
                break
        return best_q, best_e

