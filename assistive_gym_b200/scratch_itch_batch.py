"""ScratchItchJaco-v1 as a batched scene: template construction and batched reset (SURVEY.md section 8(f)3).

Restates `ScratchItchEnv.reset` (reference envs/scratch_itch.py:93-153) and what it calls: `build_assistive_env('wheelchair')`
(envs/env.py:114-134), `Human.setup_joints(..., reactive_force=1, reactive_gain=0.01)` (agents/human.py:104-127: the person's
right arm is simulated and held by weak position motors), `Tool.init` (agents/tool.py:10-47: scratcher/tool_scratch.urdf on a
fixed constraint to the Jaco tool joint), `init_robot_pose` -> `Robot.ik_random_restarts` (envs/env.py:276-310), `generate_target`
(scratch_itch.py:134-147, util.point_on_capsule util.py:58-78).  As in the other tasks both genders are instantiated and one
is switched off per env; the person's `tremor` impairment is not drawn by default (a controllable person's with `human_impairment`, `start_coop`), `weakness` scales the arm's motor force."""
import numpy as np

from . import capi
from .feeding_batch import JACO as FEED_JACO
from .feeding_batch import coop_params, pack_mlp
from .human_model import create_human
from .kinematics import BodyKinematics, q_from_rpy, q_mul, q_rot
from .scene import SceneBuilder, quat_from_rpy

MOTOR_POSITION = 1
JACO = dict(FEED_JACO, gripper_pos=1.0, tool_pos_offset=[0, 0, 0.02], tool_orient_offset=[0, -np.pi / 2.0, 0], ee_orient_rpy=[0, np.pi / 2.0, 0])   # jaco.py:19-42
RIGHT_ARM_JOINTS = list(range(0, 10))                    # human.right_arm_joints (scratch_itch_envs.py:15)
R_SHOULDER, R_ELBOW, R_WRIST = 5, 7, 9
R_ARM_LIMIT_JOINTS = [3, 4, 5, 6]                        # shoulder x, y, z and elbow: the classifier's inputs (human.py:137-140)
HUMAN_PRESET = {3: 30, 6: -90, 16: -90, 28: -90, 31: 80, 35: -90, 38: 80}      # degrees, scratch_itch.py:104
LIMBS = {'male': ((R_SHOULDER, 0.279, 0.043), (R_ELBOW, 0.257, 0.033)), 'female': ((R_SHOULDER, 0.264, 0.0355), (R_ELBOW, 0.234, 0.027))}   # scratch_itch.py:136-139


def point_on_capsule(rng, length, radius, n):
    """util.point_on_capsule (util.py:58-78) for p1 = 0, p2 = (0, 0, -length): `n` random points on the cylinder wall."""
    rl = rng.uniform(radius, length, size=n)
    theta = rng.uniform(0, 2 * np.pi, size=n)
    axis = np.array([0.0, 0.0, -1.0])
    ortho = np.array([1.0, 0.0, 0.0])                    # util.orthogonal_vector of the z axis (any unit vector orthogonal to it serves)
    normal = np.cross(axis, ortho)
    return rl[:, None] * axis + radius * np.cos(theta)[:, None] * ortho + radius * np.sin(theta)[:, None] * normal


class ScratchItchBatch:
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
                if j not in RIGHT_ARM_JOINTS:
                    b.change_dynamics(hb, j, mass=0)
            b.set_gravity([0, 0, 0], body=hb)                                       # scratch_itch.py:123
            self.humans[gender] = hb
        self.wheelchair = b.load_urdf('wheelchair_jaco', base_pos=wheelchair_pos, fixed_base=False)
        self.tool = b.load_urdf('tool_scratch')
        for j in JACO['gripper_collision']:                                          # tool.py:41-44
            for tj in (-1, 0, 1):
                b.set_collision_filter_pair(self.robot, self.tool, j, tj, False)
        self.tool_pos_offset = np.array(JACO['tool_pos_offset'], dtype=np.float64)
        self.tool_quat_offset = quat_from_rpy(JACO['tool_orient_offset'])
        b.create_fixed_constraint(self.robot, JACO['tool_joint'], self.tool, -1, self.tool_pos_offset, [0, 0, 0], self.tool_quat_offset, [0, 0, 0, 1], max_force=500)
        b.set_gravity([0, 0, 0], body=self.robot)
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
        self.human_arm_links = {g: [self.gl(hb, j) for j in RIGHT_ARM_JOINTS] for g, hb in self.humans.items()}

    def scratch_params(self):
        P = capi.AgScratchParams()
        P.robot_body, P.tool_body = self.robot, self.tool
        P.human_body_m, P.human_body_f = self.humans['male'], self.humans['female']
        for i, l in enumerate(self.arm_links):
            P.arm_links[i] = l; P.arm_lower[i] = self.arm_lower[i]; P.arm_upper[i] = self.arm_upper[i]
        P.ee_link = self.ee_link
        P.tool_link0, P.tool_tip_link = self.gl(self.tool, 0), self.gl(self.tool, 1)
        for i, l in enumerate((R_SHOULDER, R_ELBOW, R_WRIST)):
            P.arm_points_m[i] = self.gl(self.humans['male'], l); P.arm_points_f[i] = self.gl(self.humans['female'], l)
        P.action_multiplier, P.frame_skip = 0.05, 5
        P.w_distance, P.w_action, P.w_scratch = 1.0, 0.01, 1.0            # config.ini [scratch_itch]
        P.c_v, P.c_f, P.c_hf = 0.25, 0.01, 0.05                           # config.ini [human_preferences]
        P.task_success_threshold = 25.0
        return P

    def sample(self, n, rng):
        male = rng.integers(0, 2, size=n).astype(np.int32)
        limb = rng.integers(0, 2, size=n)                                 # np_random.randint(2) (scratch_itch.py:136)
        tl = np.zeros((n, 3)); limb_joint = np.zeros(n, dtype=int)
        for g, is_m in (('male', 1), ('female', 0)):
            for k in (0, 1):
                sel = (male == is_m) & (limb == k)
                lj, length, radius = LIMBS[g][k]
                tl[sel] = point_on_capsule(rng, length, radius, int(sel.sum()))
                limb_joint[sel] = lj
        imp = rng.integers(0, 3, size=n)                                  # none / limits / weakness ('no_tremor', human.py:82-83)
        s = dict(plane_friction=rng.uniform(0.025, 0.5, size=n), male=male, limb_joint=limb_joint, target_local=tl,
                 impairment=imp.astype(np.int32), strength=np.where(imp == 2, rng.uniform(0.25, 1.0, size=n), 1.0),
                 ee_offset=rng.uniform(-0.05, 0.05, size=(n, 3)))
        s['limit_scale'] = np.where(imp == 1, rng.uniform(0.5, 1.0, size=n), 1.0)      # human.py:85 (drawn last: the other fields keep their values)
        return s

    def place_tool(self, sim, qfull):
        n = sim.n
        pos, quat = self.kin.fk(np.broadcast_to(self.robot_base_pos, (n, 3)), np.broadcast_to(self.robot_base_quat, (n, 4)), qfull)
        cp, cq = self.kin.link_com_pose(pos, quat, JACO['tool_joint'] + 1)
        sim.set_base_pose(self.tool, cp + q_rot(cq, self.tool_pos_offset), q_mul(cq, np.broadcast_to(self.tool_quat_offset, (n, 4))))
        sim.set_base_velocity(self.tool, np.zeros((n, 3)), np.zeros((n, 3)))

    def reset(self, sim, rng, sample=None):
        n = sim.n
        s = sample or self.sample(n, rng)
        self.last_sample = s
        self._reset_person(sim, s)
        self._reset_mounted_arm(sim, s, rng)
        return s

    def _reset_person(self, sim, s):
        """Floor friction, both genders at ScratchItch's preset pose (one active per env), the right arm held by weak motors."""
        n = sim.n
        sc = self.scene
        male = s['male'].astype(bool)
        sim.set_link_friction(int(sc['body_link0'][self.plane]), s['plane_friction'])
        for g, hb in self.humans.items():
            nj = int(sc['body_nlinks'][hb]) - 1
            links = [self.gl(hb, j) for j in range(nj)]
            q = np.zeros(nj)
            for j, deg in HUMAN_PRESET.items():
                q[j] = np.deg2rad(deg)
            q = np.clip(q, sc['link_lower'][links], sc['link_upper'][links])
            qn = np.tile(q, (n, 1))
            sim.set_joint_state(links, q=qn, qd=np.zeros_like(qn))
            sim.set_body_active(hb, np.where(male if g == 'male' else ~male, 1, 0).astype(np.int32))
            al = self.human_arm_links[g]
            sim.set_motor(al, MOTOR_POSITION, target=np.tile(q[RIGHT_ARM_JOINTS], (n, 1)), kp=[0.01] * 10, kd=[1.0] * 10, max_force=[1.0] * 10)   # human.py:124-127
            sim.set_motor_force_scale(al, np.repeat(s['strength'][:, None], 10, axis=1))

    def _reset_mounted_arm(self, sim, s, rng):
        n = sim.n
        # robot: IK to the randomised end-effector pose, resampled while arm or tool touch the person / wheelchair (env.py:296-309)
        target = np.array([-0.6, 0, 0.8]) + s['ee_offset']
        tq = q_from_rpy(JACO['ee_orient_rpy'])
        gq = np.full((n, 3), JACO['gripper_pos'])
        sim.set_joint_state(self.gripper_links, q=gq, qd=np.zeros_like(gq))
        arm_local = np.array(JACO['arm']) + 1
        if 'q7' in s:
            q7, self.ik_err = s['q7'].copy(), s.get('ik_err', np.zeros(n))
            todo = np.zeros(n, dtype=bool)
        else:
            q7 = np.zeros((n, 7)); self.ik_err = np.full(n, np.inf); todo = np.ones(n, dtype=bool)
        obstacles = [self.humans['male'], self.humans['female'], self.wheelchair]
        for attempt in range(30):
            if todo.any():
                q, err = sim.ik_solve(self.arm_links, self.ee_link, target, tq, max_restarts=20, iters=120, threshold=0.01,
                                      seed=int(rng.integers(1, 2 ** 31 - 1)), mask=todo.astype(np.int32))
                q7[todo], self.ik_err[todo] = q[todo], err[todo]
            sim.set_joint_state(self.arm_links, q=q7, qd=np.zeros_like(q7))
            qfull = np.zeros((n, self.kin.nl)); qfull[:, arm_local] = q7; qfull[:, np.array(JACO['gripper']) + 1] = JACO['gripper_pos']
            self.place_tool(sim, qfull)
            sim.forward_kinematics()
            if 'q7' in s:
                break
            hit = np.zeros(n, dtype=bool)
            for ob in obstacles:
                hit |= sim.closest_points(self.robot, ob, 0.0, max_pts=1)[1] > 0
                hit |= sim.closest_points(self.tool, ob, 0.0, max_pts=1)[1] > 0
            todo = hit
            if not todo.any():
                break
        self.unresolved = int(todo.sum())
        s['q7'], s['ik_err'] = q7.copy(), self.ik_err.copy()
        sim.set_motor(self.arm_links, MOTOR_POSITION, target=q7, kp=[0.05] * 7, kd=[1.0] * 7, max_force=[1.0] * 7)          # robot.py:36-37
        sim.set_motor(self.gripper_links, MOTOR_POSITION, target=gq, kp=[0.05] * 3, kd=[1.0] * 3, max_force=[500.0] * 3)
        sim.forward_kinematics()

    def limb_links(self, s):
        male = s['male'].astype(bool)
        return np.array([self.gl(self.humans['male' if male[e] else 'female'], int(s['limb_joint'][e])) for e in range(len(male))], dtype=np.int32)

    def start_fused(self, sim, sample=None):
        s = sample or self.last_sample
        sim.scratch_init(self.scratch_params(), s['male'], self.limb_links(s), s['target_local'])

    def start_coop(self, sim, sample=None):
        """Arm the person's half of the fused co-optimisation step (ScratchItchJacoHuman-v1); call after `start_fused`.  The arm
        is driven with Human.motor_gains / motor_forces (0.05, 1.0), which take_step re-issues every step in place of the reset's
        0.01; the `weakness` force scale set by `reset` stays.  Limits are scaled by the sample's `limit_scale`; the right arm is
        kept inside the realistic joint limits by the classifier of limits_model."""
        from .limits_model import load_model
        s = sample or self.last_sample
        P = coop_params(self.scene, self.humans, 1, RIGHT_ARM_JOINTS, 0.05)
        w = pack_mlp(P, load_model(), R_ARM_LIMIT_JOINTS, -1.0)
        sim.coop_init(P, limit_scale=s.get('limit_scale'), mlp=w)
        imp = s.get('impairment')
        if imp is not None and np.any(imp == 3):       # a tremor person (human_impairment given to the env)
            sim.coop_set_tremor(imp == 3, self.coop_tremor_target(s), s['tremors'])

    def coop_tremor_target(self, s):
        """target_joint_angles [n, 10] of a controllable tremor person (human.py:123): the right arm's preset, clipped to the
        limits; a tremor person's limits are not scaled, so ScratchItchEnv.reset's clip leaves it as it is"""
        male = s['male'].astype(bool)
        out = np.zeros((len(male), len(RIGHT_ARM_JOINTS)))
        for g, hb in self.humans.items():
            nj = int(self.scene['body_nlinks'][hb]) - 1
            links = [self.gl(hb, j) for j in range(nj)]
            q = np.zeros(nj)
            for j, deg in HUMAN_PRESET.items():
                q[j] = np.deg2rad(deg)
            q = np.clip(q, self.scene['link_lower'][links], self.scene['link_upper'][links])
            out[male if g == 'male' else ~male] = q[RIGHT_ARM_JOINTS]
        return out
