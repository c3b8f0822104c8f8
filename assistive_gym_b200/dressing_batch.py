"""DressingPR2-v1 as a batched scene: template construction, batched reset, cloth placement.

Restates `DressingEnv.reset` (reference envs/dressing.py:108-198) and what it calls: `build_assistive_env('wheelchair_left')`
(envs/env.py:114-134), `Human.setup_joints` (agents/human.py:104-127), `PR2.init / reset_joints` (agents/pr2.py:51-69),
`init_robot_pose` -> `Robot.position_robot_toc` (envs/env.py:276-310, agents/robot.py:123-235: random base poses ranked by
goals reached and joint-limit-weighted kinematic isotropy), `p.loadCloth / p.clothParams` (dressing.py:146-147) and the
50-step settle at half gravity (dressing.py:178-193).  Scene recipe: SURVEY.md Appendix C.3.

Differences forced by lock-step batching / the 32-DoF budget of one env (DESIGN.md section 9):
  * both genders are instantiated, one is switched off per env;
  * of PR2's 44 non-fixed joints the left arm (7) and the left gripper (4) are simulated; every other joint is welded at
    the angle `reset_joints` gives it (the reference holds them with default velocity motors under zero gravity);
  * `impairment == 'limits'` scales the person's joint limits per env in the reference (human.py:85); joint limits are template
    data here, so it is drawn but has no effect; `weakness` (per-env motor force scale) and `tremor` are simulated;
  * a tremor person is clamped to its joint limits after every stepSimulation (env.py:226-229); the clamp flag is per joint,
    not per env, so it is on for the arm joints of every env (the limit rows keep non-tremor arms inside anyway).

With `controllable_person=True` (DressingPR2Human-v1) the person's left arm is a second agent.  The template is the same (the left
arm already keeps its mass); the impairment is drawn with 'no_tremor' (feeding.py:59 does the same for its co-optimisation id);
`limits` acts through the per-env scaled clamps of the co-optimisation kernels and clips the start pose; `weakness` is drawn but
does not act, because a controllable person gets no reactive force (dressing.py:124).  While the gown settles the arm is held
with gain 0.05 and force 1 (dressing.py:142-144), and no per-substep hard clamp is set on it: the reference clamps the person
once per stepSimulation (env.py:226-231), as `k_coop_limits` does.
"""
import numpy as np

from . import capi, toc
from .cloth import ClothModel
from .feeding_batch import coop_params, pack_mlp
from .human_model import create_human
from .kinematics import q_axis, q_from_rpy, q_mul, q_rot
from .toc import TocPlacement, jlwki, position_robot_toc  # noqa: F401
from .scene import SceneBuilder, quat_from_rpy

MOTOR_POSITION = 1

PR2 = dict(toc.PR2_LEFT, gripper_pos=[0.0] * 4, right_arm=toc.PR2_RIGHT['arm'], right_preset=toc.PR2_RIGHT['default_q'],
           left_preset=toc.PR2_LEFT['default_q'], toc_base_pos_offset=[1.7, 0.7, 0], ee_orient_rpy=[0, 0, np.pi],
           ee_orient_shoulder_rpy=[0, 0, np.pi * 3 / 2.0])
LEFT_ARM_JOINTS = list(range(10, 20))                       # human.left_arm_joints (dressing_envs.py)
L_SHOULDER, L_ELBOW, L_WRIST = 15, 17, 19                   # human.py:26-28
L_ARM_LIMIT_JOINTS = [13, 14, 15, 16]                       # left shoulder x, y, z and elbow: the classifier's inputs (human.py:137-140)
# degrees (dressing.py:120): right elbow, left shoulder x, left elbow, hips, knees
HUMAN_PRESET = {6: -90, 13: -45, 16: -90, 28: -90, 31: 80, 35: -90, 38: 80}
RADII = {'male': (0.043, 0.043, 0.043), 'female': (0.0355, 0.0355, 0.0355)}     # hand, elbow, shoulder (human_creation.py:89,140)
CLOTH_ANCHORS = [2086, 2087, 2088, 2041]                    # dressing.py:146
TRIANGLE1, TRIANGLE2 = [1180, 2819, 30], [1322, 13, 696]    # dressing.py:149-150
CLOTH_ORIG_POS = np.array([0.34658437, -0.30296362, 1.20023387])      # dressing.py:140
CLOTH_POSITION = np.array([0.02, -0.38, 0.84])              # dressing.py:146 (scaled with the mesh)
CLOTH_SCALE = 1.4


def sleeve_on_arm_reward(triangle1_points, triangle2_points, shoulder_pos, elbow_pos, wrist_pos, hand_radius, elbow_radius, shoulder_radius):
    """Util.sleeve_on_arm_reward (util.py:125-202) for one env, in fp64: (forearm_in_sleeve, upperarm_in_sleeve,
    distance_along_forearm, distance_along_upperarm, distance_to_hand, distance_to_elbow, distance_to_shoulder, forearm_length,
    upperarm_length).  The per-call co-optimisation step computes its reward with it; `dressing_post_body` is the fused twin."""
    def signed_volume(a, b, c, d):
        return (1.0 / 6.0) * np.dot(np.cross(b - a, c - a), d - a)

    def line_hits_triangle(p0, p1, p2, q0, q1):
        if np.sign(signed_volume(q0, p0, p1, p2)) != np.sign(signed_volume(q1, p0, p1, p2)):
            return np.sign(signed_volume(q0, q1, p0, p1)) == np.sign(signed_volume(q0, q1, p1, p2)) == np.sign(signed_volume(q0, q1, p2, p0))
        return False

    def points_around(pts, normal, origin):
        t = np.cross(np.array([1.0, 1.0, 0.0]), normal); t = t / np.linalg.norm(t)
        b = np.cross(t, normal); b = b / np.linalg.norm(b)
        dt, db = (pts - origin) @ t, (pts - origin) @ b
        return bool(np.any(dt > 0) and np.any(dt < 0) and np.any(db > 0) and np.any(db < 0))
    t1, t2 = np.asarray(triangle1_points, dtype=np.float64), np.asarray(triangle2_points, dtype=np.float64)
    sh, el, wr = (np.asarray(v, dtype=np.float64) for v in (shoulder_pos, elbow_pos, wrist_pos))
    hand_end = wr + (wr - el) / np.linalg.norm(wr - el) * hand_radius * 2
    elbow_end = el + (el - wr) / np.linalg.norm(wr - el) * elbow_radius
    shoulder_end = sh + (sh - el) / np.linalg.norm(sh - el) * shoulder_radius
    pts = np.concatenate([t1, t2], axis=0)
    nf = (hand_end - elbow_end) / np.linalg.norm(hand_end - elbow_end)
    nu = (elbow_end - shoulder_end) / np.linalg.norm(elbow_end - shoulder_end)
    forearm_in = points_around(pts, nf, hand_end) and (line_hits_triangle(*t1, hand_end, elbow_end) or line_hits_triangle(*t2, hand_end, elbow_end))
    upperarm_in = points_around(pts, nu, shoulder_end) and (line_hits_triangle(*t1, elbow_end, shoulder_end) or line_hits_triangle(*t2, elbow_end, shoulder_end))
    centre = pts.mean(axis=0)
    return (forearm_in, upperarm_in, np.linalg.norm(centre - hand_end), np.linalg.norm(centre - el), np.linalg.norm(hand_end - centre),
            np.linalg.norm(elbow_end - centre), np.linalg.norm(shoulder_end - centre), np.linalg.norm(hand_end - elbow_end), np.linalg.norm(el - sh))


class DressingBatch(TocPlacement):
    """DressingPR2-v1 / DressingPR2Human-v1.  The robot is the scene's only per-robot part: `R` and `load_robot` / `robot_links`
    (TocPlacement) build it, `CLOTH_ROBOT_JOINTS` picks the links the gown collides with, and `_reset_robot` puts it in place;
    dressing_robots_batch.py replaces these for Sawyer and Jaco and shares the rest."""
    R = PR2
    WHEELCHAIR = 'wheelchair'
    # PR2: its left arm and gripper (everything else of PR2 stays a metre away from the gown)
    CLOTH_ROBOT_JOINTS = range(PR2['arm'][0], 86)

    def __init__(self, controllable_person=False):
        self.controllable_person = bool(controllable_person)
        b = SceneBuilder()
        self.builder = b
        b.set_gravity([0, 0, -9.81])
        self.plane = b.load_urdf('plane')
        self.wheelchair = b.load_urdf(self.WHEELCHAIR, base_pos=[0, 0, 0.06], fixed_base=False)
        self.humans = {}
        for gender, z in (('male', 0.89), ('female', 0.86)):
            hb, info = create_human(b, gender=gender, static=True, cloth=True)       # env.py:38 cloth=('dressing' in task)
            b.bodies[hb].base_pos = np.array([0, 0.03, z])
            for j in range(b.num_joints(hb)):                                         # "static joints" (human.py:108-112)
                if j not in LEFT_ARM_JOINTS:
                    b.change_dynamics(hb, j, mass=0)
            b.set_gravity([0, 0, -1], body=hb)                                        # dressing.py:181
            self.humans[gender] = hb
        self.load_robot(b)                                                            # PR2: pr2.py:52
        b.set_gravity([0, 0, 0], body=self.robot)                                     # dressing.py:179-180
        self.scene = b.finalize()
        sc = self.scene
        self.robot_links(sc)
        self.tool = None
        self.obstacles = (self.humans['male'], self.humans['female'], self.wheelchair)       # collision_objects of dressing.py:134
        self.human_arm_links = {g: [self.gl(hb, j) for j in LEFT_ARM_JOINTS] for g, hb in self.humans.items()}
        # ---- cloth template and the rigid links it collides with: the person, the robot's `CLOTH_ROBOT_JOINTS`, the wheelchair
        # and the ground
        self.cloth = ClothModel.load('hospitalgown_reduced', scale=CLOTH_SCALE)
        has_col = lambda k: np.any(sc['col_link'] == k)
        links, static = [], []
        for body, is_static, rng_ in ([(self.plane, 1, None), (self.wheelchair, 1, None)] + [(hb, 0, None) for hb in self.humans.values()]
                                      + [(self.robot, 0, self.CLOTH_ROBOT_JOINTS)]):
            l0, nl = int(sc['body_link0'][body]), int(sc['body_nlinks'][body])
            for k in range(l0, l0 + nl):
                if rng_ is not None and (k - l0 - 1) not in rng_:
                    continue
                if has_col(k):
                    links.append(k)
                    static.append(is_static)
        self.cloth_links, self.cloth_static = links, static
        self.cloth_quat = quat_from_rpy([0, 0, np.pi])
        x_zero = self.cloth.place(CLOTH_POSITION * CLOTH_SCALE, self.cloth_quat)      # cloth_offset = 0 <=> end effector at cloth_orig_pos
        self.anchor_local = x_zero[CLOTH_ANCHORS] - CLOTH_ORIG_POS
        self.x_zero = x_zero

    @staticmethod
    def config(**kw):
        """AgConfig of the task: numSubSteps = 8 (dressing.py:184); a larger contact budget than the default, because the seated person's
        arm and the robot's arm sweep past the wheelchair's 44 hulls (the candidate-pair budget is 4 x max_contacts)."""
        return capi.default_config(**dict(dict(num_substeps=8, max_contacts=256), **kw))

    # ------------------------------------------------------------------ params of the fused step
    def dressing_params(self):
        P = capi.AgDressingParams()
        P.robot_body = self.robot
        P.human_body_m, P.human_body_f = self.humans['male'], self.humans['female']
        for i, l in enumerate(self.arm_links):
            P.arm_links[i] = l; P.arm_lower[i] = self.arm_lower[i]; P.arm_upper[i] = self.arm_upper[i]
        P.ee_link = self.ee_link
        for i, l in enumerate((L_SHOULDER, L_ELBOW, L_WRIST)):
            P.arm_points_m[i] = self.gl(self.humans['male'], l); P.arm_points_f[i] = self.gl(self.humans['female'], l)
        for i in range(10):
            P.human_arm_m[i] = self.human_arm_links['male'][i]; P.human_arm_f[i] = self.human_arm_links['female'][i]
        P.hand_radius_m, P.elbow_radius_m, P.shoulder_radius_m = RADII['male']
        P.hand_radius_f, P.elbow_radius_f, P.shoulder_radius_f = RADII['female']
        for i in range(3):
            P.tri1[i] = int(self.cloth.rank[TRIANGLE1[i]]); P.tri2[i] = int(self.cloth.rank[TRIANGLE2[i]])
        P.action_multiplier, P.frame_skip = 0.05, 5
        P.w_dressing, P.w_action = 1.0, 0.01                     # config.ini [dressing]
        P.c_v, P.c_d = 0.25, 0.01                                # config.ini [human_preferences]
        P.task_success_threshold = 0.4
        return P

    # ------------------------------------------------------------------ batched reset
    def sample(self, n, rng, impairment=None):
        """impairment: 'random' (human.py:80-81), 'no_tremor', or one of none / limits / weakness / tremor; by default 'random', and
        'no_tremor' for a controllable person.  A controllable person's `limit_scale` is drawn after every other field."""
        if impairment is None:
            impairment = 'no_tremor' if self.controllable_person else 'random'
        names = ('none', 'limits', 'weakness', 'tremor')
        imp = rng.integers(0, 4, size=n) if impairment == 'random' else (rng.integers(0, 3, size=n) if impairment == 'no_tremor' else np.full(n, names.index(impairment)))
        s = dict(plane_friction=rng.uniform(0.025, 0.5, size=n),                  # env.py:120
                    male=rng.integers(0, 2, size=n).astype(np.int32),                # human.py:76-77
                    impairment=imp.astype(np.int32),
                    strength=np.where(imp == 2, rng.uniform(0.25, 1.0, size=n), 1.0),                                       # human.py:86
                    tremors=np.where((imp == 3)[:, None], rng.uniform(np.deg2rad(-10), np.deg2rad(10), size=(n, 10)), 0.0),   # human.py:92
                    ee_offset=rng.uniform(-0.05, 0.05, size=(n, 3)))                 # dressing.py:129
        if self.controllable_person:
            s['limit_scale'] = np.where(imp == 1, rng.uniform(0.5, 1.0, size=n), 1.0)                                        # human.py:85
        return s

    def human_pose(self):
        out = {}
        for g, hb in self.humans.items():
            nj = int(self.scene['body_nlinks'][hb]) - 1
            links = [self.gl(hb, j) for j in range(nj)]
            q = np.zeros(nj)
            for j, deg in HUMAN_PRESET.items():
                q[j] = np.deg2rad(deg)
            q = np.clip(q, self.scene['link_lower'][links], self.scene['link_upper'][links])     # enforce_joint_limits (human.py:121)
            out[g] = (links, q)
        return out

    def position_robot_toc(self, sim, rng, start, targets, attempts=50, mask=None):
        """Robot.position_robot_toc for the left arm (dressing.py:134: right_side=False, base yaw pi, 50 attempts)."""
        base0 = np.array([-0.85, -0.4, 0]) + np.array(PR2['toc_base_pos_offset'])
        return position_robot_toc(sim, rng, self.robot, self.arm_links, self.ee_link, self.kin, np.array(PR2['arm']) + 1, PR2['ee'] + 1,
                                  self.arm_lower, self.arm_upper, base0, [start] + list(targets), right_side=False, base_yaw=np.pi,
                                  attempts=attempts, mask=mask, default_q=PR2['left_preset'])

    def reset(self, sim, rng, sample=None, attempts=50, settle_steps=50, outer_iterations=3):
        n = sim.n
        s = sample or self.sample(n, rng)
        self.last_sample = s
        limb = self._reset_person(sim, s)
        base_pos, base_quat, q7, gq = self._reset_robot(sim, s, rng, limb, attempts, outer_iterations)
        ng = len(self.gripper_links)
        sim.set_motor(self.arm_links, MOTOR_POSITION, target=q7, kp=[0.01] * 7, kd=[1.0] * 7, max_force=[1.0] * 7)       # dressing.py:117
        sim.set_motor(self.gripper_links, MOTOR_POSITION, target=gq, kp=[0.05] * ng, kd=[1.0] * ng, max_force=[500.0] * ng)
        sim.forward_kinematics()
        self.base_pos, self.base_quat = base_pos, base_quat
        self._reset_cloth(sim, settle_steps)
        return s

    def _reset_person(self, sim, s):
        """Floor friction; the person seated in the wheelchair, the left arm held by weak position motors (dressing.py:117-121);
        returns the active person's left shoulder, elbow and wrist [n, 3, 3]."""
        n = sim.n
        sc = self.scene
        male = s['male'].astype(bool)
        sim.set_link_friction(int(sc['body_link0'][self.plane]), s['plane_friction'])
        for g, hb in self.humans.items():
            links, q = self.human_pose()[g]
            qn = np.tile(q, (n, 1))
            if self.controllable_person:     # enforce_joint_limits at the `limits` impairment's scaled limits (human.py:121)
                lo, hi = self.person_limits(links)
                sc_ = np.asarray(s.get('limit_scale', np.ones(n)), dtype=np.float64)[:, None]
                qn = np.clip(qn, lo[None] * sc_, hi[None] * sc_)
            sim.set_joint_state(links, q=qn, qd=np.zeros_like(qn))
            sim.set_body_active(hb, np.where(male if g == 'male' else ~male, 1, 0).astype(np.int32))
            al = self.human_arm_links[g]
            tgt = qn[:, LEFT_ARM_JOINTS]
            if self.controllable_person:     # held while the gown settles (dressing.py:142-144); no reactive force, no strength
                sim.set_motor(al, MOTOR_POSITION, target=tgt, kp=[0.05] * 10, kd=[1.0] * 10, max_force=[1.0] * 10)
                sim.set_motor_force_scale(al, np.ones((n, 10)))
            else:
                sim.set_motor(al, MOTOR_POSITION, target=tgt, kp=[0.01] * 10, kd=[1.0] * 10, max_force=[1.0] * 10)
                sim.set_motor_force_scale(al, np.repeat(s.get('strength', np.ones(n))[:, None], 10, axis=1))                # forces = 1 * strength (human.py:126)
                sim.set_hard_limits(al, True)
        self.human_rest = np.tile(self.human_pose()['male'][1][LEFT_ARM_JOINTS], (n, 1))      # target_joint_angles (human.py:122); the presets are the same for both genders
        sim.forward_kinematics()
        limb = np.zeros((n, 3, 3))
        for g, hb in self.humans.items():
            ls = sim.get_link_states([self.gl(hb, L_SHOULDER), self.gl(hb, L_ELBOW), self.gl(hb, L_WRIST)])['pos']
            limb[male if g == 'male' else ~male] = ls[male if g == 'male' else ~male]
        return limb

    def _reset_robot(self, sim, s, rng, limb, attempts, outer_iterations):
        """PR2's base pose and start joint angles (dressing.py:129-134); returns base position, base orientation, arm angles and the
        gripper's motor targets."""
        n = sim.n
        replay = 'base_pos' in s
        tq = np.tile(q_from_rpy(PR2['ee_orient_rpy']), (n, 1)); tqs = np.tile(q_from_rpy(PR2['ee_orient_shoulder_rpy']), (n, 1))
        target = np.array([0.45, -0.3, 1.0]) + s['ee_offset']
        off = np.array([0, 0, 0.1])
        gq = np.tile(PR2['gripper_pos'], (n, 1)).astype(np.float64)
        sim.set_joint_state(self.gripper_links, q=gq, qd=np.zeros_like(gq))
        if replay:
            base_pos, base_quat, q7 = s['base_pos'].copy(), s['base_quat'].copy(), s['q7'].copy()
            self.goals_reached = s.get('goals_reached')
        else:
            todo = np.ones(n, dtype=bool)
            base_pos = np.zeros((n, 3)); base_quat = np.tile([0, 0, 0, 1.0], (n, 1)); q7 = np.zeros((n, 7)); reached = np.zeros(n, dtype=int)
            for _ in range(outer_iterations):                                        # env.py:282-309
                bp, bq, bj, num, _man = self.position_robot_toc(sim, rng, (target, tq), [(limb[:, 0] + off, tqs), (limb[:, 1] + off, tq), (limb[:, 2] + off, tq)],
                                                                attempts=attempts, mask=todo)
                base_pos[todo], base_quat[todo], q7[todo], reached[todo] = bp[todo], bq[todo], bj[todo], num[todo]
                sim.set_base_pose(self.robot, base_pos, base_quat)
                sim.set_joint_state(self.arm_links, q=q7, qd=np.zeros_like(q7))
                sim.forward_kinematics()
                todo = self.colliding(sim)
                if not todo.any():
                    break
            self.unresolved = int(todo.sum())
            self.goals_reached = reached
            s.update(base_pos=base_pos.copy(), base_quat=base_quat.copy(), q7=q7.copy(), goals_reached=reached.copy())
        sim.set_base_pose(self.robot, base_pos, base_quat)
        sim.set_joint_state(self.arm_links, q=q7, qd=np.zeros_like(q7))
        return base_pos, base_quat, q7, gq

    def _reset_cloth(self, sim, settle_steps):
        """The gown placed relative to the end effector, four nodes anchored to it, settled at half gravity (dressing.py:139-193)."""
        start_ee = sim.get_link_states([self.ee_link])['pos'][:, 0].astype(np.float64)
        self.start_ee_pos = start_ee
        x0 = self.x_zero[None] + (start_ee - CLOTH_ORIG_POS)[:, None, :]
        if not getattr(sim, 'cloth_model', None):
            sim.cloth_init(self.cloth, self.cloth_links, self.cloth_static, CLOTH_ANCHORS, self.anchor_local, gravity=(0, 0, -9.81), max_contacts=1024)
        sim.cloth_set_state(x0, np.zeros_like(x0))
        sim.cloth_set_anchor(start_ee)
        sim.cloth_set_gravity([0, 0, -9.81 / 2])
        if settle_steps:
            sim.step(settle_steps)
        sim.cloth_set_gravity([0, 0, -9.81])
        # the gown is created flat and partly INSIDE the seated person (dressing.py:146 places it relative to the gripper only): in the
        # first substeps of the settle a few per cent of the envs hold more cloth contacts than the 1 024-contact budget; reported
        # separately from the steady-state flag, which the caller reads after its own steps
        self.settle_overflow = int(sim.overflow_count()) if hasattr(sim, 'overflow_count') else 0

    def person_limits(self, links):
        """Template limits of the person's joints as the per-call Agent sees them (an unlimited joint is +-1e10, agent.py)."""
        lo, hi = self.scene['link_lower'][links].astype(np.float64), self.scene['link_upper'][links].astype(np.float64)
        free = (lo == 0) & (hi == -1)
        return np.where(free, -1e10, lo), np.where(free, 1e10, hi)

    def start_coop(self, sim, sample=None):
        """Arm the person's half of the fused co-optimisation step (DressingPR2Human-v1); call after `start_fused`.  The arm is
        driven with the gains take_step's control() issues every step (Human.motor_gains = 0.01 after dressing.py:121, motor_forces
        1.0); limits are scaled by the sample's `limit_scale`; the classifier of limits_model keeps the left arm inside the
        realistic joint limits (sign +1: the left arm's input mapping, human.py:141-145)."""
        from .limits_model import load_model
        s = sample or self.last_sample
        P = coop_params(self.scene, self.humans, 3, LEFT_ARM_JOINTS, 0.01)
        w = pack_mlp(P, load_model(), L_ARM_LIMIT_JOINTS, 1.0)
        sim.coop_init(P, limit_scale=s.get('limit_scale'), mlp=w)
        imp = s.get('impairment')
        if imp is not None and np.any(imp == 3):       # a tremor person (human_impairment given to the env)
            sim.coop_set_tremor(imp == 3, self.coop_tremor_target(s), s['tremors'])

    def coop_tremor_target(self, s):
        """target_joint_angles [n, 10] of a controllable tremor person (human.py:123): the left arm's preset, before the gown
        settles"""
        return self.human_rest

    def start_fused(self, sim, sample=None):
        s = sample or self.last_sample
        sim.dressing_init(self.dressing_params(), s['male'])
        imp = s.get('impairment')
        if imp is not None and np.any(imp == 3) and not self.controllable_person:     # a controllable person's: start_coop
            sim.dressing_set_tremor((imp == 3).astype(np.int32), self.human_rest, s['tremors'])
