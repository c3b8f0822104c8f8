"""BedBathingSawyer-v1 as a batched scene: template construction, batched reset, wiping targets.

Restates `BedBathingEnv.reset` / `generate_targets` / `update_targets` (reference envs/bed_bathing.py:113-203)
and what they call: `Furniture.init('bed')` (agents/furniture.py:18-19), `Sawyer.init` (agents/sawyer.py:51-61),
`Tool.init` for the wiper (agents/tool.py:10-47), `util.capsule_points` (envs/util.py:80-113),
`AssistiveEnv.init_robot_pose` / `Robot.position_robot_toc` (envs/env.py:276-310, agents/robot.py:123-215).

Differences forced by lock-step batching or by what the backend does not simulate yet (DESIGN.md):
  * both human genders are instantiated; per env the inactive one is switched off;
  * the person is NOT dropped onto the bed as a 47-DoF ragdoll (bed_bathing.py:121-131 lets a floating-base
    articulated body settle for 100 steps; floating-base articulations are not built): the perturbed lying
    pose is lowered until it touches the mattress and then frozen, which is the state the reference reaches
    *in kind* (static person on the bed), not the same pose;
  * the robot base pose is drawn from the distribution `position_robot_toc` samples (robot.py:142-144) and the
    first draw whose start pose is reachable and collision-free is kept; the JLWKI manipulability ranking over
    50 draws (robot.py:150-186) is not restated (reset-time code, SURVEY.md §8(f)1);
  * the 91 / 129 target marker bodies (bed_bathing.py:187-188) are not instantiated: targets are points.

With `controllable_person=True` (BedBathingSawyerHuman-v1) the person's right arm is a second agent: its ten joints keep their
mass (`setup_joints(use_static_joints=True, reactive_force=None)` with a controllable person, human.py:104-127), the active
gender is simulated instead of frozen, and the impairment is drawn with 'no_tremor' (as FeedingJacoHuman-v1 does, feeding.py:59).
`tremor` is drawn for a controllable person only when the env is given `human_impairment` (`start_coop` arms it).  `weakness` is drawn but
does not act: the task sets no reactive force, and take_step's control() drives the arm with motor_forces 1.0.  The wiping targets
then follow the arm (update_targets, bed_bathing.py:190-203), from their link frames (`target_frames`).
"""
import numpy as np

from .feeding_batch import coop_params, pack_mlp
from .human_model import create_human
from .kinematics import BodyKinematics, ik_dls, q_from_rpy, q_mul, q_rot
from .toc import position_robot_toc
from .scene import SceneBuilder, quat_from_rpy

MOTOR_POSITION = 1
SAWYER = dict(arm=[3, 8, 9, 10, 11, 13, 16], ee=19, gripper=[20, 22], tool_joint=18, gripper_collision=[18, 20, 21, 22, 23],
              gripper_pos=[0.0125, -0.0125], tool_pos_offset=[0, 0.1175, 0], tool_orient_offset=[np.pi / 2.0, 0, np.pi / 2.0],
              toc_base_pos_offset=[-0.2, 0, 0.975], ee_orient_rpy=[0, np.pi / 2.0, 0])
R_SHOULDER, R_ELBOW, R_WRIST = 5, 7, 9          # human.right_shoulder / right_elbow / right_wrist (human.py link ids)
J_RIGHT_SHOULDER_X = 3
# (upperarm length, radius, forearm length, radius), bed_bathing.py:176-181
ARM_DIMS = {'male': (0.279, 0.043, 0.257, 0.033), 'female': (0.264, 0.0355, 0.234, 0.027)}
WIPER_CLOTH_LINK = 1                             # `if linkA in [1]`, bed_bathing.py:49
RIGHT_ARM_JOINTS = list(range(0, 10))            # human.right_arm_joints (bed_bathing_envs.py)
R_ARM_LIMIT_JOINTS = [3, 4, 5, 6]                # shoulder x, y, z and elbow: the classifier's inputs (human.py:137-140)


def orthogonal_vector(v):
    """util.py:115-121: v crossed with the unit vector of the axis after v's largest component (the start of the rings of
    `capsule_points`, so the rule has to be the reference's; pinned by tests/test_reference_util_vectors.py)."""
    v = np.asarray(v, dtype=np.float64)
    y = np.zeros(3)
    y[(int(np.argmax(np.abs(v))) + 1) % 3] = 1.0
    return np.cross(v, y)


def capsule_points(p1, p2, radius, distance_between_points=0.05):
    """util.py:80-113 restated: rings of points around a capsule's cylinder, `distance_between_points` apart."""
    p1, p2 = np.asarray(p1, dtype=np.float64), np.asarray(p2, dtype=np.float64)
    axis = (p2 - p1) / np.linalg.norm(p2 - p1)
    ortho = orthogonal_vector(axis)
    ortho = ortho / np.linalg.norm(ortho)
    normal = np.cross(axis, ortho)
    sections = int(np.linalg.norm(p2 - p1) / distance_between_points)
    pts = []
    for i in range(sections):
        sec = (p2 - p1) / (sections + 1) * (i + 1)
        theta_dist = distance_between_points / radius
        for j in range(int(2 * np.pi * radius / distance_between_points)):
            th = theta_dist * j
            pts.append(p1 + sec + radius * np.cos(th) * ortho + radius * np.sin(th) * normal)
    return np.array(pts).reshape(-1, 3)


class BedBathingBatch:
    def __init__(self, controllable_person=False):
        self.controllable_person = bool(controllable_person)
        b = self._bed_and_persons()
        self.robot = b.load_urdf('sawyer', base_pos=[-1, -1, 0.975], fixed_base=True, self_collision=True)
        for i in range(3, 24):                                                   # sawyer.py:55-61
            for j in range(3, 24):
                b.set_collision_filter_pair(self.robot, self.robot, i, j, False)
        for i in range(0, 3):
            for j in range(0, 9):
                b.set_collision_filter_pair(self.robot, self.robot, i, j, False)
        self.tool = b.load_urdf('wiper')
        for j in SAWYER['gripper_collision']:                                    # tool.py:41-44
            for tj in (-1, 0, 1):
                b.set_collision_filter_pair(self.robot, self.tool, j, tj, False)
        self.tool_pos_offset = np.array(SAWYER['tool_pos_offset'], dtype=np.float64)
        self.tool_quat_offset = quat_from_rpy(SAWYER['tool_orient_offset'])
        b.create_fixed_constraint(self.robot, SAWYER['tool_joint'], self.tool, -1, self.tool_pos_offset, [0, 0, 0],
                                  self.tool_quat_offset, [0, 0, 0, 1], max_force=500)
        b.set_gravity([0, 0, 0], body=self.robot)
        b.set_gravity([0, 0, 0], body=self.tool)
        self.scene = b.finalize()
        sc = self.scene
        self.gl = lambda body, link: int(sc['body_link0'][body]) + 1 + link
        self.arm_links = [self.gl(self.robot, j) for j in SAWYER['arm']]
        self.gripper_links = [self.gl(self.robot, j) for j in SAWYER['gripper']]
        self.ee_link = self.gl(self.robot, SAWYER['ee'])
        self.kin = BodyKinematics(sc, self.robot)
        self.arm_lower = sc['link_lower'][self.arm_links].copy()
        self.arm_upper = sc['link_upper'][self.arm_links].copy()
        self._person_links()

    def _bed_and_persons(self):
        """A scene builder holding the plane, the bed and both persons as BedBathing sets them up; the robot and the wiper follow."""
        b = SceneBuilder()
        self.builder = b
        b.set_gravity([0, 0, -9.81])
        self.plane = b.load_urdf('plane')
        self.bed = b.load_urdf('bed', base_pos=[-0.1, 0, 0], fixed_base=True)
        b.change_dynamics(self.bed, -1, lateral_friction=5)                      # bed_bathing.py:117
        self.humans = {}
        for gender in ('male', 'female'):
            hb, info = create_human(b, gender=gender, static=True)
            for j in range(b.num_joints(hb)):                                    # "static joints" after the settle (bed_bathing.py:133-136)
                if not (self.controllable_person and j in RIGHT_ARM_JOINTS):  # a controllable arm keeps its mass (human.py:108-112)
                    b.change_dynamics(hb, j, mass=0)
            b.set_gravity([0, 0, -1], body=hb)
            self.humans[gender] = hb
        return b

    def _person_links(self):
        """The wiper's cloth link, the persons' kinematics and arm links, and the wiping targets, once the scene is finalised."""
        sc = self.scene
        self.cloth_link = self.gl(self.tool, WIPER_CLOTH_LINK)
        self.hkin = {g: BodyKinematics(sc, hb) for g, hb in self.humans.items()}
        # wiping targets in the upper-arm / forearm link frames (bed_bathing.py:183-184)
        self.targets_local = {}
        for g, (ul, ur, fl, fr) in ARM_DIMS.items():
            self.targets_local[g] = (capsule_points([0, 0, 0], [0, 0, -ul], ur, 0.03), capsule_points([0, 0, 0], [0, 0, -fl], fr, 0.03))
        self.max_targets = max(len(u) + len(f) for u, f in self.targets_local.values())
        self.human_arm_links = {g: [self.gl(hb, j) for j in RIGHT_ARM_JOINTS] for g, hb in self.humans.items()}

    # ------------------------------------------------------------------ params for the fused kernels
    def bathing_params(self):
        from . import capi
        sc = self.scene
        P = capi.AgBathingParams()
        P.robot_body, P.tool_body = self.robot, self.tool
        P.human_body_m, P.human_body_f = self.humans['male'], self.humans['female']
        for i, l in enumerate(self.arm_links):
            P.arm_links[i] = l; P.arm_lower[i] = self.arm_lower[i]; P.arm_upper[i] = self.arm_upper[i]
        P.ee_link, P.cloth_link = self.ee_link, self.cloth_link
        for i, l in enumerate((R_SHOULDER, R_ELBOW, R_WRIST)):
            P.arm_points_m[i] = self.gl(self.humans['male'], l); P.arm_points_f[i] = self.gl(self.humans['female'], l)
        for g, tag in (('male', 'm'), ('female', 'f')):
            hb = self.humans[g]
            l0, nl = int(sc['body_link0'][hb]), int(sc['body_nlinks'][hb])
            cols = [c for c in range(sc.n_colliders) if l0 <= sc['col_link'][c] < l0 + nl]
            assert cols == list(range(cols[0], cols[0] + len(cols)))          # a body's colliders are contiguous
            setattr(P, 'human_col0_' + tag, cols[0]); setattr(P, 'human_ncol_' + tag, len(cols))
        P.n_targets_max = self.max_targets
        P.action_multiplier, P.frame_skip = 0.05, 5
        P.w_distance, P.w_action, P.w_wiping = 1.0, 0.01, 5.0                # config.ini [bed_bathing]
        P.c_v, P.c_f, P.c_hf = 0.25, 0.01, 0.05                              # config.ini [human_preferences]
        P.task_success_threshold = 0.3
        return P

    def start_fused(self, sim, sample=None):
        """Arm the fused per-step kernels for the envs last put in place by `reset`."""
        s = sample or self.last_sample
        tw, valid = self.targets_world(sim, s)
        sim.bathing_init(self.bathing_params(), s['male'], tw, valid)
        return tw, valid

    def start_coop(self, sim, sample=None):
        """Arm the person's half of the fused co-optimisation step (BedBathingSawyerHuman-v1); call after `start_fused`.  The
        targets follow the arm from their link frames; the arm is driven with Human.motor_gains / motor_forces (0.05, 1.0), the
        gains take_step's control() issues every step; limits are scaled by the sample's `limit_scale`; the classifier of
        limits_model keeps the right arm inside the realistic joint limits."""
        from .limits_model import load_model
        s = sample or self.last_sample
        link, local = self.target_frames(s)
        sim.bathing_set_target_frames(link, local)
        P = coop_params(self.scene, self.humans, 2, RIGHT_ARM_JOINTS, 0.05)
        w = pack_mlp(P, load_model(), R_ARM_LIMIT_JOINTS, -1.0)
        sim.coop_init(P, limit_scale=s.get('limit_scale'), mlp=w)
        imp = s.get('impairment')
        if imp is not None and np.any(imp == 3):       # a tremor person (human_impairment given to the env)
            sim.coop_set_tremor(imp == 3, self.coop_tremor_target(s), s['tremors'])

    def coop_tremor_target(self, s):
        """target_joint_angles [n, 10] of a controllable tremor person (human.py:123): the right arm of the lying pose"""
        male = s['male'].astype(bool)
        poses = self.human_pose(s)
        return np.where(male[:, None], poses['male'][1][:, RIGHT_ARM_JOINTS], poses['female'][1][:, RIGHT_ARM_JOINTS])

    # ------------------------------------------------------------------ batched reset
    def sample(self, n, rng):
        nj = 41
        s = dict(
            plane_friction=rng.uniform(0.025, 0.5, size=n),                       # env.py:120
            male=rng.integers(0, 2, size=n).astype(np.int32),
            joint_noise=rng.uniform(-0.1, 0.1, size=(n, nj)),                     # bed_bathing.py:126-127
            ee_offset=rng.uniform(-0.05, 0.05, size=(n, 3)),                      # bed_bathing.py:145
        )
        if self.controllable_person:         # drawn after every other field, so that the static person's draws stay as they are
            imp = rng.integers(0, 3, size=n)                                      # none / limits / weakness ('no_tremor', human.py:82-83)
            s['impairment'] = imp.astype(np.int32)
            s['limit_scale'] = np.where(imp == 1, rng.uniform(0.5, 1.0, size=n), 1.0)      # human.py:85
            s['strength'] = np.where(imp == 2, rng.uniform(0.25, 1.0, size=n), 1.0)        # human.py:86 (drawn, no effect here)
        return s

    def human_pose(self, s):
        """Joint angles of the lying person: right shoulder x 30 deg (bed_bathing.py:119), noise on every motor joint,
        limits enforced (human.py:121)."""
        n = len(s['male'])
        out = {}
        for g, hb in self.humans.items():
            nl = int(self.scene['body_nlinks'][hb])
            links = [self.gl(hb, j) for j in range(nl - 1)]
            q = np.zeros((n, nl - 1))
            q[:, J_RIGHT_SHOULDER_X] = np.deg2rad(30)
            movable = self.scene['link_jtype'][links] == 1
            noise = np.zeros((n, nl - 1)); noise[:, movable] = s['joint_noise'][:, :movable.sum()]
            # set_joint_angles(motor_indices, noise) REPLACES the angles (bed_bathing.py:127), the shoulder preset included
            q = np.where(movable[None, :], noise, q)
            q = np.clip(q, self.scene['link_lower'][links], self.scene['link_upper'][links])
            out[g] = (links, q)
        return out

    def solve_ik(self, base_pos, base_quat, target_pos, rng, max_restarts=8, threshold=0.03, sim=None, idx=None):
        """IK of the 7 arm joints to the start pose for every env from its own base pose (robot.py:84-121, threshold
        0.03 as position_robot_toc asks).  With a `sim` that offers `ik_solve` the solve runs on the device for the envs
        `idx` (their base poses must already be set in the sim; arrays are the rows of `idx`)."""
        n = len(target_pos)
        kin = self.kin
        if sim is not None and hasattr(sim, 'ik_solve'):
            mask = np.zeros(sim.n, dtype=np.int32); mask[idx] = 1
            tp = np.zeros((sim.n, 3)); tp[idx] = target_pos
            q7, err = sim.ik_solve(self.arm_links, self.ee_link, tp, q_from_rpy(SAWYER['ee_orient_rpy']), max_restarts=max_restarts, iters=100,
                                   threshold=threshold, seed=int(rng.integers(1, 2 ** 31 - 1)), mask=mask)
            q = np.zeros((n, kin.nl)); q[:, np.array(SAWYER['arm']) + 1] = q7[idx]
            return q, err[idx].astype(np.float64)
        tq = np.broadcast_to(q_from_rpy(SAWYER['ee_orient_rpy']), (n, 4)).copy()
        joints = np.array(SAWYER['arm']) + 1
        lo, hi = self.arm_lower, self.arm_upper
        best_q = np.zeros((n, kin.nl)); best_err = np.full(n, np.inf)
        todo = np.arange(n)
        for r in range(max_restarts):
            if len(todo) == 0:
                break
            q0 = np.zeros((len(todo), kin.nl))
            q0[:, joints] = rng.uniform(np.maximum(lo, -np.pi), np.minimum(hi, np.pi), size=(len(todo), 7))
            q, pe, oe = ik_dls(kin, base_pos[todo], base_quat[todo], q0, joints, SAWYER['ee'] + 1, target_pos[todo], tq[todo], lo, hi, iters=100)
            err = np.maximum(pe, oe)
            better = err < best_err[todo]
            best_q[todo[better]] = q[better]; best_err[todo[better]] = err[better]
            todo = todo[best_err[todo] >= threshold]
        return best_q, best_err

    def place_tool(self, sim, base_pos, base_quat, qfull):
        """Wiper at the tool joint's COM frame composed with the offsets (tool.py:49-54)."""
        n = sim.n
        pos, quat = self.kin.fk(base_pos, base_quat, qfull)
        cp, cq = self.kin.link_com_pose(pos, quat, SAWYER['tool_joint'] + 1)
        tp = cp + q_rot(cq, self.tool_pos_offset)
        tq = q_mul(cq, np.broadcast_to(self.tool_quat_offset, (n, 4)))
        sim.set_base_pose(self.tool, tp, tq)
        sim.set_base_velocity(self.tool, np.zeros((n, 3)), np.zeros((n, 3)))
        return tp, tq

    def reset(self, sim, rng, sample=None, base_attempts=6, toc_attempts=50):
        s = sample or self.sample(sim.n, rng)
        self.last_sample = s
        self._reset_person(sim, s)
        self._reset_sawyer(sim, s, rng, base_attempts, toc_attempts)
        return s

    def _reset_person(self, sim, s):
        """Floor friction and both genders in the lying pose with joint noise, lowered onto the mattress; frozen, or simulated when
        the person is controllable (one gender active per env).  Sets `human_pos` / `human_quat`."""
        n = sim.n
        sc = self.scene
        male = s['male'].astype(bool)
        sim.set_link_friction(int(sc['body_link0'][self.plane]), s['plane_friction'])
        # ---- person: lying pose, lowered onto the mattress, frozen
        lie = quat_from_rpy([-np.pi / 2.0, 0, 0])
        poses = self.human_pose(s)
        hpos = np.tile([-0.15, 0.2, 0.95], (n, 1)).astype(np.float64)              # bed_bathing.py:121
        for g, hb in self.humans.items():
            links, q = poses[g]
            sim.set_joint_state(links, q=q, qd=np.zeros_like(q))
            sim.set_base_pose(hb, hpos, np.tile(lie, (n, 1)))
            # frozen (2), or simulated (1) when the person is controllable; no motors on the arm at reset (reactive_force=None)
            sim.set_body_active(hb, np.where(male if g == 'male' else ~male, 1 if self.controllable_person else 2, 0).astype(np.int32))
        sim.forward_kinematics()
        drop = np.zeros(n)
        for g, hb in self.humans.items():
            on = male if g == 'male' else ~male
            c, k = sim.closest_points(hb, self.bed, 1.0, max_pts=64)
            d = np.where(np.arange(64)[None, :] < k[:, None], c['distance'], np.inf).min(axis=1)
            drop = np.where(on & np.isfinite(d), d, drop)
        hpos[:, 2] -= drop                                                          # the mattress top is flat: the gap is vertical
        for g, hb in self.humans.items():
            sim.set_base_pose(hb, hpos, np.tile(lie, (n, 1)))
        self.human_pos, self.human_quat = hpos, np.tile(lie, (n, 1))

    def _reset_sawyer(self, sim, s, rng, base_attempts, toc_attempts):
        n = sim.n
        male = s['male'].astype(bool)
        # ---- robot base pose + start joint angles (position_robot_toc's sampling distribution, first feasible draw)
        target = np.array([-0.6, 0.2, 1.0]) + s['ee_offset']
        gq = np.tile(SAWYER['gripper_pos'], (n, 1)).astype(np.float64)
        sim.set_joint_state(self.gripper_links, q=gq, qd=np.zeros_like(gq))
        base_pos = np.zeros((n, 3)); base_quat = np.tile([0, 0, 0, 1.0], (n, 1)); qik = np.zeros((n, self.kin.nl))
        ik_err = np.full(n, np.inf)
        todo = np.arange(n)
        obstacles = [self.humans['male'], self.humans['female'], self.bed]
        self.base_draws = 0
        replay = 'base_pos' in s            # a stored reset (same draws, e.g. oracle and product side of a parity test)
        use_toc = (not replay) and toc_attempts > 0 and hasattr(sim, 'ik_solve')
        arm_local = np.array(SAWYER['arm']) + 1

        def collides(base_pos, base_quat, qik):
            """robot + tool against person and bed at this pose (env.py:300-309)"""
            sim.set_base_pose(self.robot, base_pos, base_quat)
            arm_q = qik[:, arm_local]
            sim.set_joint_state(self.arm_links, q=arm_q, qd=np.zeros_like(arm_q))
            qfull = qik.copy(); qfull[:, np.array(SAWYER['gripper']) + 1] = SAWYER['gripper_pos']
            self.place_tool(sim, base_pos, base_quat, qfull)
            sim.forward_kinematics()
            hit = np.zeros(n, dtype=bool)
            for ob in obstacles:
                hit |= sim.closest_points(self.robot, ob, 0.0, max_pts=1)[1] > 0
                hit |= sim.closest_points(self.tool, ob, 0.0, max_pts=1)[1] > 0
            return hit

        if use_toc:
            # Robot.position_robot_toc (robot.py:123-221, called from env.py:299 with attempts=50): random base poses ranked by
            # goals reached (start pose + shoulder / elbow / wrist of the arm to be washed, position only) and JLWKI
            limb = np.zeros((n, 3, 3))
            for g, hb in self.humans.items():
                on = male if g == 'male' else ~male
                ls = sim.get_link_states([self.gl(hb, R_SHOULDER), self.gl(hb, R_ELBOW), self.gl(hb, R_WRIST)])['pos']
                limb[on] = ls[on]
            tq = np.tile(q_from_rpy(SAWYER['ee_orient_rpy']), (n, 1))
            base0 = np.array([-0.85, -0.4, 0]) + np.array(SAWYER['toc_base_pos_offset'])
            mask = np.ones(n, dtype=bool)
            reached = np.zeros(n, dtype=int)
            for _ in range(3):                                                   # env.py:282
                bp, bq, bj, num, _man = position_robot_toc(sim, rng, self.robot, self.arm_links, self.ee_link, self.kin, arm_local, SAWYER['ee'] + 1,
                                                           self.arm_lower, self.arm_upper, base0, [(target, tq)] + [(limb[:, j], None) for j in range(3)],
                                                           right_side=True, base_yaw=0.0, attempts=toc_attempts, mask=mask)
                self.base_draws += int(mask.sum()) * toc_attempts
                base_pos[mask], base_quat[mask], reached[mask] = bp[mask], bq[mask], num[mask]
                qik[np.ix_(mask, arm_local)] = bj[mask]
                ik_err[mask] = np.where(num[mask] >= 1, 0.0, np.inf)
                mask = collides(base_pos, base_quat, qik) | (ik_err >= 0.03)
                if not mask.any():
                    break
            todo = np.nonzero(mask)[0]
            self.goals_reached = reached
        for attempt in range(0 if use_toc else (1 if replay else base_attempts)):
            if len(todo) == 0:
                break
            m = len(todo)
            self.base_draws += m
            if replay:
                base_pos, base_quat, qik, ik_err = s['base_pos'].copy(), s['base_quat'].copy(), s['qik'].copy(), s['ik_err'].copy()
            else:                               # a sim without the device IK (the CPU oracle): first feasible draw of the same distribution
                rp = np.stack([rng.uniform(-0.5, 0, size=m), rng.uniform(-0.5, 0.5, size=m), np.zeros(m)], axis=1)   # right_side=True
                yaw = np.deg2rad(rng.uniform(-30, 30, size=m))
                bp = np.array([-0.85, -0.4, 0]) + np.array(SAWYER['toc_base_pos_offset']) + rp
                bq = np.stack([np.zeros(m), np.zeros(m), np.sin(yaw / 2), np.cos(yaw / 2)], axis=1)
                base_pos[todo], base_quat[todo] = bp, bq
                sim.set_base_pose(self.robot, base_pos, base_quat)
                q, err = self.solve_ik(bp, bq, target[todo], rng, sim=sim, idx=todo)
                qik[todo], ik_err[todo] = q, err
            bad = collides(base_pos, base_quat, qik) | (ik_err >= 0.03)
            todo = np.nonzero(bad)[0]
        collides(base_pos, base_quat, qik)      # leaves robot, arm and tool at the chosen pose
        self.ik_err, self.unresolved = ik_err, int(len(todo))
        self.base_pos, self.base_quat = base_pos, base_quat
        if not replay:
            s.update(base_pos=base_pos.copy(), base_quat=base_quat.copy(), qik=qik.copy(), ik_err=ik_err.copy())
        arm_q = qik[:, np.array(SAWYER['arm']) + 1]
        sim.set_motor(self.arm_links, MOTOR_POSITION, target=arm_q, kp=[0.05] * 7, kd=[1.0] * 7, max_force=[1.0] * 7)
        sim.set_motor(self.gripper_links, MOTOR_POSITION, target=gq, kp=[0.05] * 2, kd=[1.0] * 2, max_force=[500.0] * 2)
        sim.forward_kinematics()

    def hover_over_forearm(self, sim, s, rng, gap=0.003):
        """Start pose for the dense tool-skin contact workload (SURVEY.md 8(d) config C2): the arm is moved so that the
        wiping pad hovers `gap` above the middle of the person's right forearm (any joint action then presses it onto the
        skin or lifts it off).  Uses the sim's own closest-point query; returns the IK error per env."""
        n = sim.n
        male = s['male'].astype(bool)
        mid = np.zeros((n, 3))
        for g, hb in self.humans.items():
            ls = sim.get_link_states([self.gl(hb, R_ELBOW), self.gl(hb, R_WRIST)])['pos']
            on = male if g == 'male' else ~male
            mid[on] = 0.5 * (ls[on, 0] + ls[on, 1])
        arm = np.array(SAWYER['arm']) + 1

        def put(q):
            qfull = q.copy(); qfull[:, np.array(SAWYER['gripper']) + 1] = SAWYER['gripper_pos']
            sim.set_joint_state(self.arm_links, q=q[:, arm], qd=np.zeros((n, 7)))
            self.place_tool(sim, self.base_pos, self.base_quat, qfull)
            sim.forward_kinematics()

        q_hi, _ = self.solve_ik(self.base_pos, self.base_quat, mid + [0, 0, 0.25], rng, max_restarts=12, sim=sim, idx=np.arange(n))
        put(q_hi)
        d = np.full(n, np.inf)
        for hb in self.humans.values():
            c, k = sim.closest_points(self.tool, hb, 1.0, max_pts=32)
            d = np.minimum(d, np.where(np.arange(32)[None, :] < k[:, None], c['distance'], np.inf).min(axis=1))
        h0 = 0.25 - (np.where(np.isfinite(d), d, 0.25) - gap)
        q_lo, err = self.solve_ik(self.base_pos, self.base_quat, mid + np.stack([0 * h0, 0 * h0, h0], axis=1), rng, max_restarts=12, sim=sim, idx=np.arange(n))
        put(q_lo)
        sim.set_motor_targets(self.arm_links, q_lo[:, arm])
        return err

    # ------------------------------------------------------------------ wiping targets (generate_targets / update_targets)
    def targets_world(self, sim, s):
        """World positions [n, max_targets, 3] of the targets on the active person's right upper arm and forearm, a
        validity mask (the two genders have 129 / 91 targets) and the split index per env."""
        n = sim.n
        male = s['male'].astype(bool)
        out = np.full((n, self.max_targets, 3), 1e6)
        valid = np.zeros((n, self.max_targets), dtype=bool)
        for g, hb in self.humans.items():
            on = male if g == 'male' else ~male
            if not on.any():
                continue
            ls = sim.get_link_states([self.gl(hb, R_SHOULDER), self.gl(hb, R_ELBOW)])
            tu, tf = self.targets_local[g]
            wu = ls['pos'][:, 0, None, :] + q_rot(ls['quat'][:, 0, None, :], tu[None, :, :])
            wf = ls['pos'][:, 1, None, :] + q_rot(ls['quat'][:, 1, None, :], tf[None, :, :])
            w = np.concatenate([wu, wf], axis=1)
            out[on, :w.shape[1]] = w[on]
            valid[on, :w.shape[1]] = True
        return out, valid

    def target_frames(self, s):
        """Per env the global link each target rides on (upper arm R_SHOULDER, forearm R_ELBOW; -1 for padding) [n, T] and the
        target in that link's frame [n, T, 3], in the order of `targets_world`."""
        male = np.asarray(s['male']).astype(bool)
        n = len(male)
        link = np.full((n, self.max_targets), -1, dtype=np.int32)
        local = np.zeros((n, self.max_targets, 3))
        for g, hb in self.humans.items():
            on = male if g == 'male' else ~male
            tu, tf = self.targets_local[g]
            nu, nt = len(tu), len(tu) + len(tf)
            link[on, :nu], link[on, nu:nt] = self.gl(hb, R_SHOULDER), self.gl(hb, R_ELBOW)
            local[on, :nt] = np.concatenate([tu, tf], axis=0)
        return link, local

    def total_force(self, sim, targets_pos_world, targets_alive, max_tool_contacts=32):
        """`BedBathingEnv.get_total_force` (bed_bathing.py:41-78) on any sim with the BatchSim getter surface: robot and
        tool forces on the person, force of the wiper cloth (tool link 1) on the person, and the wiping targets within
        0.025 m of a cloth contact point on the person (posB) -- each target counts once (`targets_alive` is updated)."""
        n = sim.n
        total = np.zeros(n); tool_on_human = np.zeros(n); new_pts = np.zeros(n, dtype=int)
        tool_force = np.asarray(sim.contact_force_sum(self.tool), dtype=np.float64)
        K = max_tool_contacts
        for hb in self.humans.values():
            total += sim.contact_force_sum(self.robot, hb)
            c, k = sim.get_contacts(self.tool, hb, max_pts=K)
            live = np.arange(K)[None, :] < k[:, None]
            f = np.where(live, c['normal_force'], 0.0)
            total += f.sum(axis=1)
            cloth = live & (c['link_a'] == self.cloth_link)
            tool_on_human += np.where(cloth, f, 0.0).sum(axis=1)
            d = np.linalg.norm(c['pos_b'][:, :, None, :].astype(np.float64) - targets_pos_world[:, None, :, :], axis=-1)   # [n, K, T]
            hit = (cloth[:, :, None] & (d < 0.025)).any(axis=1) & targets_alive
            new_pts += hit.sum(axis=1)
            targets_alive &= ~hit
        return tool_force, tool_on_human, total, new_pts
