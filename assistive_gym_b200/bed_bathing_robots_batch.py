"""BedBathingPR2-v1 and BedBathingPR2Human-v1 as a batched scene: template construction and batched reset.

The scene is BedBathingSawyer's -- the plane, the bed with lateral friction 5, both persons lying on it with gravity -1 (the
co-optimisation person's right arm keeps its mass), the wiper on a fixed constraint -- with PR2 in place of Sawyer.  The task's
constants are the reference's `'bed_bathing'` entries of agents/pr2.py:19-46; the wiper is held in the left gripper
(`tool.init(..., right=False)`, bed_bathing.py:143).  The reset follows `BedBathingEnv.reset` (bed_bathing.py:113-168): the person,
then `init_robot_pose`'s TOC branch (env.py:276-310 -> robot.py:123-221) with the robot's left arm: one start goal ([-0.6, 0.2, 1]
randomised by +-0.05, with the task's orientation) and three target goals (the person's right shoulder, elbow and wrist by
position), 50 base poses on the person's right at yaw 0, and up to three collision-check rounds of robot and wiper against the
person and the bed that re-search only the colliding envs; then the gripper is opened.

As in scratch_itch_robots_batch.py, PR2 simulates its left arm (7) and left gripper (4) and welds every other joint at the angle
`reset_joints` gives it (the right arm at [-1.75, 1.25, -1.5, -0.5, -1, 0, -1], all others 0): 11 DoF, 31 with the co-optimisation
person's right arm in both genders (2 x 10), against the 32 an env may have.  PR2 is not `mobile`, so gravity on it is off, as on
the wiper.  BedBathingJaco is not built: the reference loads a nightstand under a wheelchair-mounted robot (bed_bathing.py:150-154)."""
import numpy as np

from . import toc
from .bed_bathing_batch import R_ELBOW, R_SHOULDER, R_WRIST, BedBathingBatch
from .kinematics import q_from_rpy
from .scene import quat_from_rpy
from .toc import TocPlacement

MOTOR_POSITION = 1

PR2 = dict(toc.PR2_LEFT, gripper_pos=[0.2] * 4, tool_pos_offset=[0, 0, 0], tool_orient_offset=[0, 0, 0],
           toc_base_pos_offset=[-0.1, 0, 0], ee_orient_rpy=[0, 0, 0])
TARGET_EE_POS = np.array([-0.6, 0.2, 1.0])            # bed_bathing.py:146


class BedBathingPR2Batch(TocPlacement, BedBathingBatch):
    """BedBathing with PR2 placed by TOC.  Shares `sample`, the person's reset, `bathing_params`, `start_fused`, `start_coop` and
    the target helpers with `BedBathingBatch`; BedBathingSawyer's own template and reset are not touched."""
    R = PR2

    def __init__(self, controllable_person=False):
        R = self.R
        self.controllable_person = bool(controllable_person)
        b = self._bed_and_persons()
        self.load_robot(b)
        self.tool = b.load_urdf('wiper')
        for j in R['gripper_collision']:                                             # tool.py:41-44 with the left gripper's links
            for tj in (-1, 0, 1):
                b.set_collision_filter_pair(self.robot, self.tool, j, tj, False)
        self.tool_pos_offset = np.array(R['tool_pos_offset'], dtype=np.float64)
        self.tool_quat_offset = quat_from_rpy(R['tool_orient_offset'])
        b.create_fixed_constraint(self.robot, R['tool_joint'], self.tool, -1, self.tool_pos_offset, [0, 0, 0], self.tool_quat_offset, [0, 0, 0, 1], max_force=500)
        b.set_gravity([0, 0, 0], body=self.robot)
        b.set_gravity([0, 0, 0], body=self.tool)
        self.scene = b.finalize()
        self.robot_links(self.scene)
        self._person_links()
        self.obstacles = (self.humans['male'], self.humans['female'], self.bed)      # collision_objects of bed_bathing.py:148

    def _sawyer_only(self, *a, **k):
        raise NotImplementedError("BedBathingBatch's own IK, tool placement and reset use Sawyer's joint table; PR2 is placed by "
                                  'TocPlacement (toc_search, place_robot)')
    solve_ik = place_tool = hover_over_forearm = _reset_sawyer = _sawyer_only

    def reset(self, sim, rng, sample=None, attempts=50, max_iterations=3):
        """Put every env of `sim` into a fresh start state.  A sample that holds `base_pos`, `base_quat` and `q7` (as `reset` leaves
        it) replays that robot placement instead of searching."""
        n, R = sim.n, self.R
        s = dict(sample) if sample else self.sample(n, rng)
        self.last_sample = s
        self._reset_person(sim, s)
        sim.forward_kinematics()
        if 'base_pos' in s:
            base_pos, base_quat, q7 = s['base_pos'].copy(), s['base_quat'].copy(), s['q7'].copy()
            self.goals_reached = s.get('goals_reached')
            self.place_robot(sim, base_pos, base_quat, q7)
            self.unresolved = int(self.colliding(sim).sum())
        else:
            arm = self.arm_points(sim, s['male'].astype(bool))
            tq = np.tile(q_from_rpy(R['ee_orient_rpy']), (n, 1))
            goals = [(TARGET_EE_POS + s['ee_offset'], tq)] + [(p, None) for p in arm]
            base_pos, base_quat, q7, _ = self.toc_search(sim, rng, goals, 1, attempts, max_iterations)
            s.update(base_pos=base_pos.copy(), base_quat=base_quat.copy(), q7=q7.copy(), goals_reached=self.goals_reached.copy())
        self.base_pos, self.base_quat = base_pos, base_quat
        gq = np.tile(R['gripper_pos'], (n, 1)).astype(np.float64)                  # set_gripper_open_position (bed_bathing.py:157)
        ng = len(R['gripper'])
        sim.set_motor(self.arm_links, MOTOR_POSITION, target=q7, kp=[0.05] * 7, kd=[1.0] * 7, max_force=[1.0] * 7)          # robot.py:36-37
        sim.set_motor(self.gripper_links, MOTOR_POSITION, target=gq, kp=[0.05] * ng, kd=[1.0] * ng, max_force=[500.0] * ng)
        sim.forward_kinematics()
        return s

    def arm_points(self, sim, male):
        """The active person's right shoulder, elbow and wrist positions (bed_bathing.py:138-140): three [N, 3] arrays."""
        out = [np.zeros((sim.n, 3)) for _ in range(3)]
        for g, hb in self.humans.items():
            on = male if g == 'male' else ~male
            pos = sim.get_link_states([self.gl(hb, j) for j in (R_SHOULDER, R_ELBOW, R_WRIST)])['pos'].astype(np.float64)
            for k in range(3):
                out[k][on] = pos[on, k]
        return out
