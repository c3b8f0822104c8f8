"""ScratchItchSawyer-v1 and ScratchItchPR2-v1 (and their co-optimisation ids) as batched scenes: template construction and batched reset.

The scene is ScratchItchJaco's -- person pair with a live right arm, the scratcher on a fixed constraint -- with another robot beside
the plain wheelchair (furniture.py:16).  The reset follows `ScratchItchEnv.reset` (scratch_itch.py:93-132): the person with
ScratchItch's preset pose, then `init_robot_pose`'s TOC branch (env.py:276-310 -> robot.py:123-221) with the robot's left arm: one
start goal (the randomised end-effector pose with the task's orientation) and three target goals (the person's right shoulder, elbow
and wrist by position), 50 base poses, and up to three collision-check rounds of robot and scratcher against the person and the
wheelchair that re-search only the colliding envs; then the gripper is opened and the target put on the upper arm or forearm.  The
task constants are the reference's `'scratch_itch'` entries of agents/sawyer.py:19-46 and agents/pr2.py:19-46; the tool is held in
the left gripper (`tool.init(..., right=False)`, scratch_itch.py:112).

Differences forced by the per-env DoF budget (32 per env, 16 per articulation; DESIGN.md section 9), as in feeding_robots_batch.py:
  * Sawyer: the 7 arm joints and the 2 gripper joints are simulated; every other joint (the head pan) is welded at 0.
  * PR2: the left arm (7) and the left gripper (4) are simulated; every other joint is welded at the angle `reset_joints` gives it
    (pr2.py:60-66: the right arm at [-1.75, 1.25, -1.5, -0.5, -1, 0, -1], all others 0).
With the person's right arm in both genders (2 x 10) that is 29 and 31 DoF per env.  Neither robot is `mobile`, so gravity on it is
off (scratch_itch.py:123-126), as on the person and the scratcher."""
import numpy as np

from . import toc
from .human_model import create_human
from .kinematics import q_from_rpy
from .scene import SceneBuilder, quat_from_rpy
from .scratch_itch_batch import R_ELBOW, R_SHOULDER, R_WRIST, RIGHT_ARM_JOINTS, ScratchItchBatch
from .toc import TocPlacement

MOTOR_POSITION = 1

SAWYER = dict(toc.SAWYER, gripper_pos=[0.015, -0.015], tool_pos_offset=[0, 0.125, 0], tool_orient_offset=[0, 0, np.pi / 2.0],
              toc_base_pos_offset=[-0.1, 0, 0.975], ee_orient_rpy=[0, np.pi / 2.0, 0])
PR2 = dict(toc.PR2_LEFT, gripper_pos=[0.25] * 4, tool_pos_offset=[0, 0, 0], tool_orient_offset=[0, 0, 0],
           toc_base_pos_offset=[0.1, 0, 0], ee_orient_rpy=[0, 0, 0])
TARGET_EE_POS = np.array([-0.6, 0, 0.8])             # scratch_itch.py:114


class ScratchItchTocBatch(TocPlacement, ScratchItchBatch):
    """ScratchItch with a robot placed by TOC.  Shares `sample`, the person's reset, `limb_links`, `scratch_params`, `start_fused` and
    `start_coop` with `ScratchItchBatch`; ScratchItchJaco's own template and reset are not touched."""
    R = None

    def __init__(self):
        R = self.R
        b = SceneBuilder()
        self.builder = b
        b.set_gravity([0, 0, -9.81])
        self.plane = b.load_urdf('plane')
        self.load_robot(b)
        self.humans = {}
        for gender, z in (('male', 0.89), ('female', 0.86)):
            hb, info = create_human(b, gender=gender, static=True)
            b.bodies[hb].base_pos = np.array([0, 0.03, z])
            for j in range(b.num_joints(hb)):
                if j not in RIGHT_ARM_JOINTS:
                    b.change_dynamics(hb, j, mass=0)
            b.set_gravity([0, 0, 0], body=hb)                                       # scratch_itch.py:125
            self.humans[gender] = hb
        self.wheelchair = b.load_urdf('wheelchair', base_pos=[0, 0, 0.06], fixed_base=False)     # furniture.py:16, not mounted
        self.tool = b.load_urdf('tool_scratch')
        for j in R['gripper_collision']:                                             # tool.py:41-44 with the left gripper's links
            for tj in (-1, 0, 1):
                b.set_collision_filter_pair(self.robot, self.tool, j, tj, False)
        self.tool_pos_offset = np.array(R['tool_pos_offset'], dtype=np.float64)
        self.tool_quat_offset = quat_from_rpy(R['tool_orient_offset'])
        b.create_fixed_constraint(self.robot, R['tool_joint'], self.tool, -1, self.tool_pos_offset, [0, 0, 0], self.tool_quat_offset, [0, 0, 0, 1], max_force=500)
        b.set_gravity([0, 0, 0], body=self.robot)
        b.set_gravity([0, 0, 0], body=self.tool)
        self.scene = b.finalize()
        sc = self.scene
        self.robot_links(sc)
        self.human_arm_links = {g: [self.gl(hb, j) for j in RIGHT_ARM_JOINTS] for g, hb in self.humans.items()}
        self.obstacles = (self.humans['male'], self.humans['female'], self.wheelchair)      # collision_objects of scratch_itch.py:116

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
        gq = np.tile(R['gripper_pos'], (n, 1)).astype(np.float64)                  # set_gripper_open_position (scratch_itch.py:119)
        ng = len(R['gripper'])
        sim.set_motor(self.arm_links, MOTOR_POSITION, target=q7, kp=[0.05] * 7, kd=[1.0] * 7, max_force=[1.0] * 7)          # robot.py:36-37
        sim.set_motor(self.gripper_links, MOTOR_POSITION, target=gq, kp=[0.05] * ng, kd=[1.0] * ng, max_force=[500.0] * ng)
        sim.forward_kinematics()
        return s

    def arm_points(self, sim, male):
        """The active person's right shoulder, elbow and wrist positions (scratch_itch.py:107-109): three [N, 3] arrays."""
        out = [np.zeros((sim.n, 3)) for _ in range(3)]
        for g, hb in self.humans.items():
            on = male if g == 'male' else ~male
            pos = sim.get_link_states([self.gl(hb, j) for j in (R_SHOULDER, R_ELBOW, R_WRIST)])['pos'].astype(np.float64)
            for k in range(3):
                out[k][on] = pos[on, k]
        return out


class ScratchItchSawyerBatch(ScratchItchTocBatch):
    R = SAWYER


class ScratchItchPR2Batch(ScratchItchTocBatch):
    R = PR2
