"""DressingSawyer-v1 and DressingJaco-v1 (and their co-optimisation ids) as batched scenes: template construction and batched reset.

The scene is DressingPR2's -- the plain wheelchair, both persons with a live left arm, the gown -- with another robot holding the
gown; the person, the gown's placement, anchors and settle, the motor gains, `dressing_params`, `start_fused` and `start_coop` are
`DressingBatch`'s.  The reset follows `DressingEnv.reset` (dressing.py:112-198) with the robots' `'dressing'` constants of
agents/sawyer.py and agents/jaco.py:
  * Sawyer is placed by `init_robot_pose`'s TOC branch (env.py:276-310) with the arguments of dressing.py:134: base poses on the
    person's left (`right_side=False`) at yaw pi, 50 attempts; the start goal [0.45, -0.3, 1] + U(+-0.05) with
    `toc_ee_orient_rpy[0]`, and the targets 10 cm above the left shoulder / elbow / wrist with the orientations `[-1]`, `[0]`,
    `[0]`; up to three collision rounds of the robot against the person and the wheelchair.  Its 7 arm and 2 gripper joints are
    simulated, every other joint is welded (as in FeedingSawyer).
  * Jaco is mounted on the wheelchair's left: base at wheelchair + [0.35, -0.3, 0.3], yaw +pi/2 (dressing.py:116-118); its start
    pose is `ik_random_restarts(right=False)` to the same randomised goal with [0, -pi/2, 0], resampled while the arm touches the
    person or the wheelchair (robot.py:84-121 with collision_objects).  The reference loads `wheelchair_jaco_left.urdf`, which
    differs from `wheelchair_jaco.urdf` only in the sign of x of the visual origins of the two 1 g mount posts (they have no
    collision shape), so the `wheelchair_jaco` asset is loaded (pinned by tests/test_dressing_robots.py).

The gown collides with every robot link that has a collider: unlike PR2's torso and right arm, Sawyer's and Jaco's links are all
on the arm that holds the gown or within reach of it (Sawyer's pedestal and head stand beside the wheelchair), and the counts stay
inside the 96-link budget of `ag_cloth_init` (tests/test_dressing_robots.py prints them).

The collision rounds check the robot against the person and the wheelchair only, as the reference's do: in about a fifth of the Sawyer
envs the chosen start pose has the forearm touching Sawyer's own pedestal (a pair sawyer.py:55-61 leaves enabled), and the arm is
pushed off it during the settle."""
import numpy as np

from . import toc
from .dressing_batch import DressingBatch
from .kinematics import q_from_rpy
from .scene import quat_from_rpy

TARGET_EE_POS = np.array([0.45, -0.3, 1.0])                  # dressing.py:130
GOAL_OFFSET = np.array([0, 0, 0.1])                          # dressing.py:133

SAWYER = dict(toc.SAWYER, gripper_pos=[0, 0], toc_base_pos_offset=[1.8, 0.7, 0.975],
              ee_orient_rpy=[0, -np.pi / 2.0, 0], ee_orient_shoulder_rpy=[np.pi / 2.0, -np.pi / 2.0, 0])
WHEELCHAIR_POS = np.array([0, 0, 0.06])
JACO = dict(asset='jaco', base_pos=(WHEELCHAIR_POS + [0.35, -0.3, 0.3]).tolist(), base_yaw=np.pi / 2.0, load=dict(self_collision=True),
            arm=[1, 2, 3, 4, 5, 6, 7], ee=8, gripper=[9, 11, 13], tool_joint=8, weld_preset={}, gripper_pos=[1.33] * 3,
            ee_orient_rpy=[0, -np.pi / 2.0, 0])


class DressingSawyerBatch(DressingBatch):
    R = SAWYER
    CLOTH_ROBOT_JOINTS = None

    def _reset_robot(self, sim, s, rng, limb, attempts, outer_iterations):
        """The TOC base pose and start joint angles; a sample that holds `base_pos`, `base_quat` and `q7` (as `reset` leaves it)
        replays that placement instead of searching."""
        n, R = sim.n, self.R
        if 'base_pos' in s:
            base_pos, base_quat, q7 = s['base_pos'].copy(), s['base_quat'].copy(), s['q7'].copy()
            self.goals_reached = s.get('goals_reached')
            self.place_robot(sim, base_pos, base_quat, q7)
            self.unresolved = int(self.colliding(sim).sum())
        else:
            tq = np.tile(q_from_rpy(R['ee_orient_rpy']), (n, 1))
            tqs = np.tile(q_from_rpy(R['ee_orient_shoulder_rpy']), (n, 1))
            goals = [(TARGET_EE_POS + s['ee_offset'], tq), (limb[:, 0] + GOAL_OFFSET, tqs), (limb[:, 1] + GOAL_OFFSET, tq), (limb[:, 2] + GOAL_OFFSET, tq)]
            base_pos, base_quat, q7, _ = self.toc_search(sim, rng, goals, 1, attempts, outer_iterations, right_side=False, base_yaw=np.pi)
            s.update(base_pos=base_pos.copy(), base_quat=base_quat.copy(), q7=q7.copy(), goals_reached=self.goals_reached.copy())
        return base_pos, base_quat, q7, np.tile(R['gripper_pos'], (n, 1)).astype(np.float64)


class DressingJacoBatch(DressingBatch):
    R = JACO
    WHEELCHAIR = 'wheelchair_jaco'
    CLOTH_ROBOT_JOINTS = None

    def load_robot(self, b):
        R = self.R
        self.robot = b.load_urdf(R['asset'], base_pos=R['base_pos'], base_quat=quat_from_rpy([0, 0, R['base_yaw']]), fixed_base=True, **R['load'])
        b.weld_joints(self.robot, set(R['arm']) | set(R['gripper']), R['weld_preset'])

    def robot_links(self, sc):
        super().robot_links(sc)
        self.robot_base_quat = quat_from_rpy([0, 0, self.R['base_yaw']])

    def _reset_robot(self, sim, s, rng, limb, attempts, outer_iterations):
        """The mounted arm's start pose: IK to the randomised goal, resampled (up to 30 times) in the envs where the arm touches the
        person or the wheelchair; a sample that holds `q7` replays it.  `goals_reached` is 1 where the IK met its 1 cm threshold."""
        n, R = sim.n, self.R
        base_pos, base_quat = np.tile(self.robot_base_pos, (n, 1)), np.tile(self.robot_base_quat, (n, 1))
        if 'q7' in s:
            q7 = s['q7'].copy()
            self.goals_reached = s.get('goals_reached')
            self.place_robot(sim, base_pos, base_quat, q7)
            self.unresolved = int(self.colliding(sim).sum())
        else:
            target = TARGET_EE_POS + s['ee_offset']
            tq = q_from_rpy(R['ee_orient_rpy'])
            q7, err = self._solve_ik(sim, rng, target, tq, None)
            for attempt in range(31):
                self.place_robot(sim, base_pos, base_quat, q7)
                hit = self.colliding(sim)
                if not hit.any() or attempt == 30:
                    break
                q2, e2 = self._solve_ik(sim, rng, target, tq, hit)
                q7[hit], err[hit] = q2[hit], e2[hit]
            self.unresolved = int(hit.sum())
            self.ik_err = err
            self.goals_reached = (err < 0.01).astype(int)
            s.update(q7=q7.copy(), goals_reached=self.goals_reached.copy())
        return base_pos, base_quat, q7, np.tile(R['gripper_pos'], (n, 1)).astype(np.float64)

    def _solve_ik(self, sim, rng, target, tq, mask):
        q7, err = sim.ik_solve(self.arm_links, self.ee_link, target, tq, max_restarts=20, iters=120, threshold=0.01, seed=int(rng.integers(1, 2 ** 31 - 1)),
                               mask=None if mask is None else mask.astype(np.int32))
        return q7.astype(np.float64), err.astype(np.float64)
