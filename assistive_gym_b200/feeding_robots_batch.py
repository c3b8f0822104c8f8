"""FeedingSawyer-v1 and FeedingPR2-v1 (and their co-optimisation ids) as batched scenes: template construction and batched reset.

The scene is FeedingJaco's -- person pair, wheelchair, table, bowl, the spoon on a fixed constraint, eight food spheres -- with another
robot.  Robots that are not wheelchair-mounted load the plain wheelchair (furniture.py:16) and find their base pose with
`init_robot_pose`'s TOC branch (env.py:276-310 -> robot.py:123-215): `attempts` random base poses beside the person, ranked by goals
reached and JLWKI, then a collision check of robot and spoon against person, table and wheelchair, re-searching only the colliding
envs for up to `max_iterations` rounds.  The goals are feeding.py:141's: two start goals (the randomised spoon pose with the task's
end-effector orientation, and the mouth by position) that a base pose must both reach, and one target goal (the mouth with the
end-effector orientation).  The task constants are the reference's `'feeding'` entries of agents/sawyer.py:8-47 and agents/pr2.py:8-47.

Differences forced by the per-env DoF budget (32 per env, 16 per articulation; DESIGN.md section 9):
  * Sawyer: the 7 arm joints and the 2 gripper joints are simulated; every other joint (the head pan) is welded at 0.
  * PR2: the right arm (7) and the right gripper (4) are simulated; every other joint is welded at the angle `reset_joints` gives it
    (pr2.py:60-66: the left arm at [1.75, 1.25, 1.5, -0.5, 1, 0, 1], all others 0), as dressing_batch.py does for the other arm.
Neither robot is `mobile`, so gravity on it is off (feeding.py:150-151)."""
import numpy as np

from . import toc
from .feeding_batch import TREMOR_JOINTS, FeedingBatch
from .human_model import create_human
from .kinematics import BodyKinematics, q_from_rpy
from .scene import SceneBuilder, quat_from_rpy
from .toc import TocPlacement

MOTOR_POSITION = 1

SAWYER = dict(toc.SAWYER, gripper_pos=[0.0, 0.0], tool_pos_offset=[-0.1, 0.12, -0.02], tool_orient_offset=[np.pi / 2.0 - 0.1, 0, np.pi / 2.0],
              toc_base_pos_offset=[-0.1, 0.2, 0.975], ee_orient_rpy=[np.pi / 2.0, 0, np.pi / 2.0])
PR2 = dict(toc.PR2_RIGHT, gripper_pos=[0.03] * 4, tool_pos_offset=[0, -0.03, -0.11], tool_orient_offset=[-0.2, 0, 0],
           toc_base_pos_offset=[0.1, 0.2, 0], ee_orient_rpy=[np.pi / 2.0, 0, 0])
TARGET_EE_POS = np.array([-0.15, -0.65, 1.15])       # feeding.py:139


class FeedingTocBatch(TocPlacement, FeedingBatch):
    """Feeding with a robot placed by TOC.  Shares `sample`, the person, the bowl and the food, `feeding_params`, `start_fused` and
    `start_coop` with `FeedingBatch`; FeedingJaco's own template and reset are not touched."""
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
                if j not in TREMOR_JOINTS:
                    b.change_dynamics(hb, j, mass=0)
            self.humans[gender] = hb
        self.wheelchair = b.load_urdf('wheelchair', base_pos=[0, 0, 0.06], fixed_base=False)     # furniture.py:16, not mounted
        self.table = b.load_urdf('table_tall', base_pos=[0.25, -1.0, 0])
        sp_shape = b.create_collision_shape('mesh', mesh_asset='spoon_vhacd', mesh_scale=[0.08] * 3)
        self.tool = b.create_multibody(base_mass=1.0, base_shape=sp_shape, name='spoon')
        for j in R['gripper_collision']:
            b.set_collision_filter_pair(self.robot, self.tool, j, -1, False)
        self.tool_pos_offset = np.array(R['tool_pos_offset'], dtype=np.float64)
        self.tool_quat_offset = quat_from_rpy(R['tool_orient_offset'])
        b.create_fixed_constraint(self.robot, R['tool_joint'], self.tool, -1, self.tool_pos_offset, [0, 0, 0],
                                  self.tool_quat_offset, [0, 0, 0, 1], max_force=500)
        self.bowl = b.load_urdf('bowl', base_pos=[-0.15, -0.65, 0.75])
        fs = b.create_collision_shape('sphere', radius=0.005)
        self.foods = [b.create_multibody(base_mass=0.001, base_shape=fs, name='food%d' % i) for i in range(8)]
        b.set_gravity([0, 0, 0], body=self.robot)
        for hb in self.humans.values():
            b.set_gravity([0, 0, 0], body=hb)
        b.set_gravity([0, 0, 0], body=self.tool)
        self.scene = b.finalize()
        sc = self.scene
        self.robot_links(sc)
        self.hkin = {g: BodyKinematics(sc, hb) for g, hb in self.humans.items()}
        self.mouth = {'male': np.array([0, -0.11, 0.03]), 'female': np.array([0, -0.1, 0.03])}
        self.obstacles = (self.humans['male'], self.humans['female'], self.table, self.wheelchair)     # env.py:300-309

    def reset(self, sim, rng, settle_steps=25, sample=None, impairment='random', simulate_head=False, attempts=50, max_iterations=3):
        """Put every env of `sim` into a fresh start state.  A sample that holds `base_pos`, `base_quat` and `q7` (as `reset` leaves
        it) replays that robot placement instead of searching."""
        n = sim.n
        s = dict(sample) if sample else self.sample(n, rng, impairment)
        self.last_sample = s
        self._reset_person(sim, s, simulate_head)
        sp = self._reset_toc_robot(sim, s, rng, attempts, max_iterations)
        self._reset_bowl_food(sim, s, sp, settle_steps)
        return s

    def _reset_toc_robot(self, sim, s, rng, attempts, max_iterations):
        n, R = sim.n, self.R
        male = s['male'].astype(bool)
        if 'base_pos' in s:
            base_pos, base_quat, q7 = s['base_pos'].copy(), s['base_quat'].copy(), s['q7'].copy()
            self.goals_reached = s.get('goals_reached')
            sp = self.place_robot(sim, base_pos, base_quat, q7)
            self.unresolved = int(self.colliding(sim).sum())
        else:
            mouth = self.mouth_target(sim, male)
            target = TARGET_EE_POS + s['ee_offset']
            tq = np.tile(q_from_rpy(R['ee_orient_rpy']), (n, 1))
            base_pos, base_quat, q7, sp = self.toc_search(sim, rng, [(target, tq), (mouth, None), (mouth, tq)], 2, attempts, max_iterations)
            reached = self.goals_reached
            s.update(base_pos=base_pos.copy(), base_quat=base_quat.copy(), q7=q7.copy(), goals_reached=reached.copy())
        gq = np.tile(R['gripper_pos'], (n, 1)).astype(np.float64)
        ng = len(R['gripper'])
        sim.set_motor(self.arm_links, MOTOR_POSITION, target=q7, kp=[0.025] * 7, kd=[1.0] * 7, max_force=[1.0] * 7)       # feeding.py:122
        sim.set_motor(self.gripper_links, MOTOR_POSITION, target=gq, kp=[0.05] * ng, kd=[1.0] * ng, max_force=[500.0] * ng)
        return sp


class FeedingSawyerBatch(FeedingTocBatch):
    R = SAWYER


class FeedingPR2Batch(FeedingTocBatch):
    R = PR2
