"""DrinkingSawyer-v1 and DrinkingPR2-v1 as batched scenes: template construction and batched reset.

The scene is DrinkingJaco's -- person pair, the cup (`cup_vhacd` at scale 0.045, mass 1) on a fixed constraint at the robot's right
tool joint, 64 water spheres -- with another robot beside the plain wheelchair (furniture.py:16).  The reset follows
`DrinkingEnv.reset` (drinking.py:122-183): the person with DrinkingJaco's presets and head draw, then `init_robot_pose`'s TOC branch
(env.py:276-310 -> robot.py:123-221): two start goals (the randomised cup pose [-0.2, -0.5, 1.1] + U(+-0.05) with the task's
end-effector orientation, and the mouth by position) that a base pose must both reach and one target goal (the mouth with that
orientation), 50 base poses, and up to three collision-check rounds of robot and cup against the person and the wheelchair that
re-search only the colliding envs; then the open gripper, the robot's motor gains of drinking.py:130 (0.005), the water grid over
the cup's centre of mass and the 50-step settle.  The task constants are the reference's `'drinking'` entries of agents/sawyer.py:21-43
and agents/pr2.py:21-43.

Arm, gripper, tool joint and welded joints are FeedingSawyer's and FeedingPR2's (feeding_robots_batch.py): Sawyer simulates its 7 arm
joints and 2 gripper joints, PR2 its right arm and right gripper with the left arm welded at [1.75, 1.25, 1.5, -0.5, 1, 0, 1].  Neither
robot is `mobile`, so gravity on it is off (drinking.py:152-155), as on the person and the cup."""
import numpy as np

from . import toc
from .drinking_batch import N_WATER, WATER_MASS, WATER_RADIUS, DrinkingBatch
from .feeding_batch import TREMOR_JOINTS
from .human_model import create_human
from .kinematics import BodyKinematics, q_from_rpy
from .scene import SceneBuilder, quat_from_rpy
from .toc import TocPlacement

MOTOR_POSITION = 1

SAWYER = dict(toc.SAWYER, gripper_pos=[0.025, -0.025], tool_pos_offset=[0.05, 0.125, 0], tool_orient_offset=[0, 0, np.pi / 2.0],
              toc_base_pos_offset=[-0.1, 0.2, 0.975], ee_orient_rpy=[0, -np.pi / 2.0, np.pi])
PR2 = dict(toc.PR2_RIGHT, gripper_pos=[0.45] * 4, tool_pos_offset=[-0.01, 0, -0.05], tool_orient_offset=[np.pi / 2.0, 0, 0],
           toc_base_pos_offset=[0.2, 0.2, 0], ee_orient_rpy=[0, 0, 0])
TARGET_EE_POS = np.array([-0.2, -0.5, 1.1])          # drinking.py:145


class DrinkingTocBatch(TocPlacement, DrinkingBatch):
    """Drinking with a robot placed by TOC.  Shares `sample`, the person's reset, the water grid and its settle, `drinking_params`,
    `start_fused` and `cup_frame` with `DrinkingBatch`; DrinkingJaco's own template and reset are not touched."""
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
        cup_shape = b.create_collision_shape('mesh', mesh_asset='cup_vhacd', mesh_scale=[0.045] * 3)          # tool.py:23-34, drinking.py:136
        self.tool = b.create_multibody(base_mass=1.0, base_shape=cup_shape, name='cup')
        for j in R['gripper_collision']:
            b.set_collision_filter_pair(self.robot, self.tool, j, -1, False)
        self.tool_pos_offset = np.array(R['tool_pos_offset'], dtype=np.float64)
        self.tool_quat_offset = quat_from_rpy(R['tool_orient_offset'])
        b.create_fixed_constraint(self.robot, R['tool_joint'], self.tool, -1, self.tool_pos_offset, [0, 0, 0], self.tool_quat_offset, [0, 0, 0, 1], max_force=500)
        ws = b.create_collision_shape('sphere', radius=WATER_RADIUS)
        self.waters = [b.create_multibody(base_mass=WATER_MASS, base_shape=ws, name='water%d' % i) for i in range(N_WATER)]
        self.foods = self.waters
        b.set_gravity([0, 0, 0], body=self.robot)
        for hb in self.humans.values():
            b.set_gravity([0, 0, 0], body=hb)
        b.set_gravity([0, 0, 0], body=self.tool)
        self.scene = b.finalize()
        sc = self.scene
        self.robot_links(sc)
        self.hkin = {g: BodyKinematics(sc, hb) for g, hb in self.humans.items()}
        self.mouth = {'male': np.array([0, -0.11, 0.03]), 'female': np.array([0, -0.1, 0.03])}          # drinking.py:187
        self.obstacles = (self.humans['male'], self.humans['female'], self.wheelchair)      # collision_objects of drinking.py:147

    def reset(self, sim, rng, settle_steps=50, sample=None, impairment='random', simulate_head=False, attempts=50, max_iterations=3):
        """Put every env of `sim` into a fresh start state.  A sample that holds `base_pos`, `base_quat` and `q7` (as `reset` leaves
        it) replays that robot placement instead of searching."""
        n = sim.n
        s = dict(sample) if sample else self.sample(n, rng, impairment)
        self.last_sample = s
        self._reset_person(sim, s, simulate_head)
        self._reset_toc_robot(sim, s, rng, attempts, max_iterations)
        self._reset_water(sim, settle_steps)
        return s

    def _reset_toc_robot(self, sim, s, rng, attempts, max_iterations):
        n, R = sim.n, self.R
        if 'base_pos' in s:
            base_pos, base_quat, q7 = s['base_pos'].copy(), s['base_quat'].copy(), s['q7'].copy()
            self.goals_reached = s.get('goals_reached')
            self.place_robot(sim, base_pos, base_quat, q7)
            self.unresolved = int(self.colliding(sim).sum())
        else:
            mouth = self.mouth_target(sim, s['male'].astype(bool))
            target = TARGET_EE_POS + s['ee_offset']
            tq = np.tile(q_from_rpy(R['ee_orient_rpy']), (n, 1))
            base_pos, base_quat, q7, _ = self.toc_search(sim, rng, [(target, tq), (mouth, None), (mouth, tq)], 2, attempts, max_iterations)
            s.update(base_pos=base_pos.copy(), base_quat=base_quat.copy(), q7=q7.copy(), goals_reached=self.goals_reached.copy())
        gq = np.tile(R['gripper_pos'], (n, 1)).astype(np.float64)                  # set_gripper_open_position (drinking.py:150)
        ng = len(R['gripper'])
        sim.set_motor(self.arm_links, MOTOR_POSITION, target=q7, kp=[0.005] * 7, kd=[1.0] * 7, max_force=[1.0] * 7)          # drinking.py:130
        sim.set_motor(self.gripper_links, MOTOR_POSITION, target=gq, kp=[0.05] * ng, kd=[1.0] * ng, max_force=[500.0] * ng)


class DrinkingSawyerBatch(DrinkingTocBatch):
    R = SAWYER


class DrinkingPR2Batch(DrinkingTocBatch):
    R = PR2
