"""`Robot` / `Jaco` — robot metadata of the reference (envs/agents/robot.py:5-39, jaco.py:8-54).
Only the constants the hot path needs are carried; IK lives in `feeding_batch.py` / `kinematics.py`."""
import numpy as np

from .agent import Agent


class Robot(Agent):
    def __init__(self, controllable_joints, right_arm_joint_indices, left_arm_joint_indices, wheel_joint_indices,
                 right_end_effector, left_end_effector, right_gripper_indices, left_gripper_indices, gripper_pos,
                 right_tool_joint, left_tool_joint, tool_pos_offset, tool_orient_offset, right_gripper_collision_indices,
                 left_gripper_collision_indices, toc_base_pos_offset, toc_ee_orient_rpy, wheelchair_mounted,
                 half_range=False, action_duplication=None, action_multiplier=1, flags=None):
        super().__init__()
        self.controllable_joints = controllable_joints
        self.right_arm_joint_indices, self.left_arm_joint_indices = right_arm_joint_indices, left_arm_joint_indices
        self.wheel_joint_indices = wheel_joint_indices
        self.mobile = 'wheel' in controllable_joints
        self.controllable_joint_indices = (self.wheel_joint_indices if self.mobile else []) + (
            right_arm_joint_indices if 'right' in controllable_joints else left_arm_joint_indices if 'left' in controllable_joints
            else right_arm_joint_indices + left_arm_joint_indices)
        self.right_end_effector, self.left_end_effector = right_end_effector, left_end_effector
        self.right_gripper_indices, self.left_gripper_indices = right_gripper_indices, left_gripper_indices
        self.gripper_pos = gripper_pos
        self.right_tool_joint, self.left_tool_joint = right_tool_joint, left_tool_joint
        self.tool_pos_offset, self.tool_orient_offset = tool_pos_offset, tool_orient_offset
        self.right_gripper_collision_indices, self.left_gripper_collision_indices = right_gripper_collision_indices, left_gripper_collision_indices
        self.toc_base_pos_offset, self.toc_ee_orient_rpy = toc_base_pos_offset, toc_ee_orient_rpy
        self.wheelchair_mounted = wheelchair_mounted
        self.half_range = half_range
        self.action_duplication, self.action_multiplier = action_duplication, action_multiplier
        self.flags = flags
        self.has_single_arm = right_end_effector == left_end_effector
        self.motor_forces = 1.0          # robot.py:36
        self.motor_gains = 0.05          # robot.py:37
        self.skip_pose_optimization = False

    def init(self, body, sim, np_random):
        super().init(body, sim, np_random)
        self.right_arm_lower_limits = [self.lower_limits[i] for i in self.right_arm_joint_indices]
        self.right_arm_upper_limits = [self.upper_limits[i] for i in self.right_arm_joint_indices]

    def set_gripper_open_position(self, indices, positions, set_instantly=False, force=500):
        n = len(indices)
        tgt = np.broadcast_to(np.asarray(positions, dtype=np.float32), (self.sim.n, n))
        self.sim.set_motor([self._gl(j) for j in indices], 1, target=tgt, kp=[0.05] * n, kd=[1.0] * n, max_force=[force] * n)
        if set_instantly:
            self.set_joint_angles(indices, positions, use_limits=True)


class Jaco(Robot):
    def __init__(self, controllable_joints='right'):
        arm = [1, 2, 3, 4, 5, 6, 7]
        pos = [-0.35, -0.3, 0.3]
        super().__init__(controllable_joints, arm, arm, [], 8, 8, [9, 11, 13], [9, 11, 13],
                         {'scratch_itch': [1] * 3, 'feeding': [1.33] * 3, 'drinking': [0.63] * 3, 'bed_bathing': [1.1] * 3,
                          'dressing': [1.33] * 3, 'arm_manipulation': [1.05] * 3},
                         8, 8,
                         {'scratch_itch': [0, 0, 0.02], 'feeding': [0.1, -0.0225, 0.03], 'drinking': [0.05, -0.005, 0],
                          'bed_bathing': [-0.01, 0, 0.03], 'arm_manipulation': [0.075, 0, 0.14]},
                         {'scratch_itch': [0, -np.pi / 2.0, 0], 'feeding': [-0.1, -np.pi / 2.0, 0], 'drinking': [0, -np.pi / 2.0, np.pi / 2.0],
                          'bed_bathing': [0, -np.pi / 2.0, 0], 'arm_manipulation': [np.pi / 2.0, -np.pi / 2.0, 0]},
                         list(range(7, 15)), list(range(7, 15)),
                         {'scratch_itch': pos, 'feeding': pos, 'drinking': pos, 'bed_bathing': [-0.05, 1.05, 0.6],
                          'dressing': [0.35, -0.3, 0.3], 'arm_manipulation': [-0.25, 1.15, 0.6]},
                         {'scratch_itch': [0, np.pi / 2.0, 0], 'feeding': [np.pi / 2.0, 0, np.pi / 2.0], 'drinking': [0, np.pi / 2.0, 0],
                          'bed_bathing': [0, np.pi / 2.0, 0], 'dressing': [[0, -np.pi / 2.0, 0]], 'arm_manipulation': [0, np.pi / 2.0, 0]},
                         wheelchair_mounted=True, half_range=False)


class Sawyer(Robot):
    """reference envs/agents/sawyer.py:6-49 (the constants of the hot path)."""

    def __init__(self, controllable_joints='right'):
        arm = [3, 8, 9, 10, 11, 13, 16]
        super().__init__(controllable_joints, arm, arm, [], 19, 19, [20, 22], [20, 22],
                         {'scratch_itch': [0.015, -0.015], 'feeding': [0, 0], 'drinking': [0.025, -0.025], 'bed_bathing': [0.0125, -0.0125],
                          'dressing': [0, 0], 'arm_manipulation': [0.01, -0.01]},
                         18, 18,
                         {'scratch_itch': [0, 0.125, 0], 'feeding': [-0.1, 0.12, -0.02], 'drinking': [0.05, 0.125, 0],
                          'bed_bathing': [0, 0.1175, 0], 'arm_manipulation': [0.075, 0.235, 0]},
                         {'scratch_itch': [0, 0, np.pi / 2.0], 'feeding': [np.pi / 2.0 - 0.1, 0, np.pi / 2.0], 'drinking': [0, 0, np.pi / 2.0],
                          'bed_bathing': [np.pi / 2.0, 0, np.pi / 2.0], 'arm_manipulation': [0, 0, np.pi / 2.0]},
                         [18, 20, 21, 22, 23], [18, 20, 21, 22, 23],
                         {'scratch_itch': [-0.1, 0, 0.975], 'feeding': [-0.1, 0.2, 0.975], 'drinking': [-0.1, 0.2, 0.975],
                          'bed_bathing': [-0.2, 0, 0.975], 'dressing': [1.8, 0.7, 0.975], 'arm_manipulation': [-0.3, 0.6, 0.975]},
                         {'scratch_itch': [0, np.pi / 2.0, 0], 'feeding': [np.pi / 2.0, 0, np.pi / 2.0], 'drinking': [0, -np.pi / 2.0, np.pi],
                          'bed_bathing': [0, np.pi / 2.0, 0], 'dressing': [[0, -np.pi / 2.0, 0], [np.pi / 2.0, -np.pi / 2.0, 0]],
                          'arm_manipulation': [0, -np.pi / 2.0, np.pi]},
                         wheelchair_mounted=False, half_range=False)


class PR2(Robot):
    """reference envs/agents/pr2.py:7-49 (the constants of the ScratchItch, Feeding, Drinking, BedBathing and Dressing hot paths; the wheel /
    right-arm tables are kept because `controllable_joints` selects among them)."""

    def __init__(self, controllable_joints='right'):
        super().__init__(controllable_joints, [42, 43, 44, 46, 47, 49, 50], [64, 65, 66, 68, 69, 71, 72], list(range(3, 15)), 54, 76,
                         [57, 58, 59, 60], [79, 80, 81, 82],
                         {'scratch_itch': [0.25] * 4, 'feeding': [0.03] * 4, 'drinking': [0.45] * 4, 'bed_bathing': [0.2] * 4, 'dressing': [0] * 4}, 54, 76,
                         {'scratch_itch': [0, 0, 0], 'feeding': [0, -0.03, -0.11], 'drinking': [-0.01, 0, -0.05], 'bed_bathing': [0, 0, 0]},
                         {'scratch_itch': [0, 0, 0], 'feeding': [-0.2, 0, 0], 'drinking': [np.pi / 2.0, 0, 0], 'bed_bathing': [0, 0, 0]},
                         list(range(49, 64)), list(range(71, 86)),
                         {'scratch_itch': [0.1, 0, 0], 'feeding': [0.1, 0.2, 0], 'drinking': [0.2, 0.2, 0], 'bed_bathing': [-0.1, 0, 0], 'dressing': [1.7, 0.7, 0]},
                         {'scratch_itch': [0, 0, 0], 'feeding': [np.pi / 2.0, 0, 0], 'drinking': [0, 0, 0], 'bed_bathing': [0, 0, 0],
                          'dressing': [[0, 0, np.pi], [0, 0, np.pi * 3 / 2.0]]},
                         wheelchair_mounted=False, half_range=False)
