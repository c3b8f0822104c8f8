from .agents.human import Human, left_arm_joints
from .agents.robot import PR2
from .dressing import DressingEnv

robot_arm = 'left'
human_controllable_joint_indices = left_arm_joints          # dressing_envs.py:13


class DressingPR2Env(DressingEnv):
    """`assistive_gym:DressingPR2-v1` (reference envs/dressing_envs.py:14-16)."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, toc_attempts=50):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config, toc_attempts=toc_attempts)


class DressingPR2HumanEnv(DressingEnv):
    """`assistive_gym:DressingPR2Human-v1` (reference envs/dressing_envs.py:39-42): robot and person are both agents; `step` takes
    {'robot': a7, 'human': a10} and returns dict observations (24 and 28 floats) / rewards / dones (RLlib MultiAgentEnv shape,
    learn.py:41-59).  The person's left arm is driven by its action and kept inside the realistic joint limits while the robot
    pulls the gown's sleeve onto it.  Per-call API path; `step_fused` is the same step on the device."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, toc_attempts=50):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, toc_attempts=toc_attempts)
