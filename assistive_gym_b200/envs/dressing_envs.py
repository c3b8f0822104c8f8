from .agents.human import Human, left_arm_joints
from .agents.robot import PR2, Jaco, Sawyer
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

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, toc_attempts=50, human_impairment=None):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, toc_attempts=toc_attempts, human_impairment=human_impairment)


class DressingSawyerEnv(DressingEnv):
    """`assistive_gym:DressingSawyer-v1` (reference envs/dressing_envs.py:23-25): Sawyer beside the wheelchair, its base placed by TOC."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, toc_attempts=50):
        super().__init__(robot=Sawyer(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config, toc_attempts=toc_attempts)


class DressingJacoEnv(DressingEnv):
    """`assistive_gym:DressingJaco-v1` (reference envs/dressing_envs.py:27-29): Jaco mounted on the wheelchair's left."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, toc_attempts=50):
        super().__init__(robot=Jaco(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config, toc_attempts=toc_attempts)


class DressingSawyerHumanEnv(DressingEnv):
    """`assistive_gym:DressingSawyerHuman-v1` (reference envs/dressing_envs.py:49-52): DressingPR2Human-v1's two agents with Sawyer."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, toc_attempts=50, human_impairment=None):
        super().__init__(robot=Sawyer(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, toc_attempts=toc_attempts, human_impairment=human_impairment)


class DressingJacoHumanEnv(DressingEnv):
    """`assistive_gym:DressingJacoHuman-v1` (reference envs/dressing_envs.py:54-57): DressingPR2Human-v1's two agents with Jaco."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, toc_attempts=50, human_impairment=None):
        super().__init__(robot=Jaco(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, toc_attempts=toc_attempts, human_impairment=human_impairment)
