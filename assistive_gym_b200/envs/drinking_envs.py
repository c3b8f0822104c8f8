from .agents.human import Human, head_joints
from .agents.robot import PR2, Jaco, Sawyer
from .drinking import DrinkingEnv

robot_arm = 'right'
human_controllable_joint_indices = head_joints


class DrinkingJacoEnv(DrinkingEnv):
    """`assistive_gym:DrinkingJaco-v1` (reference envs/drinking_envs.py:27-29), per-call API path."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=Jaco(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class DrinkingSawyerEnv(DrinkingEnv):
    """`assistive_gym:DrinkingSawyer-v1` (reference envs/drinking_envs.py:23-25): Sawyer beside the wheelchair, its base placed by TOC."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=Sawyer(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class DrinkingPR2Env(DrinkingEnv):
    """`assistive_gym:DrinkingPR2-v1` (reference envs/drinking_envs.py:15-17): PR2's right arm, its base placed by TOC."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)
