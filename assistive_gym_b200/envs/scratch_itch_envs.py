from .agents.human import Human, right_arm_joints
from .agents.robot import PR2, Jaco, Sawyer
from .scratch_itch import ScratchItchEnv

robot_arm = 'left'
human_controllable_joint_indices = right_arm_joints         # scratch_itch_envs.py:15


class ScratchItchJacoEnv(ScratchItchEnv):
    """`assistive_gym:ScratchItchJaco-v1` (reference envs/scratch_itch_envs.py)."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=Jaco(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class ScratchItchJacoHumanEnv(ScratchItchEnv):
    """`assistive_gym:ScratchItchJacoHuman-v1` (reference envs/scratch_itch_envs.py): robot and person are both agents; `step` takes
    {'robot': a7, 'human': a10} and returns dict observations / rewards / dones (RLlib MultiAgentEnv shape, learn.py:41-59).  The
    person's right arm is driven by its action and kept inside the realistic joint limits; per-call API path."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, human_impairment=None):
        super().__init__(robot=Jaco(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, human_impairment=human_impairment)


class ScratchItchSawyerEnv(ScratchItchEnv):
    """`assistive_gym:ScratchItchSawyer-v1` (reference envs/scratch_itch_envs.py:25-27): Sawyer beside the wheelchair, its base placed by TOC."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=Sawyer(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class ScratchItchPR2Env(ScratchItchEnv):
    """`assistive_gym:ScratchItchPR2-v1` (reference envs/scratch_itch_envs.py:17-19): PR2's left arm, its base placed by TOC."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class ScratchItchSawyerHumanEnv(ScratchItchEnv):
    """`assistive_gym:ScratchItchSawyerHuman-v1` (reference envs/scratch_itch_envs.py:51-54): as ScratchItchJacoHuman-v1, with Sawyer."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, human_impairment=None):
        super().__init__(robot=Sawyer(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, human_impairment=human_impairment)


class ScratchItchPR2HumanEnv(ScratchItchEnv):
    """`assistive_gym:ScratchItchPR2Human-v1` (reference envs/scratch_itch_envs.py:41-44): as ScratchItchJacoHuman-v1, with PR2's left arm."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, human_impairment=None):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, human_impairment=human_impairment)
