from .agents.human import Human
from .agents.robot import PR2, Sawyer
from .bed_bathing import BedBathingEnv

robot_arm = 'left'
human_controllable_joint_indices = list(range(0, 10))      # human.right_arm_joints (bed_bathing_envs.py)


class BedBathingSawyerEnv(BedBathingEnv):
    """`assistive_gym:BedBathingSawyer-v1` (reference envs/bed_bathing_envs.py)."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=Sawyer(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class BedBathingSawyerHumanEnv(BedBathingEnv):
    """`assistive_gym:BedBathingSawyerHuman-v1` (reference envs/bed_bathing_envs.py): robot and person are both agents; `step` takes
    {'robot': a7, 'human': a10} and returns dict observations (24 and 28 floats) / rewards / dones (RLlib MultiAgentEnv shape,
    learn.py:41-59).  The person's right arm is driven by its action and kept inside the realistic joint limits; the wiping targets
    follow the arm.  Per-call API path; `step_fused` is the same step on the device."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=Sawyer(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class BedBathingPR2Env(BedBathingEnv):
    """`assistive_gym:BedBathingPR2-v1` (reference envs/bed_bathing_envs.py:15-17): PR2's left arm, its base placed by TOC."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class BedBathingPR2HumanEnv(BedBathingEnv):
    """`assistive_gym:BedBathingPR2Human-v1` (reference envs/bed_bathing_envs.py:39-41): as BedBathingSawyerHuman-v1, with PR2's left arm."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config)
