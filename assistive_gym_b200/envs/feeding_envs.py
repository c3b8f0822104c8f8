from .agents.human import Human, head_joints
from .agents.robot import PR2, Jaco, Sawyer
from .feeding import FeedingEnv

robot_arm = 'right'
human_controllable_joint_indices = head_joints


class FeedingJacoEnv(FeedingEnv):
    """`assistive_gym:FeedingJaco-v1` (reference envs/feeding_envs.py:29-31)."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=Jaco(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class FeedingJacoHumanEnv(FeedingEnv):
    """`assistive_gym:FeedingJacoHuman-v1` (reference envs/feeding_envs.py:56-59): robot and person are both agents; `step` takes
    {'robot': a7, 'human': a4} and returns dict observations / rewards / dones, as RLlib's MultiAgentEnv expects (learn.py:41-59).
    The person's four head joints are simulated in every env; this path goes through the per-call API (take_step + _get_obs)."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, human_impairment=None):
        super().__init__(robot=Jaco(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, human_impairment=human_impairment)


class FeedingSawyerEnv(FeedingEnv):
    """`assistive_gym:FeedingSawyer-v1` (reference envs/feeding_envs.py:25-27): Sawyer beside the wheelchair, its base placed by TOC."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=Sawyer(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class FeedingPR2Env(FeedingEnv):
    """`assistive_gym:FeedingPR2-v1` (reference envs/feeding_envs.py:17-19): PR2's right arm, its base placed by TOC."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=False),
                         n_envs=n_envs, device=device, seed=seed, config=config)


class FeedingSawyerHumanEnv(FeedingEnv):
    """`assistive_gym:FeedingSawyerHuman-v1` (reference envs/feeding_envs.py:51-54): as FeedingJacoHuman-v1, with Sawyer."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, human_impairment=None):
        super().__init__(robot=Sawyer(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, human_impairment=human_impairment)


class FeedingPR2HumanEnv(FeedingEnv):
    """`assistive_gym:FeedingPR2Human-v1` (reference envs/feeding_envs.py:41-44): as FeedingJacoHuman-v1, with PR2's right arm."""

    def __init__(self, n_envs=1, device=0, seed=1001, config=None, human_impairment=None):
        super().__init__(robot=PR2(robot_arm), human=Human(human_controllable_joint_indices, controllable=True),
                         n_envs=n_envs, device=device, seed=seed, config=config, human_impairment=human_impairment)
