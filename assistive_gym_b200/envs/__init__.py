from .bed_bathing_envs import BedBathingSawyerEnv, BedBathingSawyerHumanEnv  # noqa: F401
from .dressing_envs import DressingPR2Env, DressingPR2HumanEnv  # noqa: F401
from .drinking_envs import DrinkingJacoEnv  # noqa: F401
from .feeding_envs import FeedingJacoEnv, FeedingJacoHumanEnv  # noqa: F401
from .scratch_itch_envs import ScratchItchJacoEnv, ScratchItchJacoHumanEnv  # noqa: F401

ENV_REGISTRY = {'FeedingJaco-v1': FeedingJacoEnv, 'BedBathingSawyer-v1': BedBathingSawyerEnv, 'DressingPR2-v1': DressingPR2Env, 'ScratchItchJaco-v1': ScratchItchJacoEnv,
                'FeedingJacoHuman-v1': FeedingJacoHumanEnv, 'ScratchItchJacoHuman-v1': ScratchItchJacoHumanEnv, 'DrinkingJaco-v1': DrinkingJacoEnv,
                'BedBathingSawyerHuman-v1': BedBathingSawyerHumanEnv, 'DressingPR2Human-v1': DressingPR2HumanEnv}


def make(env_id, **kw):
    """`gym.make('assistive_gym:FeedingJaco-v1')` equivalent (reference assistive_gym/__init__.py:6-13).
    Episodes end after 200 steps inside the env itself (feeding.py:37), as in the reference."""
    env_id = env_id.split(':')[-1]
    if env_id not in ENV_REGISTRY:
        raise KeyError('%s is not built on this backend yet (available: %s)' % (env_id, sorted(ENV_REGISTRY)))
    return ENV_REGISTRY[env_id](**kw)
