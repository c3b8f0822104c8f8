from .bed_bathing_envs import BedBathingSawyerEnv, BedBathingSawyerHumanEnv  # noqa: F401
from .dressing_envs import DressingJacoEnv, DressingJacoHumanEnv, DressingPR2Env, DressingPR2HumanEnv, DressingSawyerEnv, DressingSawyerHumanEnv  # noqa: F401
from .drinking_envs import DrinkingJacoEnv, DrinkingPR2Env, DrinkingSawyerEnv  # noqa: F401
from .feeding_envs import FeedingJacoEnv, FeedingJacoHumanEnv, FeedingPR2Env, FeedingPR2HumanEnv, FeedingSawyerEnv, FeedingSawyerHumanEnv  # noqa: F401
from .scratch_itch_envs import ScratchItchJacoEnv, ScratchItchJacoHumanEnv, ScratchItchPR2Env, ScratchItchPR2HumanEnv, ScratchItchSawyerEnv, ScratchItchSawyerHumanEnv  # noqa: F401

ENV_REGISTRY = {'FeedingJaco-v1': FeedingJacoEnv, 'BedBathingSawyer-v1': BedBathingSawyerEnv, 'DressingPR2-v1': DressingPR2Env, 'ScratchItchJaco-v1': ScratchItchJacoEnv,
                'FeedingJacoHuman-v1': FeedingJacoHumanEnv, 'ScratchItchJacoHuman-v1': ScratchItchJacoHumanEnv, 'DrinkingJaco-v1': DrinkingJacoEnv,
                'BedBathingSawyerHuman-v1': BedBathingSawyerHumanEnv, 'DressingPR2Human-v1': DressingPR2HumanEnv,
                'FeedingSawyer-v1': FeedingSawyerEnv, 'FeedingPR2-v1': FeedingPR2Env, 'FeedingSawyerHuman-v1': FeedingSawyerHumanEnv,
                'FeedingPR2Human-v1': FeedingPR2HumanEnv, 'ScratchItchSawyer-v1': ScratchItchSawyerEnv, 'ScratchItchPR2-v1': ScratchItchPR2Env,
                'ScratchItchSawyerHuman-v1': ScratchItchSawyerHumanEnv, 'ScratchItchPR2Human-v1': ScratchItchPR2HumanEnv,
                'DrinkingSawyer-v1': DrinkingSawyerEnv, 'DrinkingPR2-v1': DrinkingPR2Env,
                'DressingSawyer-v1': DressingSawyerEnv, 'DressingJaco-v1': DressingJacoEnv, 'DressingSawyerHuman-v1': DressingSawyerHumanEnv,
                'DressingJacoHuman-v1': DressingJacoHumanEnv}


def make(env_id, **kw):
    """`gym.make('assistive_gym:FeedingJaco-v1')` equivalent (reference assistive_gym/__init__.py:6-13).
    Episodes end after 200 steps inside the env itself (feeding.py:37), as in the reference."""
    env_id = env_id.split(':')[-1]
    if env_id not in ENV_REGISTRY:
        raise KeyError('%s is not built on this backend yet (available: %s)' % (env_id, sorted(ENV_REGISTRY)))
    return ENV_REGISTRY[env_id](**kw)
