"""`assistive_gym.envs` of the drop-in shim: the env classes the reference exports for the ids built here
(reference assistive_gym/envs/__init__.py), so `getattr(importlib.import_module('assistive_gym.envs'), name + 'Env')`
(learn.py:65-66) works."""
from assistive_gym_b200.envs import BedBathingSawyerEnv, BedBathingSawyerHumanEnv, DressingJacoEnv, DressingJacoHumanEnv, DressingPR2Env, DressingPR2HumanEnv, DressingSawyerEnv, DressingSawyerHumanEnv, DrinkingJacoEnv, DrinkingPR2Env, DrinkingSawyerEnv, FeedingJacoEnv, FeedingJacoHumanEnv, FeedingPR2Env, FeedingPR2HumanEnv, FeedingSawyerEnv, FeedingSawyerHumanEnv, ScratchItchJacoEnv, ScratchItchJacoHumanEnv, ScratchItchPR2Env, ScratchItchPR2HumanEnv, ScratchItchSawyerEnv, ScratchItchSawyerHumanEnv  # noqa: F401
