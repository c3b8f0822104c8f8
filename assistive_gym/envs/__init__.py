"""`assistive_gym.envs` of the drop-in shim: the env classes the reference exports for the ids built here
(reference assistive_gym/envs/__init__.py), so `getattr(importlib.import_module('assistive_gym.envs'), name + 'Env')`
(learn.py:65-66) works."""
from assistive_gym_b200.envs import BedBathingSawyerEnv, BedBathingSawyerHumanEnv, DressingPR2Env, DressingPR2HumanEnv, DrinkingJacoEnv, FeedingJacoEnv, FeedingJacoHumanEnv, ScratchItchJacoEnv, ScratchItchJacoHumanEnv  # noqa: F401
