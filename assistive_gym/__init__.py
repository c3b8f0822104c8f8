"""`import assistive_gym` drop-in for the reference package (reference assistive_gym/__init__.py:1-33).

Registers the `-v1` ids this backend has built with gym (when gym is importable), exactly as the reference does, so that
`gym.make('assistive_gym:FeedingJaco-v1')` and `learn.py:61-69 make_env` resolve to the H100 batched backend with
`n_envs=1`; `assistive_gym.make(id, n_envs=...)` gives the batched env without gym.  Ids the backend has not built
raise the registry's KeyError (nothing is silently substituted)."""
from assistive_gym_b200.envs import ENV_REGISTRY, make  # noqa: F401

__agphys_shim__ = True          # bench.py's reference arm must not mistake this package for the real reference

try:                                        # pragma: no cover - depends on the box
    from gym.envs.registration import register
    for _id in ENV_REGISTRY:
        register(id=_id, entry_point='assistive_gym.envs:%sEnv' % _id.split('-')[0], max_episode_steps=200)
except Exception:                           # gym absent (build container) or already registered
    pass
