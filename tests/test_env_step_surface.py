"""What `reset`, `step`, `step_fused` and `step_reference_api` return for every registered id, at one env and at two: Python types,
dict / list structure, keys, array dtypes and shapes.  The tasks differ on purpose, and each difference is written out below:

- FeedingEnv.step (single agent) returns a list of per-env info dicts of Python scalars when n_envs > 1; the other fused steps
  return one dict of arrays.
- DrinkingEnv.step is the per-call step and step_fused the fused one; both return float64 obs and reward.  The other single-agent
  steps are fused and return float32 obs and reward.
- step_reference_api of Feeding and ScratchItch keeps info as it is and the reward a NumPy value when n_envs == 1; Dressing's and
  BedBathing's unwrap info and return a float reward and a bool done.
- step_fused of a single-agent id other than Drinking raises RuntimeError."""
import numpy as np
import pytest

from assistive_gym_b200 import envs

F32, F64, I64, BOOL = np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.int64), np.dtype(bool)


def _check(x, spec, where='out'):
    """`spec`: a type (`type(x) is spec`), a (dtype, shape) tuple for an ndarray, or a dict / list of specs"""
    if isinstance(spec, dict):
        assert type(x) is dict and list(x) == list(spec), (where, x)
        for k in spec:
            _check(x[k], spec[k], '%s[%r]' % (where, k))
    elif isinstance(spec, list):
        assert type(x) is list and len(x) == len(spec), (where, x)
        for i, s in enumerate(spec):
            _check(x[i], s, '%s[%d]' % (where, i))
    elif isinstance(spec, tuple):
        assert type(x) is np.ndarray and (x.dtype, x.shape) == spec, (where, type(x), getattr(x, 'dtype', None), np.shape(x), spec)
    else:
        assert type(x) is spec, (where, type(x), spec)


def _info(force, success):
    return {'total_force_on_human': force, 'task_success': success,
            'action_robot_len': int, 'action_human_len': int, 'obs_robot_len': int, 'obs_human_len': int}


def _by_agent(obs, reward, done, info):
    return [obs, {'robot': reward, 'human': reward}, {'robot': done, 'human': done, '__all__': bool}, {'robot': info, 'human': info}]


def _expected(env_id, env, n):
    """{method: spec of its return value, or RuntimeError}"""
    task = next(t for t in ('Feeding', 'ScratchItch', 'BedBathing', 'Dressing', 'Drinking') if env_id.startswith(t))
    coop = 'Human' in env_id
    one = n == 1
    per_env = lambda dtype, *shape: (dtype, (() if one else (n,)) + shape)
    vec = lambda dtype: (dtype, (n,))
    robot_obs = per_env(F64, env.obs_robot_len)
    obs = {'robot': robot_obs, 'human': per_env(F64, env.obs_human_len)} if coop else robot_obs
    if task in ('Feeding', 'ScratchItch'):        # NumPy scalars and info as it is
        ref = [obs, np.float64 if one else vec(F64), np.bool_ if one else vec(BOOL), _info(vec(F64), vec(I64))]
    else:                                         # a float, a bool and env 0's info when n_envs == 1
        ref = [obs, float if one else vec(F64), bool if one else vec(BOOL), _info(np.float64 if one else vec(F64), np.int64 if one else vec(I64))]
    if task == 'Drinking':
        return {'reset': obs, 'step': ref, 'step_fused': ref}
    if coop:
        fused = _by_agent(obs, np.float64 if one else vec(F64), np.bool_ if one else vec(BOOL), _info(vec(F64), vec(I64)))
        return {'reset': obs, 'step': _by_agent(*ref), 'step_fused': fused, 'step_reference_api': ref}
    if task == 'Feeding':
        info = _info(float, int) if one else [_info(float, int)] * n
    else:
        info = _info(np.float32, np.int64) if one else _info(vec(F32), vec(I64))
    step = [per_env(F32, env.obs_robot_len), float if one else vec(F32), bool if one else vec(BOOL), info]
    return {'reset': obs, 'step': step, 'step_fused': RuntimeError, 'step_reference_api': ref}


@pytest.mark.parametrize('n', [1, 2])
@pytest.mark.parametrize('env_id', list(envs.ENV_REGISTRY))
def test_env_step_surface(emu_lib, env_id, n):
    env = envs.make(env_id, n_envs=n, **({'toc_attempts': 6} if env_id.startswith('Dressing') else {}))
    env._sim_lib = emu_lib
    expected = _expected(env_id, env, n)
    assert sorted(m for m in ('step_fused', 'step_reference_api') if hasattr(env, m)) == sorted(set(expected) - {'reset', 'step'})
    _check(env.reset(), expected['reset'], 'reset')
    rng = np.random.default_rng(0)
    for name in ('step', 'step_fused', 'step_reference_api'):
        if name not in expected:
            continue
        a = rng.uniform(-1, 1, size=(n, env.action_space.shape[0])).astype(np.float32)
        if env.human.controllable and name != 'step_reference_api':
            a = {'robot': a[:, :env.action_robot_len], 'human': a[:, env.action_robot_len:]}
        if expected[name] is RuntimeError:
            with pytest.raises(RuntimeError):
                getattr(env, name)(a)
        else:
            out = getattr(env, name)(a)
            assert type(out) is tuple, (name, type(out))
            _check(list(out), expected[name], name)
    env.close()
