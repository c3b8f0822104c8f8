"""`AssistiveVecEnv` — the batched env as a learner sees it (SURVEY.md §8(b) "fused vector path", §8(f)2).

The reference trains one `gym.Env` per RLlib worker process (`learn.py:26,61-69`); here ONE object steps
`n_envs` environments on one GPU.  `step(actions)` takes and returns torch CUDA tensors: the action tensor's
`data_ptr()` goes straight into the task's fused step (`ag_feeding_step_dev`, `ag_bathing_step_dev`, `ag_dressing_step_dev`,
`ag_scratch_step_dev`, `ag_drinking_step_dev`), observations / rewards / dones are
written into pre-allocated device tensors on the simulation's own stream, and nothing crosses PCIe.  Episodes of
all envs have the same length (200 steps, feeding.py:37), so the batch resets together; `auto_reset` does it inside
`step` the way vector-env wrappers do (the terminal observation is kept in `info['terminal_observation']`).
With numpy inputs the host-buffer entry points are used instead (pinned staging inside the C ABI).

The co-optimisation ids (FeedingJacoHuman-v1, ScratchItchJacoHuman-v1, BedBathingSawyerHuman-v1, DressingPR2Human-v1) run
`ag_coop_step_dev`: actions are {'robot': [N, 7], 'human': [N, k]}, observations {'robot': [N, 25 | 30 | 24 | 24],
'human': [N, 23 | 34 | 28 | 28]}, and rewards, dones and infos
come in the dict shape of the env's `step` (dones with '__all__')."""
import numpy as np


class AssistiveVecEnv:
    def __init__(self, env_id='assistive_gym:FeedingJaco-v1', n_envs=4096, device=0, seed=1001, auto_reset=True, config=None, _lib=None,
                 double_buffer=False, **env_kw):
        """double_buffer: a second copy of the batch is re-randomised by a background thread (the C ABI releases the GIL; its
        kernels run on that copy's own stream) while the first one is stepped; at the end of an episode the two swap, so
        `step` never waits for the 0.5 s of reset orchestration (reference env.py:92-97 rebuilds the world at every reset)."""
        from . import envs
        self.env = envs.make(env_id, n_envs=n_envs, device=device, seed=seed, config=config, **env_kw)
        if _lib is not None:
            self.env._sim_lib = _lib
        self._standby = None
        if double_buffer:
            self._standby = envs.make(env_id, n_envs=n_envs, device=device, seed=seed + 7919, config=config, **env_kw)
            if _lib is not None:
                self._standby._sim_lib = _lib
        self._bg, self._bg_obs, self._bg_err = None, None, None
        self.n_envs, self.device, self.auto_reset = n_envs, device, auto_reset
        self.task = self.env.task
        self.observation_space, self.action_space = self.env.observation_space, self.env.action_space
        self.obs_dim, self.act_dim = self.observation_space.shape[0], self.action_space.shape[0]
        self.coop = self.task in ('feeding', 'scratch_itch', 'bed_bathing', 'dressing') and bool(self.env.human.controllable)
        self._step_dev = None
        self._buf = None

    # ------------------------------------------------------------------ gym-style API
    def _reset_standby(self):
        try:
            self._bg_obs = self._batch_obs(self._standby.reset())
        except Exception as ex:          # surfaced by the next reset()
            self._bg_err = ex

    def _start_standby(self):
        import threading
        self._bg_obs, self._bg_err = None, None
        self._bg = threading.Thread(target=self._reset_standby, daemon=True)
        self._bg.start()

    def reset(self):
        if self._standby is not None and self._bg is not None:
            self._bg.join()
            if self._bg_err is not None:
                raise self._bg_err
            self.env, self._standby = self._standby, self.env          # the freshly reset copy becomes the live one
            obs = self._bg_obs
            self._buf = None                                            # device tensors are bound to a sim's stream
        else:
            obs = self._batch_obs(self.env.reset())
        if self._standby is not None:
            self._start_standby()
        sim = self.env.id
        self._t = 0
        if self.coop:
            self._step_dev, self._step_host = sim.coop_step_dev, sim.coop_step_host
            return obs
        self._step_dev = {'feeding': sim.feeding_step_dev, 'bed_bathing': sim.bathing_step_dev, 'dressing': sim.dressing_step_dev, 'scratch_itch': sim.scratch_step_dev,
                          'drinking': sim.drinking_step_dev}[self.task]
        self._step_host = {'feeding': sim.feeding_step_host, 'bed_bathing': sim.bathing_step_host, 'dressing': sim.dressing_step_host, 'scratch_itch': sim.scratch_step_host,
                           'drinking': sim.drinking_step_host}[self.task]
        return obs

    def _batch_obs(self, obs):
        if isinstance(obs, dict):
            return {k: np.atleast_2d(v) for k, v in obs.items()}
        return np.atleast_2d(obs)

    def _tensors(self, like):
        import torch
        if self._buf is None or self._buf[0].device != like.device:
            n = self.n_envs
            mk = lambda *shape: torch.zeros(shape, device=like.device, dtype=torch.float32)
            if self.coop:
                self._buf = (mk(n, self.env.obs_robot_len), mk(n, self.env.obs_human_len), mk(n), mk(n), mk(n, 4))
            else:
                self._buf = (mk(n, self.obs_dim), mk(n), mk(n), mk(n, 4))
            self._stream = torch.cuda.ExternalStream(self.env.id.stream_ptr(), device=like.device)
        return self._buf

    def step(self, actions):
        """actions: torch CUDA tensor [n_envs, act_dim] (float32, contiguous) -> device tensors, or numpy -> numpy."""
        if self._step_dev is None:
            raise RuntimeError('call reset() first')
        if self.coop:
            return self._step_coop(actions)
        is_torch = hasattr(actions, 'data_ptr')
        if is_torch:
            import torch
            a = actions.to(dtype=torch.float32).contiguous()
            obs, rew, done, info = self._tensors(a)
            # the caller's stream produced `a`; the simulation runs on its own stream
            self._stream.wait_stream(torch.cuda.current_stream(a.device))
            self._step_dev(a.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
            torch.cuda.current_stream(a.device).wait_stream(self._stream)
            out = (obs, rew, done > 0.5, {'total_force_on_human': info[:, 0], 'task_success': info[:, 1]})
            finished = None     # decided from the step counter: no device read-back
        else:
            obs, rew, done, info = self._step_host(np.asarray(actions, dtype=np.float32).reshape(self.n_envs, -1))
            out = (obs, rew, done > 0.5, {'total_force_on_human': info[:, 0], 'task_success': info[:, 1]})
        self._t += 1
        self.env.iteration = self._t
        if self.auto_reset and self._t >= 200:
            term = out[0].clone() if is_torch else out[0].copy()
            new_obs = self.reset()
            if is_torch:
                import torch
                new_obs = torch.as_tensor(new_obs, device=out[0].device, dtype=torch.float32)
            out = (new_obs, out[1], out[2], dict(out[3], terminal_observation=term))
        return out

    def _step_coop(self, actions):
        """actions {'robot': [n, 7], 'human': [n, k]}: torch CUDA tensors -> device tensors, or numpy -> numpy"""
        is_torch = hasattr(actions['robot'], 'data_ptr')
        if is_torch:
            import torch
            a = torch.cat([actions['robot'].to(dtype=torch.float32), actions['human'].to(dtype=torch.float32)], dim=1).contiguous()
            obs_r, obs_h, rew, done, info = self._tensors(a)
            self._stream.wait_stream(torch.cuda.current_stream(a.device))
            self._step_dev(a.data_ptr(), obs_r.data_ptr(), obs_h.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
            torch.cuda.current_stream(a.device).wait_stream(self._stream)
        else:
            a = np.concatenate([np.asarray(actions['robot'], dtype=np.float32).reshape(self.n_envs, -1),
                                np.asarray(actions['human'], dtype=np.float32).reshape(self.n_envs, -1)], axis=1)
            obs_r, obs_h, rew, done, info = self._step_host(a)
        self._t += 1
        self.env.iteration = self._t
        d = done > 0.5
        inf = {'total_force_on_human': info[:, 0], 'task_success': info[:, 1]}
        obs = {'robot': obs_r, 'human': obs_h}
        dones = {'robot': d, 'human': d, '__all__': self._t >= 200}       # every env's episode ends at step 200 (feeding.py:37)
        infos = {'robot': inf, 'human': dict(inf)}
        if self.auto_reset and self._t >= 200:
            term = {k: (v.clone() if is_torch else v.copy()) for k, v in obs.items()}
            new_obs = self.reset()
            if is_torch:
                import torch
                new_obs = {k: torch.as_tensor(v, device=obs_r.device, dtype=torch.float32) for k, v in new_obs.items()}
            obs = new_obs
            infos = {k: dict(v, terminal_observation=term[k]) for k, v in infos.items()}
        return obs, {'robot': rew, 'human': rew}, dones, infos

    def close(self):
        if self._bg is not None:
            self._bg.join()
        self.env.close()
        if self._standby is not None:
            self._standby.close()


class AssistiveRLlibVectorEnv:
    """The batched backend behind the interface RLlib's `VectorEnv` asks of a vectorised env (`vector_reset`, `reset_at`,
    `vector_step`, `get_sub_environments`; reference learn.py:41,61-69 hands RLlib one `gym.Env` per worker -- with this
    adapter one worker owns `n_envs` lock-step envs on its GPU).  RLlib itself is not a dependency: the class is duck-typed,
    `ray.rllib.env.VectorEnv.register` / `to_base_env` accept it where RLlib is installed.

    Episodes of all envs end together (200 steps, feeding.py:37): the first `reset_at` after the batch is done re-randomises
    the whole batch, the following `reset_at(i)` calls of the same round read row i of that reset."""

    def __init__(self, env_id='assistive_gym:FeedingJaco-v1', n_envs=64, device=0, seed=1001, config=None, _lib=None, **env_kw):
        self.vec = AssistiveVecEnv(env_id, n_envs=n_envs, device=device, seed=seed, auto_reset=False, config=config, _lib=_lib, **env_kw)
        self.num_envs = n_envs
        self.observation_space, self.action_space = self.vec.observation_space, self.vec.action_space
        self._obs = None
        self._fresh = np.zeros(n_envs, dtype=bool)

    def vector_reset(self):
        self._obs = self.vec.reset()
        self._fresh[:] = False
        return [self._obs[i] for i in range(self.num_envs)]

    def reset_at(self, index=None):
        index = 0 if index is None else int(index)
        if self._obs is None or self._fresh[index] or self.vec._t >= 200:
            self._obs = self.vec.reset()
            self._fresh[:] = False
        self._fresh[index] = True
        return self._obs[index]

    def vector_step(self, actions):
        obs, rew, done, info = self.vec.step(np.asarray(actions, dtype=np.float32).reshape(self.num_envs, -1))
        self._obs = obs
        self._fresh[:] = False
        infos = [{k: (v[i].item() if hasattr(v[i], 'item') else v[i]) for k, v in info.items()} for i in range(self.num_envs)]
        over = self.vec._t >= 200               # the env's own counter says the same (feeding.py:37); this one survives a replayed state
        return [obs[i] for i in range(self.num_envs)], [float(r) for r in rew], [bool(d) or over for d in done], infos

    def get_sub_environments(self):
        return []        # there are no per-env Python objects: the sub-environments are lanes of one simulation

    def try_render_at(self, index=None):
        return None
