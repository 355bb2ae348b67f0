"""Host-side synchronous vector env over per-env thunks (reference: SyncVectorEnv,
openrl/envs/vec_env/sync_venv.py:129-247, with the single-agent wrapping of
envs/wrappers/multiagent_wrapper.py:33-79): steps N Python envs in a loop and returns the
reference's batched 4-tuple — obs (N, A, d) (a dict of such arrays for Dict observations), rewards (N, A, 1),
dones (N, A), infos (list of N dicts) — auto-resetting finished envs with `final_observation` / `final_info` stashed in the info
(sync_venv.py:213-218).  This is the env side of host-stepped workloads (MuJoCo-class simulators,
BASELINE configs[4]); `HostVecEnv` adds the pinned staging that feeds the device path.

Sub-envs may follow the gymnasium API (`reset(seed=) -> (obs, info)`, `step -> (obs, r, terminated,
truncated, info)`) or the 4-tuple API (`step -> (obs, r, done, info)`); seeds are `seed + i * 10086`
like the reference (sync_venv.py:137)."""
from copy import deepcopy

import numpy as np


class SyncHostVecEnv:
    def __init__(self, env_fns, auto_reset=True, env_name=None):
        self.envs = [fn() for fn in env_fns]
        self.parallel_env_num = len(self.envs)
        self.auto_reset = auto_reset
        e0 = self.envs[0]
        self.agent_num = int(getattr(e0, "agent_num", 1))
        self.observation_space = e0.observation_space
        self.action_space = e0.action_space
        self.env_name = env_name or type(e0).__name__
        self.use_monitor = False
        self.closed = False

    # -- reference surface -------------------------------------------------------------------
    def _obs(self, obs_list):
        """Stack the envs' observations to float32 (N, A, d); Dict observations (`{"policy": ..., "critic": ...}`, each
        (d,) for a single agent or (A, d)) stack per key, as the reference's concatenate of a Dict space does."""
        if isinstance(obs_list[0], dict):
            return {k: self._obs([x[k] for x in obs_list]) for k in obs_list[0]}
        o = np.stack([np.asarray(x, dtype=np.float32) for x in obs_list])
        return o.reshape(len(obs_list), self.agent_num, -1)

    def reset(self, seed=None, options=None):
        obs, infos = [], []
        for i, env in enumerate(self.envs):
            kw = {} if seed is None else {"seed": seed + i * 10086}
            out = env.reset(**kw)
            if isinstance(out, tuple) and len(out) == 2 and isinstance(out[1], dict):
                o, info = out
            else:
                o, info = out, {}
            obs.append(o)
            infos.append(info)
        return self._obs(obs), infos

    def step(self, actions, extra_data=None):
        return self.step_range(0, self.parallel_env_num, actions)

    def step_range(self, lo, hi, actions):
        """Step envs [lo, hi) only (`actions` holds their hi - lo actions): lets `HostVecEnv` ping-pong two env groups so
        that the device works on one group while the host steps the other."""
        N, A = hi - lo, self.agent_num
        rewards = np.zeros((N, A, 1), np.float64)
        dones = np.zeros((N, A), bool)
        obs, infos = [], []
        for i, env in enumerate(self.envs[lo:hi]):
            a = np.asarray(actions[i])
            if A == 1:
                a = a.reshape(-1)
                a = a[0] if (hasattr(self.action_space, "n") or a.size == 1 and getattr(self.action_space, "shape", (1,)) == ()) else a
            ret = env.step(a)
            if len(ret) == 5:
                o, r, term, trunc, info = ret
                done = np.logical_or(term, trunc)
            elif len(ret) == 4:
                o, r, done, info = ret
            else:
                raise NotImplementedError(f"Not support step return length: {len(ret)}")
            rewards[i] = np.asarray(r, dtype=np.float64).reshape(A, 1)
            dones[i] = np.asarray(done, dtype=bool).reshape(-1)
            if self.auto_reset and dones[i].all():
                old_o, old_info = o, info
                out = env.reset()
                o, info = out if (isinstance(out, tuple) and len(out) == 2 and isinstance(out[1], dict)) else (out, {})
                info = deepcopy(info)
                info["final_observation"] = old_o
                info["final_info"] = old_info
            obs.append(o)
            infos.append(info)
        return self._obs(obs), rewards, dones, infos

    def random_action(self, infos=None):
        return np.array([[self.action_space.sample() for _ in range(self.agent_num)] for _ in range(self.parallel_env_num)])

    # call / exec_func / set_attr: base_venv.py:231-302
    def call(self, name, *args, **kwargs):
        out = []
        for env in self.envs:
            f = getattr(env, name)
            out.append(f(*args, **kwargs) if callable(f) else f)
        return out

    def get_attr(self, name):
        return self.call(name)

    def set_attr(self, name, values):
        if not isinstance(values, (list, tuple)):
            values = [values for _ in range(self.parallel_env_num)]
        if len(values) != self.parallel_env_num:
            raise ValueError(f"Values must be a list or tuple with length equal to the number of environments. "
                             f"Got `{len(values)}` values for {self.parallel_env_num} environments.")
        for env, v in zip(self.envs, values):
            setattr(env, name, v)

    def exec_func(self, func, indices=None, *args, **kwargs):
        idx = range(self.parallel_env_num) if indices is None else indices
        return [func(self.envs[i], *args, **kwargs) for i in idx]

    def close(self):
        for env in self.envs:
            if hasattr(env, "close"):
                env.close()
        self.closed = True
