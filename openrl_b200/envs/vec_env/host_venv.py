"""Host-stepped vec-env adapter (SURVEY.md §8f-4, BASELINE config 5): the env.step stays on the
host (MuJoCo-class simulators, the reference's own SyncVectorEnv/AsyncVectorEnv, ...) while the
policy forward, buffer, GAE and update run on the device.

Wraps any object with the reference's BaseVecEnv duck type — `reset(seed=) -> obs | (obs, infos)`,
`step(actions) -> (obs (N,A,d), rewards (N,A,1), dones (N,A), infos)`, `parallel_env_num`,
`agent_num`, `observation_space`, `action_space` — and adds pinned staging buffers so that each step
costs one D2H copy (actions) and one H2D copy (obs, rewards, dones and, for Discrete actions, the legal-move masks the
envs report in `info["action_masks"]`).  An env whose observation space is Dict {"policy", "critic"} gives the critic
its own observation (the reference's MAPPO envs: get_policy_obs / get_critic_obs, buffers/utils/util.py:22-55); both
ride in the same copy.  `kind = ORL_ENV_NONE` tells
the driver to run the per-step loop (onpolicy_driver.py:154-203 semantics)."""
import numpy as np
import torch

from ... import lib


def prepare_action_masks(info, agent_num=1):
    """openrl/envs/vec_env/utils/util.py:54-88: per-env `info["action_masks"]` ((n,) for every agent, or (A, n) one row per
    agent) -> int8 (N*A, n); None when any env's info lacks the key (all actions available).  As in the reference the
    values are cast to int8, so an entry in (-1, 1) such as 0.5 masks its action (0 = illegal).  An info that is None
    counts as one without the key (the reference fails on it)."""
    if info is None:
        return None
    rows = []
    for env_info in info:
        if env_info is None or "action_masks" not in env_info:
            return None
        m = np.asarray(env_info["action_masks"])
        if m.ndim not in (1, 2):
            raise ValueError(m.ndim)
        rows.extend(m[a] if m.ndim == 2 else m for a in range(agent_num))
    return np.asarray(rows, dtype=np.int8).reshape(len(rows), -1)


def dict_obs_dims(space, wide_observations=False):
    """(policy width, critic width) of a Dict observation space with exactly the keys "policy" and "critic", each a flat
    Box of width 1..64 (the widths the device networks take), or 1..256 with `wide_observations` (the feed-forward nets
    of cfg.use_wide_observations); NotImplementedError naming the cause otherwise."""
    bound = 256 if wide_observations else 64
    keys = sorted(space.keys())
    if keys != ["critic", "policy"]:
        raise NotImplementedError(f"HostVecEnv stages Dict observation spaces with exactly the keys 'policy' and 'critic'; "
                                  f"this one has {keys}")
    dims = []
    for k in ("policy", "critic"):
        sub = space[k]
        shape = getattr(sub, "shape", None)
        if sub.__class__.__name__ != "Box" or shape is None or len(shape) != 1:
            raise NotImplementedError(f"HostVecEnv stages flat Box entries of a Dict observation space; '{k}' is {sub}")
        if not 1 <= shape[0] <= bound:
            raise NotImplementedError(f"the '{k}' observation has width {shape[0]}; the device networks take widths 1..{bound}"
                                      + ("" if wide_observations else " (1..256 with use_wide_observations)"))
        dims.append(int(shape[0]))
    return tuple(dims)


class HostVecEnv:
    def __init__(self, env, device="cuda:0", wide_observations=False):
        self.env = env
        self.kind = lib.ENV_NONE
        self.device = torch.device(device)
        self.parallel_env_num = env.parallel_env_num
        self.agent_num = env.agent_num
        self.observation_space = env.observation_space
        self.action_space = env.action_space
        self.env_name = getattr(env, "env_name", type(env).__name__)
        self.use_monitor = False
        self.env_table, self.env_table_len = None, 0
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        self.dict_obs = self.observation_space.__class__.__name__ == "Dict"
        if self.dict_obs:
            self.obs_dim, self.critic_obs_dim = dict_obs_dims(self.observation_space, wide_observations)
        else:
            if not hasattr(self.observation_space, "shape") or self.observation_space.shape is None:
                raise NotImplementedError(f"HostVecEnv stages flat Box or Dict {{'policy', 'critic'}} observations; "
                                          f"got {self.observation_space}")
            self.obs_dim = self.critic_obs_dim = self.observation_space.shape[0]
        self._staged_dc = self.critic_obs_dim if self.dict_obs else 0    # width of the block's critic section
        self._discrete = hasattr(self.action_space, "n")
        # masks of Box action spaces are ignored, like the reference's buffer (replay_data.py:148-159)
        self.n_mask = int(self.action_space.n) if self._discrete else 0

    def reset(self, seed=None, options=None):
        out = self.env.reset(seed=seed) if seed is not None else self.env.reset()
        if isinstance(out, tuple):
            return out
        return out, [{} for _ in range(self.parallel_env_num)]

    def reset_into(self, obs_out, critic_obs_out=None, action_masks_out=None):
        """Slot 0 of the buffer from env.reset(): the observations (with Dict observations the "policy" entry, and the
        "critic" entry into `critic_obs_out` when it is given) and, when every env's reset info carries `action_masks` and
        `action_masks_out` is given, the masks (init_buffer, replay_data.py:286-298).  Returns whether masks were written."""
        obs, infos = self.reset()
        if self.dict_obs:
            if critic_obs_out is not None:
                critic_obs_out.copy_(torch.as_tensor(np.asarray(obs["critic"], dtype=np.float32)).view_as(critic_obs_out))
            obs = obs["policy"]
        obs_out.copy_(torch.as_tensor(np.asarray(obs, dtype=np.float32)).view_as(obs_out), non_blocking=False)
        am = self._masks(infos, self.parallel_env_num)
        if am is None or action_masks_out is None:
            return False
        action_masks_out.copy_(torch.from_numpy(am.astype(np.float32)).view_as(action_masks_out), non_blocking=False)
        return True

    def _masks(self, infos, n_envs):
        """(n_envs*A, n) int8 masks of a step's (or a reset's) infos, or None (no Discrete actions, or an env without the
        key)."""
        if not self.n_mask:
            return None
        am = prepare_action_masks(infos, agent_num=self.agent_num)
        if am is not None and am.shape != (n_envs * self.agent_num, self.n_mask):
            raise ValueError(f"info['action_masks'] gives masks of shape {am.shape}; expected "
                             f"{(n_envs * self.agent_num, self.n_mask)} (one row of n = {self.n_mask} per agent)")
        return am

    def _stage_step(self, buf, obs, rewards, dones, infos, n_envs):
        """Write one step into the pinned block [obs (| critic obs) | rewards | dones (| masks)]; returns the floats to
        upload and whether masks were staged."""
        B, d = n_envs * self.agent_num, self.obs_dim + self._staged_dc
        if self.dict_obs:
            buf[:B * self.obs_dim] = np.asarray(obs["policy"], dtype=np.float32).reshape(-1)
            buf[B * self.obs_dim:B * d] = np.asarray(obs["critic"], dtype=np.float32).reshape(-1)
        else:
            buf[:B * d] = np.asarray(obs, dtype=np.float32).reshape(-1)
        buf[B * d:B * d + B] = np.asarray(rewards, dtype=np.float32).reshape(-1)
        buf[B * d + B:B * (d + 2)] = np.asarray(dones, dtype=np.float32).reshape(-1)
        am = self._masks(infos, n_envs)
        if am is None:
            return B * (d + 2), False
        buf[B * (d + 2):B * (d + 2 + self.n_mask)] = am.reshape(-1)
        return B * (d + 2 + self.n_mask), True

    def step(self, actions, extra_data=None):
        return self.env.step(actions)

    # -- staged stepping of an env range: the whole range, or one of the groups of the ping-pong loop ---------------
    @property
    def supports_groups(self):
        """True when the wrapped vec-env can step a sub-range of its envs (`step_range(lo, hi, actions)`)."""
        return hasattr(self.env, "step_range") and self.parallel_env_num >= 2

    def group_bounds(self, n_groups=2):
        N = self.parallel_env_num
        cuts = [N * g // n_groups for g in range(n_groups + 1)]
        return [(cuts[g], cuts[g + 1]) for g in range(n_groups)]

    def _range_stage(self, lo, hi):
        """The staging of envs [lo, hi): pinned action and step buffers, the device block and the actions' event (a
        CPU device copies synchronously and needs neither pinning nor events)."""
        if getattr(self, "_stages", None) is None:
            self._stages = {}
        if (lo, hi) not in self._stages:
            n, A, w = hi - lo, self.agent_num, self.obs_dim + self._staged_dc + 2 + self.n_mask
            cuda = self.device.type == "cuda"
            self._stages[lo, hi] = dict(
                inp=torch.empty(n * A * w, dtype=torch.float32, pin_memory=cuda),     # obs (| critic obs) | rewards | dones (| masks)
                act=None, dev=torch.empty(n * A * w, dtype=torch.float32, device=self.device),
                ev=torch.cuda.Event() if cuda else None)
        return self._stages[lo, hi]

    def fetch_actions(self, lo, hi, actions_dev):
        """Enqueue the D2H copy of the actions (rows, w) of envs [lo, hi) into their pinned buffer and mark it with an
        event."""
        st = self._range_stage(lo, hi)
        if st["act"] is None or st["act"].shape != actions_dev.shape:
            st["act"] = torch.empty(actions_dev.shape, dtype=torch.float32, pin_memory=st["ev"] is not None)
        st["act"].copy_(actions_dev, non_blocking=True)
        if st["ev"] is not None:
            st["ev"].record()
        self.d2h_bytes += actions_dev.numel() * 4

    def step_staged(self, lo, hi):
        """Wait for the actions of envs [lo, hi) (`fetch_actions`), step them on the host (`env.step` for every env,
        `env.step_range` for a sub-range), stage the results in pinned memory and enqueue ONE H2D copy.  Returns the device
        block [obs (| critic obs) | rewards | dones (| masks)] (the layout orl_host_insert reads), the host-side step outputs and whether
        the block carries the envs' action masks (every stepped env's info has `action_masks`): a 6-tuple
        (dev, obs, rewards, dones, infos, has_masks)."""
        st = self._range_stage(lo, hi)
        if st["ev"] is not None:
            st["ev"].synchronize()
        n_envs = hi - lo
        a = st["act"].numpy().reshape(n_envs, self.agent_num, -1)
        if self._discrete:                                       # the reference hands integer indices to env.step
            a = a.astype(np.int64)
        if n_envs == self.parallel_env_num:
            obs, rewards, dones, infos = self.env.step(a)
        else:
            obs, rewards, dones, infos = self.env.step_range(lo, hi, a)
        n, has_masks = self._stage_step(st["inp"].numpy(), obs, rewards, dones, infos, n_envs)
        dev = st["dev"][:n]
        dev.copy_(st["inp"][:n], non_blocking=True)
        self.h2d_bytes += n * 4
        return dev, obs, rewards, dones, infos, has_masks

    def random_action(self, infos=None):
        return np.array([[self.action_space.sample() for _ in range(self.agent_num)] for _ in range(self.parallel_env_num)])

    # call / exec_func / set_attr (base_venv.py:231-302): forwarded to the wrapped host vec-env
    def call(self, name, *args, **kwargs):
        return self.env.call(name, *args, **kwargs)

    def get_attr(self, name):
        return self.env.call(name)

    def set_attr(self, name, values):
        return self.env.set_attr(name, values)

    def exec_func(self, func, indices=None, *args, **kwargs):
        return self.env.exec_func(func, indices, *args, **kwargs)

    def batch_rewards(self, buffer):
        return {}

    def statistics(self, buffer):
        return {}

    def close(self):
        if hasattr(self.env, "close"):
            self.env.close()
