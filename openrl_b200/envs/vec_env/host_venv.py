"""Host-stepped vec-env adapter (SURVEY.md §8f-4, BASELINE config 5): the env.step stays on the
host (MuJoCo-class simulators, the reference's own SyncVectorEnv/AsyncVectorEnv, ...) while the
policy forward, buffer, GAE and update run on the device.

Wraps any object with the reference's BaseVecEnv duck type — `reset(seed=) -> obs | (obs, infos)`,
`step(actions) -> (obs (N,A,d), rewards (N,A,1), dones (N,A), infos)`, `parallel_env_num`,
`agent_num`, `observation_space`, `action_space` — and adds pinned staging buffers so that each step
costs one D2H copy (actions) and one H2D copy (obs, rewards, dones and, for Discrete actions, the legal-move masks the
envs report in `info["action_masks"]`).  `kind = ORL_ENV_NONE` tells
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


class HostVecEnv:
    def __init__(self, env, device="cuda:0"):
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
        N, A = self.parallel_env_num, self.agent_num
        if not hasattr(self.observation_space, "shape") or self.observation_space.shape is None:
            raise NotImplementedError("HostVecEnv stages flat Box observations; Dict observation spaces are not supported")
        d = self.observation_space.shape[0]
        self.obs_dim = d
        self._discrete = hasattr(self.action_space, "n")
        # masks of Box action spaces are ignored, like the reference's buffer (replay_data.py:148-159)
        self.n_mask = int(self.action_space.n) if self._discrete else 0
        self._stage = torch.empty(N * A * (d + 2 + self.n_mask), dtype=torch.float32, pin_memory=torch.cuda.is_available())

    def reset(self, seed=None, options=None):
        out = self.env.reset(seed=seed) if seed is not None else self.env.reset()
        if isinstance(out, tuple):
            return out
        return out, [{} for _ in range(self.parallel_env_num)]

    def reset_into(self, obs_out, critic_obs_out=None, action_masks_out=None):
        """Slot 0 of the buffer from env.reset(): the observations and, when every env's reset info carries
        `action_masks` and `action_masks_out` is given, the masks (init_buffer, replay_data.py:286-298).  Returns whether
        masks were written."""
        obs, infos = self.reset()
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
        """Write one step into the pinned block [obs | rewards | dones (| masks)]; returns the floats to upload and
        whether masks were staged."""
        B, d = n_envs * self.agent_num, self.obs_dim
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

    def step_staged(self, actions_dev):
        """actions (B, w) device tensor -> host env.step -> the device block [obs | rewards | dones (| masks)] (one pinned
        H2D copy, the layout orl_host_insert reads) plus the host-side step outputs and whether the block carries the
        envs' action masks (every env's info has `action_masks`): a 6-tuple (dev, obs, rewards, dones, infos, has_masks)."""
        N, A = self.parallel_env_num, self.agent_num
        a = actions_dev.cpu().numpy().reshape(N, A, -1)          # D2H (synchronises the stream)
        self.d2h_bytes += a.nbytes
        if self._discrete:                                       # the reference hands integer indices to env.step
            a = a.astype(np.int64)
        obs, rewards, dones, infos = self.env.step(a)
        n, has_masks = self._stage_step(self._stage.numpy(), obs, rewards, dones, infos, N)
        dev = self._stage[:n].to(self.device, non_blocking=True)      # one H2D copy
        self.h2d_bytes += n * 4
        return dev, obs, rewards, dones, infos, has_masks

    # -- two-group ping-pong (double-buffered ingest) ---------------------------------------------
    @property
    def supports_groups(self):
        """True when the wrapped vec-env can step a sub-range of its envs (`step_range(lo, hi, actions)`)."""
        return hasattr(self.env, "step_range") and self.parallel_env_num >= 2

    def group_bounds(self, n_groups=2):
        N = self.parallel_env_num
        cuts = [N * g // n_groups for g in range(n_groups + 1)]
        return [(cuts[g], cuts[g + 1]) for g in range(n_groups)]

    def _group_stage(self, g, lo, hi):
        key = (g, lo, hi)
        if getattr(self, "_gstages", None) is None:
            self._gstages = {}
        if key not in self._gstages:
            n, A, w = hi - lo, self.agent_num, self.obs_dim + 2 + self.n_mask
            pin = torch.cuda.is_available()
            self._gstages[key] = dict(
                inp=torch.empty(n * A * w, dtype=torch.float32, pin_memory=pin),     # obs | rewards | dones (| masks)
                act=None, dev=torch.empty(n * A * w, dtype=torch.float32, device=self.device),
                ev=torch.cuda.Event() if pin else None)
        return self._gstages[key]

    def group_fetch_actions(self, g, lo, hi, actions_dev):
        """Enqueue the D2H copy of this group's actions into its pinned buffer and mark it with an event."""
        st = self._group_stage(g, lo, hi)
        if st["act"] is None or st["act"].shape != actions_dev.shape:
            st["act"] = torch.empty(actions_dev.shape, dtype=torch.float32, pin_memory=torch.cuda.is_available())
        st["act"].copy_(actions_dev, non_blocking=True)
        if st["ev"] is not None:
            st["ev"].record()
        self.d2h_bytes += actions_dev.numel() * 4

    def group_step(self, g, lo, hi):
        """Wait for the group's actions, step its envs on the host, stage the results in pinned memory and enqueue ONE
        H2D copy; returns the device block [obs | rewards | dones (| masks)] (the layout orl_host_insert reads) plus the
        host-side step outputs and whether the block carries masks (every env of the group reported them): a 6-tuple
        (dev, obs, rewards, dones, infos, has_masks)."""
        st = self._group_stage(g, lo, hi)
        if st["ev"] is not None:
            st["ev"].synchronize()
        n_envs, A = hi - lo, self.agent_num
        a = st["act"].numpy().reshape(n_envs, A, -1)
        if self._discrete:
            a = a.astype(np.int64)
        obs, rewards, dones, infos = self.env.step_range(lo, hi, a)
        n, has_masks = self._stage_step(st["inp"].numpy(), obs, rewards, dones, infos, n_envs)
        st["dev"][:n].copy_(st["inp"][:n], non_blocking=True)
        self.h2d_bytes += n * 4
        return st["dev"], obs, rewards, dones, infos, has_masks

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
