"""`make()` with the reference's signature (openrl/envs/common/registration.py:35-182).

Ids with a CUDA step function (CartPole-v1, GridWorldEnv, simple_spread) return a `DeviceVecEnv`.  Every other id is
served the reference's way — per-env thunks from the user's `make_custom_envs` hook (registration.py:64-67) or from
`gymnasium.make` when gymnasium is installed — stepped on the host by `SyncHostVecEnv` (sync_venv.py semantics) and
wrapped in `HostVecEnv`, whose pinned staging feeds the device policy / buffer / GAE / update (BASELINE configs[4])."""
from typing import Callable, Optional

from .. import _kinds
from ..vec_env.device_venv import DeviceVecEnv


def _gymnasium_thunks(id, env_num, render_mode, **kwargs):
    try:
        import gymnasium
    except ImportError as e:
        raise NotImplementedError(
            f"env id {id!r} has no device-resident step function (device ids: {sorted(_kinds.ENV_SPECS)}) and gymnasium is not "
            f"installed: pass make_custom_envs=<fn(id, env_num, render_mode, **kw) -> list of env thunks> (registration.py:64-67)") from e
    return [(lambda: gymnasium.make(id, render_mode=render_mode, **kwargs)) for _ in range(env_num)]


def make(id: str, env_num: int = 1, asynchronous: bool = False, add_monitor: bool = True, render_mode=None,
         make_custom_envs: Optional[Callable] = None, auto_reset: bool = True, device="cuda:0", **kwargs):
    if id in _kinds.ENV_SPECS and make_custom_envs is None:
        if not auto_reset:
            raise NotImplementedError("auto_reset=False is not supported by the device vec-env")
        return DeviceVecEnv(id, env_num, device=device, **kwargs)
    from ..vec_env.host_sync import SyncHostVecEnv
    from ..vec_env.host_venv import HostVecEnv

    if make_custom_envs is not None:
        env_fns = make_custom_envs(id=id, env_num=env_num, render_mode=render_mode, **kwargs)
    else:
        env_fns = _gymnasium_thunks(id, env_num, render_mode, **kwargs)
    # `asynchronous` selects the reference's AsyncVectorEnv (one process per env); the host stepping here is synchronous —
    # the overlap with the device comes from HostVecEnv's double-buffered staging, not from worker processes
    # the reference's make receives cfg in kwargs (registration.py:45); either wide-observation option (feed-forward or
    # GRU nets) lets Dict entries be 65..256 wide, and each network checks the option of its own kind
    cfg = kwargs.get("cfg")
    wide = cfg is not None and bool(getattr(cfg, "use_wide_observations", False) or getattr(cfg, "use_wide_recurrent_observations", False))
    return HostVecEnv(SyncHostVecEnv(env_fns, auto_reset=auto_reset, env_name=id), device=device, wide_observations=wide)
