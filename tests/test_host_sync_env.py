"""Host vec-env semantics of `make()` for ids without a device step function (reference:
openrl/envs/common/registration.py:35-182, vec_env/sync_venv.py:129-247, base_venv.py:231-302; the reference's own
checks: tests/test_env/test_sync_env.py)."""
import numpy as np
import pytest

from helpers import CountEnv
from openrl_b200.envs.vec_env.host_sync import SyncHostVecEnv


def test_sync_host_vec_env_matches_reference_semantics():
    v = SyncHostVecEnv([(lambda i=i: CountEnv(i)) for i in range(4)])
    obs, infos = v.reset(seed=7)
    assert obs.shape == (4, 1, 2) and len(infos) == 4
    assert [e.seed_seen for e in v.envs] == [7 + i * 10086 for i in range(4)]       # sync_venv.py:137
    for t in range(1, 3):
        obs, rew, done, infos = v.step(np.full((4, 1, 1), 2))
        assert obs.shape == (4, 1, 2) and rew.shape == (4, 1, 1) and done.shape == (4, 1) and rew.dtype == np.float64
        assert not done.any() and (obs[:, 0, 0] == t).all() and (rew == 2).all()
    obs, rew, done, infos = v.step(np.zeros((4, 1, 1)))
    assert done.all() and (obs[:, 0, 0] == 0).all()                                 # auto-reset: the reset observation comes back
    assert all("final_observation" in i and i["final_observation"][0] == 3 and i["final_info"] == {"t": 3} for i in infos)
    # call / get_attr / set_attr / exec_func (base_venv.py:231-302)
    assert v.call("tag") == ["x"] * 4
    v.set_attr("tag", ["a", "b", "c", "d"])
    assert v.get_attr("tag") == ["a", "b", "c", "d"]
    with pytest.raises(ValueError):
        v.set_attr("tag", [1, 2])
    assert v.exec_func(lambda e: e.ident * 10, indices=[1, 3]) == [10, 30]
    v.close()
    assert v.closed


def test_make_defers_to_custom_host_envs(monkeypatch):
    """make(id, make_custom_envs=...) builds host thunks (registration.py:64-67) behind the HostVecEnv staging adapter."""
    import torch

    from openrl_b200.envs.common import make
    from openrl_b200.envs.vec_env import HostVecEnv

    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)    # pinned staging falls back to pageable memory on a CPU box
    seen = {}

    def custom(id, env_num, render_mode=None, **kw):
        seen.update(id=id, env_num=env_num, kw=kw)
        return [(lambda i=i: CountEnv(i)) for i in range(env_num)]

    env = make("MyHostEnv-v0", env_num=3, make_custom_envs=custom, device="cpu", flavour="plain")
    assert isinstance(env, HostVecEnv) and env.parallel_env_num == 3 and env.agent_num == 1 and env.env_name == "MyHostEnv-v0"
    assert seen == {"id": "MyHostEnv-v0", "env_num": 3, "kw": {"flavour": "plain"}}
    obs, infos = env.reset(seed=1)
    assert obs.shape == (3, 1, 2)
    o, r, d, i = env.step(np.ones((3, 1, 1)))
    assert o.shape == (3, 1, 2) and r.shape == (3, 1, 1) and d.shape == (3, 1)
    assert env.call("ident") == [0, 1, 2]
    with pytest.raises(NotImplementedError, match="make_custom_envs"):
        make("Unknown-v0", env_num=1, device="cpu")
