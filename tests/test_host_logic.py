"""Host-side pieces that need no GPU: config parser (flag names / defaults of the reference,
openrl/configs/config.py), spaces, callback plumbing, make() dispatch, loud failure without the library."""
import numpy as np
import pytest


def test_config_defaults_match_reference_table():
    from openrl_b200.configs.config import create_config_parser

    cfg = create_config_parser().parse_args([])
    # SURVEY.md §5.6 (file:line of each default in the reference)
    want = dict(seed=0, episode_length=200, hidden_size=64, layer_N=1, activation_id=1, use_popart=False, use_valuenorm=True,
                use_feature_normalization=False, use_orthogonal=True, gain=0.01, use_recurrent_policy=False, recurrent_N=1,
                data_chunk_length=2, lr=5e-4, critic_lr=5e-4, opti_eps=1e-5, weight_decay=0, ppo_epoch=10,
                use_clipped_value_loss=True, clip_param=0.2, num_mini_batch=1, entropy_coef=0.01, value_loss_coef=0.5,
                max_grad_norm=10, use_gae=True, gamma=0.99, gae_lambda=0.95, use_proper_time_limits=False,
                use_huber_loss=True, huber_delta=10, use_value_active_masks=True, use_policy_active_masks=True,
                use_adv_normalize=False, use_linear_lr_decay=False, log_interval=5, use_share_model=False)
    for k, v in want.items():
        assert getattr(cfg, k) == v, k


def test_config_flags_and_yaml(tmp_path):
    from openrl_b200.configs.config import create_config_parser

    y = tmp_path / "c.yaml"
    y.write_text("globals:\n  L: 25\nepisode_length: {{ L }}\nlr: 7e-4\nuse_adv_normalize: true\n")
    cfg = create_config_parser().parse_args(["--config", str(y), "--ppo_epoch", "4", "--use_valuenorm", "false"])
    assert (cfg.episode_length, cfg.lr, cfg.use_adv_normalize, cfg.ppo_epoch, cfg.use_valuenorm) == (25, 7e-4, True, 4, False)
    cfg.num_agents = 3  # components write to cfg (ppo_net.py:69-81)
    assert "num_agents" in cfg


def test_spaces():
    from openrl_b200 import spaces

    b = spaces.Box(-1, 1, (3,), np.float32)
    assert b.shape == (3,) and b.contains(b.sample()) and b.__class__.__name__ == "Box"
    d = spaces.Discrete(5)
    assert d.n == 5 and d.contains(d.sample()) and d.sample(mask=np.array([0, 0, 1, 0, 0])) == 2
    di = spaces.Dict({"policy": b, "critic": spaces.Box(-1, 1, (9,), np.float32)})
    assert di["critic"].shape == (9,) and di.__class__.__name__ == "Dict"


def test_callback_list_contract():
    from openrl_b200.utils.callbacks import BaseCallback, CallbackList, StopTrainingOnMaxSteps

    class Agent:
        num_time_steps = 0

    class Count(BaseCallback):
        needs_per_step = False

        def _on_step(self):
            return True

    ag = Agent()
    cl = CallbackList([Count(), StopTrainingOnMaxSteps(3)])
    cl.init_callback(ag)
    assert cl.needs_per_step  # one member needs per-step locals -> the driver must not fuse the rollout
    cl.on_training_start({}, {})
    res = []
    for _ in range(4):
        ag.num_time_steps += 8
        cl.update_locals({"obs": 1})
        res.append(cl.on_step())
    assert res == [True, True, False, False]
    assert CallbackList([Count()]).needs_per_step is False


def test_make_rejects_unknown_ids():
    from openrl_b200.envs.common import make

    with pytest.raises(NotImplementedError):
        make("HalfCheetah-v4", env_num=2)


def test_missing_library_fails_loudly(tmp_path):
    from openrl_b200 import lib

    with pytest.raises(lib.OrlLibraryError):
        lib.load(str(tmp_path / "nope.so"))


def test_opponent_pool_records_the_snapshots_activation():
    """The vec-env step API evaluates the pool with the activation its snapshots were trained with; one pool holds one."""
    import torch

    from openrl_b200.selfplay import OpponentPool

    pool = OpponentPool(2, 10, device="cpu")
    assert pool.activation_id == 1
    for k in range(3):
        pool.add(torch.full((10,), float(k)), activation_id=0)
    assert pool.activation_id == 0 and pool.count == 3 and pool.params[0, 0] == 2.0
    with pytest.raises(ValueError, match="activation_id"):
        pool.add(torch.zeros(10), activation_id=3)
    assert pool.count == 3


def test_cpu_device_is_refused():
    """There is no CPU fallback: PPONet refuses non-CUDA devices before touching any kernel."""
    from openrl_b200 import spaces
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet

    class Env:
        agent_num, parallel_env_num = 1, 2
        observation_space, action_space = spaces.Box(-1, 1, (4,), np.float32), spaces.Discrete(2)

        def reset(self, seed=None):
            return np.zeros((2, 1, 4), np.float32)

    with pytest.raises(RuntimeError, match="CUDA only"):
        PPONet(Env(), cfg=create_config_parser().parse_args([]), device="cpu")


def test_chunk_row_indices_follow_the_reference_cast():
    """Chunks of the recurrent generator address the (T, B) device buffer exactly like the reference's
    agent-major / time-minor `_cast` flattening (buffers/utils/util.py:96-97), including chunks that straddle rows."""
    import torch

    from openrl_b200.buffers.replay_data import chunk_row_indices
    from oracle.loop_ma import _cast

    T, N, A, L = 25, 4, 3, 2
    B = N * A
    x = np.arange(T * B, dtype=np.int64).reshape(T, N, A, 1)   # value = its own buffer row index t*B + row
    flat = _cast(x)[:, 0]                                       # reference order of the samples
    chunks = (T * B) // L
    ids = torch.randperm(chunks)
    got = chunk_row_indices(ids, L, T, B).numpy().reshape(chunks, L)
    want = np.stack([flat[c * L:c * L + L] for c in ids.numpy()])
    assert np.array_equal(got, want)
    assert any((w // 1)[0] % B != (w // 1)[1] % B for w in want)   # some chunks straddle two rows (T odd, L = 2)
