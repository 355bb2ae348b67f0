"""PPOAgent(net).train(total_time_steps) / act / save / load
(reference: openrl/runners/common/ppo_agent.py:39-158, rl_agent.py:35-216, base_agent.py:31)."""
import io
import pathlib

import numpy as np
import torch

from ...algorithms.ppo import PPOAlgorithm
from ...buffers import NormalReplayBuffer
from ...drivers.onpolicy_driver import OnPolicyDriver
from ...envs.vec_env.host_venv import prepare_action_masks
from ...utils.callbacks import BaseCallback, CallbackList
from ...utils.logger import Logger
from ... import lib


class PPOAgent:
    def __init__(self, net, env=None, run_dir=None, env_num=None, rank=0, world_size=1, use_wandb=False,
                 use_tensorboard=False, project_name="PPOAgent"):
        self.net = net
        self._cfg = net.cfg
        self._use_wandb, self._use_tensorboard = use_wandb, use_tensorboard
        self.project_name = project_name
        self._env = env if env is not None else net.env
        self.net.reset()
        self._cfg.n_rollout_threads = self._env.parallel_env_num if env_num is None else env_num
        self._cfg.learner_n_rollout_threads = self._cfg.n_rollout_threads
        self.env_num = self._cfg.n_rollout_threads
        self.run_dir = run_dir
        self.rank, self.world_size = rank, world_size
        self.client = None
        self.agent_num = self._env.agent_num
        self.num_time_steps = 0
        self._episode_num = 0
        self._total_time_steps = 0
        self.driver = None

    def train(self, total_time_steps, callback=None, train_algo_class=PPOAlgorithm, logger=None,
              driver_class=OnPolicyDriver):
        self._cfg.num_env_steps = total_time_steps
        self._total_time_steps = total_time_steps
        self.config = {"cfg": self._cfg, "num_agents": self.agent_num, "run_dir": self.run_dir, "envs": self._env,
                       "device": self.net.device}
        # device objects (scratch, rollout buffer) are kept across train() calls while the shapes
        # and classes are unchanged: a second call starts without allocations
        key = (train_algo_class, driver_class, self._cfg.episode_length, self._cfg.n_rollout_threads, self.agent_num,
               id(self._env), self._cfg.ppo_epoch, self._cfg.num_mini_batch)
        if self.driver is not None and getattr(self, "_driver_key", None) == key:
            trainer, buffer = self.driver.trainer, self.driver.buffer
        else:
            trainer = train_algo_class(cfg=self._cfg, init_module=self.net.module, device=self.net.device,
                                       agent_num=self.agent_num)
            buffer = NormalReplayBuffer(self._cfg, self.agent_num, self._env.observation_space, self._env.action_space,
                                        data_client=None, device=self.net.device)
        self._driver_key = key
        if logger is None:
            logger = Logger(cfg=self._cfg, project_name=self.project_name, quiet=getattr(self._cfg, "quiet", False))
        self._logger = logger
        callback = self._setup_callback(callback)
        prev = self.driver
        driver = driver_class(config=self.config, trainer=trainer, buffer=buffer, agent=self, client=self.client,
                              rank=self.rank, world_size=self.world_size, logger=logger, callback=callback)
        if prev is not None and prev.trainer is trainer:
            driver.rng_counter = prev.rng_counter  # keep the device noise stream moving forward
        self.driver = driver
        if callback is not None:
            callback.on_training_start(locals(), globals())
        driver.run()
        if callback is not None:
            callback.on_training_end()
        logger.close()

    def _setup_callback(self, callback):
        if callback is None:
            return None
        if isinstance(callback, (list, tuple)):
            callback = CallbackList(callback)
        callback.init_callback(self)
        return callback

    def act(self, observation, info=None, deterministic=True, episode_starts=None):
        """ppo_agent.py:134-158: observation (N, A, d) -> actions (N, A, 1) numpy."""
        if isinstance(observation, dict):   # Dict spaces: the actor reads the "policy" entry (policy_network.py:137-139)
            observation = observation["policy"]
        obs = np.asarray(observation, dtype=np.float32)
        N, A = obs.shape[0], obs.shape[1]
        action_masks = prepare_action_masks(info, agent_num=self.agent_num) if info is not None else None
        actions, rnn_state = self.net.act(obs.reshape(N * A, -1), action_masks=action_masks, deterministic=deterministic,
                                          episode_starts=episode_starts)
        out = actions.view(N, A, -1).cpu().numpy()   # np.split(_t2n(action), env_num): (N, A, act_shape)
        if self.net.module.models["policy"].head_kind == lib.HEAD_CATEGORICAL:
            out = out.astype(np.int64)                # Categorical.sample() yields integer indices
        return out, rnn_state

    def get_env(self):
        return self._env

    @property
    def logger(self):
        return getattr(self, "_logger", None)

    def set_env(self, env):
        self.net.reset(env)
        self._env = env
        self.env_num = env.parallel_env_num
        self.agent_num = env.agent_num

    def save(self, path):
        """rl_agent.py:187-191: `torch.save(self.net.module, path / "module.pt")` — the pickled module (models with the
        reference's state_dict names, optimiser state, Adam step counters)."""
        path = pathlib.Path(path)
        path.mkdir(parents=True, exist_ok=True)
        torch.save(self.net.module, path / "module.pt")

    def load(self, path):
        """rl_agent.py:193-213.  Accepts (i) a module pickled by `save`, (ii) a round-1 checkpoint (dict of
        state_dicts), (iii) any pickled object with `.models[k].state_dict()` under the reference's key names (a
        reference `PPOModule`, when its package is importable): (ii) and (iii) are copied into the live module."""
        path = pathlib.Path(path)
        f = path / "module.pt" if path.is_dir() else path
        assert f.exists(), f"{f} does not exist"
        obj = torch.load(f, map_location=self.net.device, weights_only=False)
        m = self.net.module
        if isinstance(obj, type(m)):
            self.net.module = obj
        elif isinstance(obj, dict) and "models" in obj:
            for k, sd in obj["models"].items():
                m.models[k].load_state_dict(sd)
            for k, sd in obj.get("optimizers", {}).items():
                m.optimizers[k].load_state_dict(sd)
            if "adam_steps" in obj:
                m.adam_steps.copy_(obj["adam_steps"])
        elif hasattr(obj, "models"):
            for k, model in obj.models.items():
                m.models[k].load_state_dict({kk: vv.to(self.net.device) for kk, vv in model.state_dict().items()}, strict=False)
        else:
            raise TypeError(f"{f}: unrecognised checkpoint object {type(obj).__name__}")
        self.net.reset()
