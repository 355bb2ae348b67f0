"""Save what K = 3 device iterations leave behind on every PPO update path, and compare two such saves.

    python tools/update_outputs.py --out DIR            # needs a GPU; about a minute
    python tools/update_outputs.py --compare DIR_A DIR_B

`bench.py --dump-outputs` covers the C2 tensor-core update only.  This tool runs, from the seed, each update kernel
family and each rollout kernel at a small shape: C2 on tensor cores, on FFMA, with the shared model and with dual clip /
plain MSE value loss; C2's flags on GridWorldEnv (rollout_tc_kernel) and with a GRU policy; C4 (GridWorld self-play,
5 actions); C3 GRU, C3 JRPO and C3 with MLP nets (the simple_spread FFMA rollout); C5 (Gaussian head, host-stepped
synthetic env); and host-stepped synthetic envs of wide shapes: SMAC 8m's (8 agents, Dict observations of 80 policy and
168 critic features, Discrete(14) with env-reported masks) with GRU and with MLP nets, and Box(256) observations with
Discrete(64) and GRU nets (the one-row-per-warp GRU act and update).  Per path it saves the policy and critic (or shared model) `flat_params`, their Adam moment buffers,
`adam_steps`, the ValueNorm state, `train_info` and the rollout buffer the last iteration leaves (`buffer_<name>`) as
DIR/<path>/<name>.npy.  `--compare` prints the largest distance in units in the last place per array, so a refactor
that must not change results can be checked bit for bit (distance 0) against its parent commit.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

K = 3
ENVS = 64
PATHS = {
    "c2_tc": ("c2", []),
    "c2_ffma": ("c2", ["--use_tensor_cores", "false"]),
    "c2_share": ("c2", ["--use_share_model", "true"]),
    "c2_dualclip_mse": ("c2", ["--dual_clip_ppo", "true", "--use_huber_loss", "false", "--use_clipped_value_loss", "false"]),
    "c2_gridworld": ("gridworld", []),
    "c2_gru": ("c2", ["--use_recurrent_policy", "true"]),
    "c4": ("c4", []),
    "c3_gru": ("c3", []),
    "c3_jrpo": ("c3", ["--use_joint_action_loss", "true"]),
    "c3_mlp": ("c3", ["--use_recurrent_policy", "false"]),
    "c5_gaussian_host": (None, []),
    "smac8m_gru_host": ("host", ["--use_recurrent_policy", "true", "--use_wide_recurrent_head", "true",
                                 "--use_wide_recurrent_observations", "true"]),
    "smac8m_mlp_host": ("host", ["--use_wide_observations", "true"]),
    "box256_gru_host": ("host", ["--use_recurrent_policy", "true", "--use_wide_recurrent_head", "true",
                                 "--use_wide_recurrent_observations", "true"]),
}
# host-stepped wide paths: (agents, policy features, critic features or None for a Box observation, actions, masks)
HOST_SHAPES = {"smac8m_gru_host": (8, 80, 168, 14, True), "smac8m_mlp_host": (8, 80, 168, 14, True),
               "box256_gru_host": (1, 256, None, 64, False)}
HOST_ENVS, HOST_T = 16, 16


BUFFER = ("actions", "action_log_probs", "policy_obs", "critic_obs", "rewards", "masks", "active_masks", "value_preds", "returns",
          "rnn_states", "rnn_states_critic")


def state_arrays(driver):
    trainer, data = driver.trainer, driver.buffer.data
    m = trainer.algo_module
    out = {"adam_steps": m.adam_steps, "train_info": trainer.train_info}
    for name in BUFFER:   # rnn_states* are None for MLP policies
        if getattr(data, name, None) is not None:
            out[f"buffer_{name}"] = getattr(data, name)
    for net in ("policy", "critic", "model"):   # "model": the shared policy-value network (use_share_model)
        model, opt = m.models.get(net), m.optimizers.get(net)
        if model is not None:
            out[f"{net}_params"] = model.flat_params
            vn = getattr(model, "value_normalizer", None)
            if vn is not None:
                out["valuenorm_state"] = vn.state
        if opt is not None:
            out[f"{net}_exp_avg"], out[f"{net}_exp_avg_sq"] = opt.exp_avg, opt.exp_avg_sq
    return {k: v.detach().cpu().numpy() for k, v in out.items()}


def run_device(workload, flags):
    import bench

    # GridWorldEnv is on no bench workload: C2's flags on it
    bench.WORKLOADS.setdefault("gridworld", dict(bench.WORKLOADS["c2"], env="GridWorldEnv"))
    cfg, env, net, agent = bench.build_agent(0, 1, workload, ENVS, flags)
    drv = bench.make_driver(cfg, env, net, agent, 0, 1)
    for _ in range(K):
        drv.device_iteration()
    return state_arrays(drv)


def run_host_gaussian():
    import torch

    import bench
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(list(bench.FLAGS))
    cfg.quiet = True
    env = HostVecEnv(bench.SyntheticHostEnv(ENVS, seed=0))
    agent = PPOAgent(PPONet(env, cfg=cfg, device=f"cuda:{torch.cuda.current_device()}"))
    agent.train(total_time_steps=ENVS * cfg.episode_length * K, logger=Logger(quiet=True))
    return state_arrays(agent.driver)


class WideHostEnv:
    """Host-stepped synthetic env: n envs x agents, observations ~ N(0, 1) (a Dict {"policy": d, "critic": dc}, or a Box
    of d when dc is None), Discrete(n_actions) with a random legal subset in info["action_masks"] when masks, rewards
    ~ N(0, 1), done ~ Bernoulli(0.05) per env."""

    def __init__(self, n, agents, d, dc, n_actions, masks, seed=0):
        from openrl_b200 import spaces

        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.parallel_env_num, self.agent_num, self.d, self.dc, self.n, self.masks = n, agents, d, dc, n_actions, masks
        self.observation_space = box(d) if dc is None else spaces.Dict({"policy": box(d), "critic": box(dc)})
        self.action_space = spaces.Discrete(n_actions)
        self.rng = np.random.default_rng(seed)

    def _obs(self):
        x = lambda w: self.rng.standard_normal((self.parallel_env_num, self.agent_num, w)).astype(np.float32)  # noqa: E731
        return x(self.d) if self.dc is None else {"policy": x(self.d), "critic": x(self.dc)}

    def _infos(self):
        if not self.masks:
            return [{} for _ in range(self.parallel_env_num)]
        m = (self.rng.random((self.parallel_env_num, self.agent_num, self.n)) < 0.7).astype(np.int8)
        m[..., 0] = 1
        return [{"action_masks": m[i]} for i in range(self.parallel_env_num)]

    def reset(self, seed=None):
        return self._obs(), self._infos()

    def step(self, actions):
        done = np.repeat(self.rng.random((self.parallel_env_num, 1)) < 0.05, self.agent_num, axis=1)
        return self._obs(), self.rng.standard_normal((self.parallel_env_num, self.agent_num, 1)), done, self._infos()


def run_host_wide(name, flags):
    import torch

    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--seed", "0", "--episode_length", str(HOST_T), "--ppo_epoch", "2", "--num_mini_batch",
                                             "2", "--data_chunk_length", "8", "--log_interval", "1000000"] + flags)
    cfg.quiet = True
    env = HostVecEnv(WideHostEnv(HOST_ENVS, *HOST_SHAPES[name]), wide_observations=True)
    agent = PPOAgent(PPONet(env, cfg=cfg, device=f"cuda:{torch.cuda.current_device()}"))
    agent.train(total_time_steps=HOST_ENVS * HOST_T * K, logger=Logger(quiet=True))
    return state_arrays(agent.driver)


def save(out_dir):
    import torch

    assert torch.cuda.is_available(), "update_outputs.py --out needs a CUDA device"
    for name, (workload, flags) in PATHS.items():
        arrays = (run_host_gaussian() if workload is None else run_host_wide(name, flags) if workload == "host"
                  else run_device(workload, flags))
        d = os.path.join(out_dir, name)
        os.makedirs(d, exist_ok=True)
        for k, a in arrays.items():
            np.save(os.path.join(d, k + ".npy"), a)
        print(f"{name}: {', '.join(sorted(arrays))}", flush=True)


def ulp_distance(a, b):
    """Largest distance in units in the last place between two float arrays of one dtype (integers: largest |a - b|);
    two NaNs are at distance 0."""
    if a.size == 0:
        return 0
    if a.dtype.kind != "f":
        return int(np.max(np.abs(a.astype(np.int64) - b.astype(np.int64))))
    it = {4: np.int32, 8: np.int64}[a.dtype.itemsize]

    def ordered(x):   # IEEE bit patterns mapped onto a monotone integer line
        i = x.view(it).astype(np.int64)
        return np.where(i < 0, np.iinfo(it).min - i, i)

    with np.errstate(over="ignore"):
        d = np.abs(ordered(a) - ordered(b))
    return int(np.max(np.where(np.isnan(a) & np.isnan(b), 0, d)))


def compare(dir_a, dir_b):
    worst = 0
    for name in sorted(os.listdir(dir_a)):
        pa, pb = os.path.join(dir_a, name), os.path.join(dir_b, name)
        if not os.path.isdir(pa):
            continue
        for f in sorted(os.listdir(pa)):
            if not os.path.exists(os.path.join(pb, f)):
                print(f"{name}/{f[:-4]}: missing in {dir_b}")
                worst = max(worst, 1)
                continue
            a, b = np.load(os.path.join(pa, f)), np.load(os.path.join(pb, f))
            if a.shape != b.shape or a.dtype != b.dtype:
                print(f"{name}/{f[:-4]}: shape/dtype {a.shape} {a.dtype} vs {b.shape} {b.dtype}")
                worst = max(worst, 1)
                continue
            u = ulp_distance(a, b)
            worst = max(worst, u)
            print(f"{name}/{f[:-4]}: max ulp {u}" + ("" if u == 0 else f"  ({int(np.sum(a != b))} of {a.size} differ)"))
    return worst


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    g = ap.add_mutually_exclusive_group(required=True)
    g.add_argument("--out", metavar="DIR")
    g.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.out:
        save(args.out)
    else:
        print("largest ulp distance:", compare(*args.compare))


if __name__ == "__main__":
    main()
