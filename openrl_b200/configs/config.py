"""Configuration flags of the rollout + PPO-update hot path.

Mirror of the reference's `create_config_parser()` (openrl/configs/config.py:24) restricted to
the flags the path reads; names and defaults are the reference's (SURVEY.md §5.6 lists the
file:line of each).  `cfg` is a mutable namespace that components also write to, as in the
reference (ppo_net.py:69-81, rl_agent.py:73-74).  `--config file.yaml` is accepted (plain YAML
key: value pairs; the reference's Jinja `globals:` block is resolved when present).
"""
import argparse
import re

import yaml


def _bool(v):
    if isinstance(v, bool):
        return v
    if str(v).lower() in ("true", "1", "yes", "y", "t"):
        return True
    if str(v).lower() in ("false", "0", "no", "n", "f"):
        return False
    raise argparse.ArgumentTypeError(f"bool expected, got {v!r}")


# (name, type, default)
FLAGS = [
    ("seed", int, 0),
    ("env_name", str, "StarCraft2"), ("scenario_name", str, "default"), ("algorithm_name", str, "ppo"),
    ("experiment_name", str, "default"), ("run_dir", str, "./run_results/"),
    ("num_env_steps", float, 10e6), ("episode_length", int, 200), ("n_rollout_threads", int, 32),
    ("learner_n_rollout_threads", int, 32), ("n_eval_rollout_threads", int, 1), ("n_render_rollout_threads", int, 1),
    ("hidden_size", int, 64), ("layer_N", int, 1), ("activation_id", int, 1),
    ("use_popart", _bool, False), ("use_valuenorm", _bool, True), ("use_feature_normalization", _bool, False),
    ("use_orthogonal", _bool, True), ("gain", float, 0.01),
    ("rnn_type", str, "gru"), ("use_naive_recurrent_policy", _bool, False), ("use_recurrent_policy", _bool, False),
    ("recurrent_N", int, 1), ("data_chunk_length", int, 2),
    ("lr", float, 5e-4), ("critic_lr", float, 5e-4), ("opti_eps", float, 1e-5), ("weight_decay", float, 0.0),
    ("ppo_epoch", int, 10), ("use_clipped_value_loss", _bool, True), ("clip_param", float, 0.2),
    ("num_mini_batch", int, 1), ("entropy_coef", float, 0.01), ("value_loss_coef", float, 0.5),
    ("use_max_grad_norm", _bool, True), ("max_grad_norm", float, 10.0),
    ("use_gae", _bool, True), ("gamma", float, 0.99), ("gae_lambda", float, 0.95),
    ("use_proper_time_limits", _bool, False), ("use_huber_loss", _bool, True),
    ("use_value_active_masks", _bool, True), ("use_policy_active_masks", _bool, True), ("huber_delta", float, 10.0),
    ("use_adv_normalize", _bool, False), ("use_linear_lr_decay", _bool, False),
    ("log_interval", int, 5), ("log_each_episode", _bool, True),
    ("use_share_model", _bool, False), ("use_joint_action_loss", _bool, False), ("dual_clip_ppo", _bool, False),
    ("dual_clip_coeff", float, 3.0), ("use_policy_vhead", _bool, False), ("use_single_network", _bool, False),
    ("use_amp", _bool, False), ("use_deepspeed", _bool, False), ("use_fp16", _bool, False),
    ("program_type", str, "local"), ("distributed_type", str, "sync"), ("actor_num", int, 1),
    ("model_dir", str, None), ("load_optimizer", _bool, False), ("disable_wandb", _bool, True),
    ("use_render", _bool, False), ("use_transmit", _bool, False), ("only_eval", _bool, False),
    ("save_interval", int, 1), ("use_eval", _bool, False), ("eval_interval", int, 25),
    ("use_attn", _bool, False), ("use_conv1d", _bool, False), ("use_influence_policy", _bool, False),
    # openrl_b200 additions (not in the reference): how sampling noise / minibatch order are drawn
    ("parity_mode", _bool, False),
    # 64x64 trunk GEMMs of the update on wgmma tensor cores (split-fp16 operands, FP32 accumulate:
    # fp32-class accuracy, so it is also the parity-mode update); Categorical heads, obs widths <= 8,
    # fp32 FFMA kernel otherwise.  `use_tf32` is the round-1 name of the same switch.
    ("use_tensor_cores", _bool, True),
    # replay one captured CUDA graph per iteration (rollout + critic + GAE + all updates + slot shift) instead of ~25
    # launches; used when no callback needs rollout hooks, outside parity_mode, on device-resident envs
    ("use_cuda_graph", _bool, True),
    # self-play (GridWorldSelfPlay): every `selfplay_save_freq` iterations the policy is snapshotted into the opponent pool
    ("selfplay_save_freq", int, 5),
    # host-stepped envs: step two env groups in ping-pong so that the device work of one overlaps the host stepping of the
    # other.  Pays off when env.step is slow relative to the per-step launch cost (MuJoCo-class); for cheap host envs the
    # doubled launch count costs more than the overlap hides (bench extras, c5: 54 ms vs 44 ms per iteration), so off by default
    ("host_env_groups", _bool, False),
    # GRU policies (use_recurrent_policy / use_naive_recurrent_policy) with Discrete action spaces of 9..64 actions: the
    # 64-wide head of the GRU act and update kernels.  Off, a GRU policy keeps its limit of 8 actions (NotImplementedError
    # above); heads of up to 8 actions run the same kernels either way
    ("use_wide_recurrent_head", _bool, False),
    # feed-forward policies and critics with observations of 65..256 features (the policy's, and the critic's of a Dict
    # {"policy", "critic"} env), such as the centralised critic of a many-agent MAPPO env: fc1 as a loop over 64-wide
    # panels of the observation in the act, value, eval and FFMA update kernels.  Off, every network keeps its limit of
    # 64 features (NotImplementedError); GRU policies, use_share_model and the device envs keep it either way
    ("use_wide_observations", _bool, False),
    # GRU policies and critics (use_recurrent_policy / use_naive_recurrent_policy) with observations of 65..256 features,
    # such as SMAC maps beyond the smallest: W1 staged at a wider leading dimension in the GRU act, critic and update
    # kernels, and dW1 reduced in 64-column panels.  Off, a GRU net keeps its limit of 64 features (NotImplementedError);
    # JRPO, use_share_model and the device-env GRU rollout keep it either way
    ("use_wide_recurrent_observations", _bool, False),
    # feed-forward policies with DiagGaussian heads of 9..64 dimensions (Box action spaces such as dm_control's humanoid,
    # 21 actions): the 64-wide head tile of the host act, eval and FFMA update kernels (ORL_HEAD_GAUSSIAN_WIDE).  Off, a
    # DiagGaussian head keeps its limit of 8 dimensions (NotImplementedError above); heads of up to 8 dimensions run the
    # same kernels either way, and GRU policies, use_share_model and JRPO keep the limit with the option on
    ("use_wide_gaussian_head", _bool, False),
    # GRU policies (use_recurrent_policy / use_naive_recurrent_policy) with DiagGaussian heads of 1..8 dimensions on
    # host-stepped Box-action envs (continuous control under partial observability): the GRU act and chunked update with
    # the head as ORL_HEAD_GAUSSIAN.  Off, a GRU policy on a Box action space is refused (NotImplementedError above);
    # Box(9+), JRPO, use_share_model and the device-env GRU rollout refuse it with the option on
    ("use_recurrent_gaussian_head", _bool, False),
    # with use_recurrent_gaussian_head: GRU policies with DiagGaussian heads of 9..64 dimensions (Box action spaces such
    # as dm_control's humanoid, 21 actions, or quadruped, 12): the 64-wide head of the GRU act and update kernels
    # (ORL_HEAD_GAUSSIAN_WIDE).  Off, a GRU policy's DiagGaussian head keeps its limit of 8 dimensions (NotImplementedError
    # above); heads of up to 8 dimensions run the same kernels either way, and JRPO, use_share_model and the device-env
    # GRU rollout refuse it with the option on
    ("use_wide_recurrent_gaussian_head", _bool, False),
    ("use_tf32", _bool, True),
]


class _YamlConfig(argparse.Action):
    """--config x.yaml (reference: ProcessYamlAction, openrl/configs/utils.py:28-101)."""

    def __call__(self, parser, ns, values, option_string=None):
        with open(values) as f:
            content = f.read()
        m = re.search(r"^globals:\n((?:  [^\n]*\n)*)", content, re.MULTILINE)
        if m:
            g = yaml.safe_load("globals:\n" + m.group(1)).get("globals", {})
            content = re.sub(r"^globals:\n((?:  [^\n]*\n)*)", "", content, flags=re.MULTILINE)
            for k, v in g.items():
                content = content.replace("{{ " + k + " }}", str(v))
        data = yaml.safe_load(content) or {}
        known = {a.dest: a for a in parser._actions}
        for k, v in data.items():
            if k in known and known[k].type is not None and v is not None and not isinstance(v, (dict, list)):
                v = known[k].type(v)
            setattr(ns, k, v)


class Config(argparse.Namespace):
    def __contains__(self, k):
        return hasattr(self, k)

    def get(self, k, default=None):
        return getattr(self, k, default)


def create_config_parser():
    parser = argparse.ArgumentParser(description="openrl_b200")
    parser.add_argument("--config", action=_YamlConfig)
    for name, typ, default in FLAGS:
        parser.add_argument("--" + name, type=typ, default=default)
    parser.add_argument("--callbacks", type=yaml.safe_load, default=None)
    orig = parser.parse_args

    def parse_args(args=None, namespace=None):
        return orig(args, namespace if namespace is not None else Config())

    parser.parse_args = parse_args
    return parser
