"""Opponent pool of the device self-play path (reference control flow: SURVEY.md §3.5 —
`OpponentPoolWrapper` openrl/selfplay/wrappers/opponent_pool_wrapper.py:30-120, sampling strategies
selfplay/sample_strategy/{random,last}_opponent.py, snapshot cadence `SelfplayCallback._on_step`
selfplay/callbacks/selfplay_callback.py:124-144).

The pool is a ring of `capacity` policy-parameter snapshots in HBM (20 KB each for the GridWorld policy): the
rollout kernel draws an opponent per episode and evaluates its policy straight from the ring.  `add()` copies the
learner's flat parameters into the next slot and bumps the device counter — plain device ops, so a captured
iteration graph sees new snapshots without re-capture.  With env-sharded multi-GPU training every rank holds the
same parameters (lockstep replicas), so each rank snapshots locally: no broadcast is needed."""
import torch

from .. import lib

STRATEGIES = {"RandomOpponent": lib.SP_RANDOM, "LastOpponent": lib.SP_LAST}


class OpponentPool:
    def __init__(self, capacity, param_count, strategy="RandomOpponent", device="cuda:0"):
        if strategy not in STRATEGIES:
            raise NotImplementedError(f"sample strategy {strategy!r} (built: {sorted(STRATEGIES)})")
        self.capacity, self.strategy_name, self.strategy = int(capacity), strategy, STRATEGIES[strategy]
        self.stride = (int(param_count) + 3) & ~3
        self.device = torch.device(device)
        self.params = torch.zeros(max(self.capacity, 1), self.stride, dtype=torch.float32, device=self.device)
        self.count_dev = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.stats = torch.zeros(self.capacity + 1, 3, dtype=torch.int32, device=self.device)   # wins / losses / draws per slot; last row: random opponent
        self.count = 0          # host mirror of count_dev
        self.steps_of_slot = [None] * self.capacity
        self.activation_id = 1  # hidden activation of the snapshots' policy (cfg.activation_id): the step API evaluates them with it

    def add(self, flat_params, num_time_steps=None, activation_id=1):
        """SelfplayCallback.save_opponent: the learner's current parameters become the newest opponent.  `activation_id` is
        the policy's hidden activation; every snapshot of one pool shares it."""
        if self.count > 0 and activation_id != self.activation_id:
            raise ValueError(f"the pool holds snapshots of activation_id {self.activation_id}, not {activation_id}")
        self.activation_id = int(activation_id)
        if self.capacity == 0:
            return
        slot = self.count % self.capacity
        self.params[slot, :flat_params.numel()].copy_(flat_params)
        self.stats[slot].zero_()                      # the slot now holds a different opponent
        self.count_dev.add_(1)
        self.count += 1
        self.steps_of_slot[slot] = num_time_steps

    def battle_results(self):
        """{slot or "random": (wins, losses, draws) of the training agent} (api_client.add_battle_result's tally)."""
        st = self.stats.cpu().numpy()
        out = {i: tuple(int(v) for v in st[i]) for i in range(min(self.count, self.capacity))}
        out["random"] = tuple(int(v) for v in st[self.capacity])
        return out
