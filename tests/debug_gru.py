"""Debug helper (not a test): one recurrent update on the device vs the torch oracle on the same rollout.
Run on a GPU box:  python tests/debug_gru.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    from oracle import loop_ma
    from openrl_b200.utils.logger import Logger
    from helpers import product

    d = np.load(os.path.join(ROOT, "tests", "golden", "trace_mpe_gru.npz"), allow_pickle=True)
    N = int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split()
    cfg, env, net, agent = product("simple_spread", N, flags, golden=d)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    b = drv.buffer.data
    drv.episode = 0
    drv.actor_rollout()
    drv.compute_returns()
    snap = {k: getattr(b, k).cpu().numpy().copy() for k in
            ("policy_obs", "critic_obs", "rnn_states", "rnn_states_critic", "value_preds", "returns", "masks", "bad_masks",
             "active_masks", "action_masks", "actions", "action_log_probs", "rewards")}
    init = {mk: {k: v.detach().cpu().clone() for k, v in net.module.models[mk].state_dict().items() if "value_normalizer" not in k}
            for mk in ("policy", "critic")}
    rng = torch.get_rng_state()
    tr = drv.trainer
    tr.ppo_epoch = 1
    info1 = tr.train(b)
    my_grads = tr.rnn_grads.cpu().numpy().copy()
    print("device update 1:", info1)
    print("golden update 1:", d["it0/updates"][0])

    # oracle on the same rollout
    ocfg = cfg
    ocfg_epoch = ocfg.ppo_epoch
    ocfg.ppo_epoch = 1
    mt = loop_ma.MATrainer(ocfg, "simple_spread", N)
    for mk, params in (("policy", mt.pol), ("critic", mt.cri)):
        for k in params:
            params[k].data.copy_(init[mk][k])
    for k, v in snap.items():
        setattr(mt.buf, k, v.copy())
    torch.set_rng_state(rng)
    ups, _ = mt.train()
    print("oracle update 1:", ups[0])
    ocfg.ppo_epoch = ocfg_epoch
    for net_i, (mk, params) in enumerate((("policy", mt.pol), ("critic", mt.cri))):
        off = 0
        for k, p in params.items():
            n = p.numel()
            mine = my_grads[net_i, off:off + n].reshape(p.shape)
            ref = p.grad.numpy()
            err = np.abs(mine - ref).max()
            print(f"{mk:7s} {k:34s} |ref|max {np.abs(ref).max():.3e}  max err {err:.3e}")
            off += n
    # tape check (critic tape is the last one written): numpy reductions of the tape vs device grads vs oracle
    WT = tr._lib.orl_rnn_tape_width()
    tape = tr.tape[:300 * WT].view(300, WT).cpu().numpy().astype(np.float64)
    TP_DZ1, TP_DZ3, TP_DGI, TP_DGH, TP_DLOG = 0, 64, 128, 320, 512
    TQ_X, TQ_Y1, TQ_Y3, TQ_HM, TQ_O = 520, 584, 648, 712, 776
    dc = 54
    red = {
        "base.mlp.fc1.0.weight": tape[:, TP_DZ1:TP_DZ1 + 64].T @ tape[:, TQ_X:TQ_X + dc],
        "base.mlp.fc3.0.weight": tape[:, TP_DZ3:TP_DZ3 + 64].T @ tape[:, TQ_Y1:TQ_Y1 + 64],
        "rnn.rnn.weight_ih_l0": tape[:, TP_DGI:TP_DGI + 192].T @ tape[:, TQ_Y3:TQ_Y3 + 64],
        "rnn.rnn.weight_hh_l0": tape[:, TP_DGH:TP_DGH + 192].T @ tape[:, TQ_HM:TQ_HM + 64],
        "v_out.weight": tape[:, TP_DLOG:TP_DLOG + 1].T @ tape[:, TQ_O:TQ_O + 64],
    }
    off = 0
    for k, p in mt.cri.items():
        n = p.numel()
        if k in red:
            mine = my_grads[1, off:off + n].reshape(p.shape)
            print(f"tape-check {k:28s} numpy(tape) vs device {np.abs(red[k] - mine).max():.3e}   numpy(tape) vs oracle {np.abs(red[k] - p.grad.numpy()).max():.3e}")
        off += n
    print("tape rows", tape.shape, "nonfinite", int((~np.isfinite(tape)).sum()))
    # element-wise: CPU core (g++ build of orl_rnn_core.h) on the same chunk inputs vs the device tape
    import ctypes
    import subprocess
    so = "/tmp/rnn_core_shim.so"
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-I", os.path.join(ROOT, "openrl_b200", "csrc"),
                    os.path.join(ROOT, "tests", "rnn_core_shim.cpp"), "-o", so], check=True)
    shim = ctypes.CDLL(so)
    torch.set_rng_state(rng)
    perm = torch.randperm(150).numpy()
    T, B, L, nch = 25, 12, 2, 150
    tape32 = tr.tape[:300 * WT].view(300, WT).cpu().numpy()
    dev = tape32[:nch * L].reshape(nch, L, -1)[:, :, :1224]   # [cpos][l], the fields shared with the CPU core
    X = np.zeros((L, nch, dc), np.float32); M = np.zeros((L, nch), np.float32); DL = np.zeros((L, nch, 1), np.float32)
    H0 = np.zeros((nch, 64), np.float32)
    hc = snap["rnn_states_critic"].reshape(26, B, 64); mk = snap["masks"].reshape(26, B); co = snap["critic_obs"].reshape(26, B, dc)
    for cpos, c in enumerate(perm):
        for l in range(L):
            f = c * L + l
            row, t = f // T, f % T
            X[l, cpos] = co[t, row]; M[l, cpos] = mk[t, row]; DL[l, cpos, 0] = dev[cpos, l, TP_DLOG]
            if l == 0:
                H0[cpos] = hc[t, row]
    print("X vs tape X:", np.abs(X.transpose(1, 0, 2) - dev[:, :, TQ_X:TQ_X + dc]).max())
    P = np.concatenate([init["critic"][k].numpy().ravel() for k in mt.cri]).astype(np.float32)
    out = np.zeros((L * nch, 1), np.float32); cpu_tape = np.zeros((L * nch, 1224), np.float32)
    fp = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    shim.shim_chunk_fwdbwd(fp(P), dc, 1, int(cfg.activation_id), L, nch, fp(np.ascontiguousarray(X)), fp(H0), fp(np.ascontiguousarray(M)),
                           fp(np.ascontiguousarray(DL)), fp(out), fp(cpu_tape))
    cpu = cpu_tape.reshape(L, nch, 1224).transpose(1, 0, 2)  # -> [cpos][l]
    # alternative (a): l=0 steps alone (no gradient arriving from l=1)
    out1 = np.zeros((nch, 1), np.float32); tape1 = np.zeros((nch, 1224), np.float32)
    shim.shim_chunk_fwdbwd(fp(P), dc, 1, int(cfg.activation_id), 1, nch, fp(np.ascontiguousarray(X[0])), fp(H0),
                           fp(np.ascontiguousarray(M[0])), fp(np.ascontiguousarray(DL[0])), fp(out1), fp(tape1))
    print("alt(a) no-chain DGI l=0 vs device:", np.abs(tape1[:, 128:320] - dev[:, 0, 128:320]).max(),
          " vs cpu-chain:", np.abs(tape1[:, 128:320] - cpu[:, 0, 128:320]).max())
    xe = np.abs(cpu[:, :, 520:584] - dev[:, :, 520:584])
    print("X field mismatches per k:", (xe > 1e-6).sum(axis=(0, 1)).tolist())
    print("X dev  chunk0 l0:", np.round(dev[0, 0, 520:584], 3).tolist())
    print("X want chunk0 l0:", np.round(cpu[0, 0, 520:584], 3).tolist())
    names = dict(DZ1=0, DZ3=64, DGI=128, DGH=320, DLOG=512, X=520, Y1=584, Y3=648, HM=712, O=776, DY1N1=840, DY1=904, DY3N3=968,
                 DY3=1032, DONO=1096, DO=1160)
    widths = dict(DGI=192, DGH=192, DLOG=8)
    for nm, o0 in names.items():
        w = widths.get(nm, 64)
        for l in range(L):
            e = np.abs(cpu[:, l, o0:o0 + w] - dev[:, l, o0:o0 + w])
            print(f"field {nm:6s} l={l} max|cpu| {np.abs(cpu[:, l, o0:o0 + w]).max():.3e} max err {e.max():.3e} worst chunk {int(e.max(axis=1).argmax())}")
    # parameters after the update
    for mk, params in (("policy", mt.pol), ("critic", mt.cri)):
        sd = net.module.models[mk].state_dict()
        worst = max(float(np.abs(sd[k].cpu().numpy() - params[k].detach().numpy()).max()) for k in params)
        print(mk, "max param diff after update 1:", worst)


if __name__ == "__main__":
    main()
