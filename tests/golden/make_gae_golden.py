"""Generates tests/golden/gae_reference.npz: the reference's own A2CNetwork / PPONetwork at n_steps = 1 and n_steps = T, the anchors of the
λ-returns at λ = 0 and λ = 1 (tests/gae_ref.py GOLDEN_CASES).  Run with a checkout of the reference project:
    MARL_REFERENCE_ROOT=<checkout> python tests/golden/make_gae_golden.py"""
import os
import sys
from collections import namedtuple

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import learner_ref as lr  # noqa: E402
from oracle import ref_shim  # noqa: E402
from tests import gae_ref as gr  # noqa: E402
from tests.helpers import GOLDEN, STRIDE, ac_oracle_batch, load_params  # noqa: E402

Batch = namedtuple("Batch", ["obss", "actions", "rewards", "dones", "filled", "action_masks"])


def main():
    ref = ref_shim.load()
    N, D, A, T = gr.N, gr.D, gr.A, gr.T
    out = {}
    for key, (cls, _, _, P, steps, epochs, clip, sharing, centralised, std, n_steps, _) in gr.GOLDEN_CASES.items():
        st = gr.golden_state(key)
        cfg = ref_shim.a2c_cfg(grad_clip=clip, num_epochs=epochs, ppo_clip=0.2, target_update_interval_or_tau=2, standardise_returns=std, n_steps=n_steps)
        model = getattr(ref.ac_model, cls)([ref_shim.Space(shape=(D,))] * N, [ref_shim.Space(n=A)] * N, cfg, ref_shim.net_cfg(parameter_sharing=sharing),
                                           ref_shim.net_cfg(parameter_sharing=sharing, centralised=centralised), "cpu")
        kind, n_nets = ("networks", 1) if sharing else ("independent", N)
        load_params(model, lr, (f"actor.{kind}",), st.actor, n_nets, D, A)
        load_params(model, lr, (f"critic.{kind}", f"target_critic.{kind}"), st.critic, n_nets, N * D if centralised else D, 1)
        metrics = []
        for u, (step, s) in enumerate(zip(steps, gr.golden_batches(key))):
            b = ac_oracle_batch(s)
            batch = Batch(b["obss"], b["actions"], b["rewards"], b["dones"].bool(), b["filled"], None)
            if u == 0:   # the first update's returns, as the reference's update computes them (before the running statistics)
                with torch.no_grad():
                    nv, _ = model.get_value(model.split_obs(batch.obss), None, target=True)
                done = batch.dones.float().unsqueeze(-1).repeat(1, 1, N)
                out[f"{key}_returns0"] = ref.utils.compute_nstep_returns(batch.rewards, done, nv, n_steps, cfg.gamma).numpy()
            want = model.update(batch, step)
            metrics.append([float(want[k]) for k in gr.GOLDEN_METRICS])
        out[f"{key}_metrics"] = np.array(metrics, np.float64)
        if std:
            out[f"{key}_ret_mean"], out[f"{key}_ret_var"] = model.ret_ms.mean.numpy(), model.ret_ms.var.numpy()
            out[f"{key}_ret_count"] = np.float64(model.ret_ms.count)
        sd = model.state_dict()
        for name, prefix in (("actor", f"actor.{kind}"), ("critic", f"critic.{kind}"), ("target", f"target_critic.{kind}")):
            out[f"{key}_{name}"] = lr.flat_from_state_dict(sd, prefix, n_nets).numpy()[::STRIDE]
        print(key, metrics)
    np.savez_compressed(os.path.join(GOLDEN, "gae_reference.npz"), **out)


if __name__ == "__main__":
    main()
