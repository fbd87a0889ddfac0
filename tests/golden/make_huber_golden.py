"""Generates tests/golden/huber_reference.npz: the reference's own QNetwork, VDNetwork and QMixNetwork with torch.nn.functional.mse_loss replaced by
torch.nn.functional.huber_loss(delta=δ), the definition of algorithm.huber_delta (DESIGN.md §4.4e), on tests/huber_ref.py GOLDEN_CASES.  Run with a
checkout of the reference project:
    MARL_REFERENCE_ROOT=<checkout> python tests/golden/make_huber_golden.py"""
import functools
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import learner_ref as lr  # noqa: E402
from oracle import ref_shim  # noqa: E402
from tests import huber_ref as hr  # noqa: E402
from tests import qmix_options_ref as qo  # noqa: E402
from tests.helpers import GOLDEN, STRIDE, load_params  # noqa: E402


def _grads(module, prefix):
    return {f"{prefix}.{k}": (p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p)) for k, p in module.named_parameters()}


def main():
    ref = ref_shim.load()
    mse = torch.nn.functional.mse_loss
    out = {}
    for key, c in hr.GOLDEN_CASES.items():
        st = hr.golden_state(c)
        kind, n_nets = ("networks", 1) if c.sharing else ("independent", c.N)
        spaces = ([ref_shim.Space(shape=(c.D,))] * c.N, [ref_shim.Space(n=hr.GOLDEN_A)] * c.N)
        cfg = ref_shim.dqn_cfg(target_update_interval_or_tau=2, double_q=c.double_q)
        qmix = c.cls == "QMixNetwork"
        if qmix:
            model = ref.dqn_model.QMixNetwork(*spaces, cfg, [128, 128], c.sharing, False, True, dict(embed_dim=64, hypernet_layers=c.hl, hypernet_embed=32), "cpu")
        else:
            model = getattr(ref.dqn_model, c.cls)(*spaces, cfg, [128, 128], c.sharing, False, True, "cpu")
        load_params(model, lr, (f"critic.{kind}", f"target.{kind}"), st.theta, n_nets, c.D, hr.GOLDEN_A)
        if qmix:
            msd = {}
            for prefix in ("mixer", "target_mixer"):
                msd.update(qo.mixer_state_dict_from_flat(st.mix, prefix, c.N, c.N * c.D, 64, 32, c.hl))
            model.load_state_dict(msd, strict=False)
        torch.nn.functional.mse_loss = functools.partial(torch.nn.functional.huber_loss, delta=c.delta)
        try:
            losses = []
            for u, b in enumerate(hr.golden_batches(c)):
                batch = ref.dqn_train.Batch(b["obss"], b["actions"], b["rewards"], b["dones"], b["filled"], None)
                if u == 0:   # the first update's gradient before the clip (every STRIDE-th element, as the parameters)
                    model.optimizer.zero_grad()
                    model._compute_loss(batch).backward()
                    out[f"{key}_grad0"] = lr.flat_from_state_dict(_grads(model.critic, "critic"), f"critic.{kind}", n_nets).numpy()[::STRIDE]
                    if qmix:
                        out[f"{key}_mix_grad0"] = qo.mixer_flat_from_state_dict(_grads(model.mixer, "mixer"), "mixer", c.hl).numpy()[::STRIDE]
                losses.append(model.update(batch)["loss"])
        finally:
            torch.nn.functional.mse_loss = mse
        sd = model.state_dict()
        out[f"{key}_loss"] = np.array(losses, np.float64)
        out[f"{key}_theta"] = lr.flat_from_state_dict(sd, f"critic.{kind}", n_nets).numpy()[::STRIDE]
        out[f"{key}_theta_tgt"] = lr.flat_from_state_dict(sd, f"target.{kind}", n_nets).numpy()[::STRIDE]
        if qmix:
            out[f"{key}_mix"] = qo.mixer_flat_from_state_dict(sd, "mixer", c.hl).numpy()[::STRIDE]
            out[f"{key}_mix_tgt"] = qo.mixer_flat_from_state_dict(sd, "target_mixer", c.hl).numpy()[::STRIDE]
        print(key, losses)
    np.savez_compressed(os.path.join(GOLDEN, "huber_reference.npz"), **out)


if __name__ == "__main__":
    main()
