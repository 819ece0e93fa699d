"""CPU: the encoder engine's training step at dropout 0.1 against oracle autograd with the engine's own masks.

The engine (espresso_b200/modules/encoder_engine.py) never stores a dropout mask: the backward pass regenerates every
forward mask from a hand-numbered seed _seed(layer, op), some handed across modules through next_drop=(p, seed, scale).
Here the engine runs on the per-op oracle (oracle/ops_ref.py, which draws the kernels' exact counter-RNG masks), and the
fp32 oracle model receives the mask of every site from the seed table in tests/dropout_parity.py.  A wrong seed, index
or scale anywhere in the forward masks or in the chain the backward regenerates breaks the loss, the logits or the
gradients of that sub-layer."""
import pytest
import torch

import dropout_parity as DP
from oracle import ops_ref


@pytest.fixture()
def cpu_ops(monkeypatch):
    from espresso_b200 import ops

    for name in dir(ops_ref):
        if name.startswith("_") or not callable(getattr(ops_ref, name)) or not hasattr(ops, name):
            continue
        monkeypatch.setattr(ops, name, getattr(ops_ref, name))
    ops_ref.set_seed_tensor(None)
    yield ops
    ops_ref.set_seed_tensor(None)


@pytest.mark.parametrize("heads", [4, 2])
@pytest.mark.parametrize("layer_type", ["conformer", "transformer"])
def test_engine_matches_oracle_with_engine_masks_at_dropout(layer_type, heads, golden_dir, cpu_ops):
    """heads=4: the recorded toy fixture (head width 16, unfused attention chain); heads=2: d 128 (head width 64, the
    fused attention forward and backward)."""
    p = 0.1
    sd, g, dims = DP.case(golden_dir, layer_type, heads)
    assert (g["lens"] < g["lens"].max()).any()  # a padded batch: length masks and dropout interact
    m = DP.build(layer_type, sd, p, "cpu", **dims)
    eng = DP.run_engine(m, g, "cpu")
    masks = DP.engine_mask_provider(m.encoder.engine, layer_type, p)
    orc = DP.run_oracle(sd, g, layer_type, p, masks, **dims)
    assert masks.seen == set(DP.site_seed_table(layer_type, 2)), "every dropout site of the oracle drew an engine mask"
    e = DP.compare(layer_type, eng, orc)
    print(layer_type, "loss %.2e logits %.2e worst %s median %.2e" % (e["loss"], e["logits"], e["worst"][:4], e["median"]))
    # bf16 activations end to end against fp32 (the host path's dropout-0 bounds vs the reference fixture)
    assert e["loss"] < 0.03, e["loss"]
    assert e["logits"] < 0.06, e["logits"]
    assert e["worst"][0][0] < 0.25, e["worst"][:5]
    assert e["worst_body"] < 0.1, e["worst"][:8]
    assert e["median"] < 0.05, e["median"]


def test_engine_masks_follow_the_device_seed(golden_dir, cpu_ops):
    """With a device seed installed (what the trainer does for graph replay) every kernel adds it to its op seed: the
    oracle must see the same sum, so the comparison still holds, and the masks differ from the no-device-seed ones."""
    p = 0.1
    sd, g, dims = DP.case(golden_dir, "conformer", 2)
    dev_seed = 2 ** 64 - 12345
    ops_ref.set_seed_tensor(torch.tensor([dev_seed - 2 ** 64], dtype=torch.int64))
    m = DP.build("conformer", sd, p, "cpu", **dims)
    eng = DP.run_engine(m, g, "cpu")
    eng_masks = DP.engine_mask_provider(m.encoder.engine, "conformer", p, device_seed=dev_seed)
    e = DP.compare("conformer", eng, DP.run_oracle(sd, g, "conformer", p, eng_masks, **dims))
    assert e["loss"] < 0.03 and e["logits"] < 0.06 and e["worst_body"] < 0.1 and e["median"] < 0.05, e
    # the same step without the device seed term in the oracle's masks is a different model
    no_dev = DP.engine_mask_provider(m.encoder.engine, "conformer", p)
    e_wrong = DP.compare("conformer", eng, DP.run_oracle(sd, g, "conformer", p, no_dev, **dims))
    assert e_wrong["worst_body"] > 0.1, e_wrong["worst"][:3]
