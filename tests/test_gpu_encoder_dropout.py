"""GPU: the native encoder's training step at dropout 0.1 through the CUDA kernels against oracle autograd with the
kernels' own masks (tests/dropout_parity.py), without and with a device seed, and one CUDA-graph replay of the
Trainer's step at dropout 0.1 against an eager step under the same device-seed value."""
import os

import numpy as np
import pytest
import torch

import dropout_parity as DP
from oracle import ops_ref

pytestmark = pytest.mark.gpu


@pytest.fixture()
def no_device_seed():
    from espresso_b200 import ops

    ops.set_seed_tensor(None)
    ops_ref.set_seed_tensor(None)
    yield
    ops.set_seed_tensor(None)
    ops_ref.set_seed_tensor(None)


@pytest.mark.parametrize("device_seed", [0, 2 ** 64 - 98765], ids=["no_device_seed", "device_seed"])
@pytest.mark.parametrize("layer_type,heads", [("conformer", 4), ("conformer", 2), ("transformer", 4), ("transformer", 2)])
def test_encoder_dropout_vs_oracle_with_kernel_masks(layer_type, heads, device_seed, golden_dir, parity, no_device_seed):
    from espresso_b200 import lib, ops

    p = 0.1
    dev = torch.device("cuda:0")
    if device_seed:
        ops.set_seed_tensor(torch.tensor([device_seed - 2 ** 64], dtype=torch.int64, device=dev))
    sd, g, dims = DP.case(golden_dir, layer_type, heads)
    m = DP.build(layer_type, sd, p, dev, **dims)
    n0 = lib.launch_count()
    eng = DP.run_engine(m, g, dev)
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 > 50  # the native kernels really ran
    masks = DP.engine_mask_provider(m.encoder.engine, layer_type, p, device_seed=device_seed)
    e = DP.compare(layer_type, eng, DP.run_oracle(sd, g, layer_type, p, masks, **dims))
    assert masks.seen == set(DP.site_seed_table(layer_type, 2))
    tag = "encoder %s H=%d dropout 0.1%s" % (layer_type, heads, " + device seed" if device_seed else "")
    parity("%s: CTC loss rel err vs oracle with kernel masks" % tag, e["loss"], 5e-3)
    parity("%s: train logits max abs / max |ref|" % tag, e["logits"], 2e-2)
    parity("%s: worst gradient rel-Frobenius (%s)" % (tag, e["worst"][0][1]), e["worst"][0][0], 0.25)
    parity("%s: worst gradient outside the conv front" % tag, e["worst_body"], 0.1)
    parity("%s: median gradient rel-Frobenius" % tag, e["median"], 0.05)


def test_graph_replay_at_dropout_matches_eager_step(golden_dir, no_device_seed):
    """The bench trains through captured CUDA graphs at dropout 0.1: a replayed step must draw the masks of the device
    seed it finds in memory -- the same gradient as an eager step under that seed value, and not the masks of the step
    that was captured."""
    from espresso_b200.criterions import CtcLossCriterion
    from espresso_b200.optim import NoamLRScheduler
    from espresso_b200.trainer import Trainer

    dev = torch.device("cuda:0")
    g = np.load(os.path.join(golden_dir, "encoder_conformer.npz"))
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    m = DP.build("conformer", sd, 0.1, dev)
    lt = torch.from_numpy(g["lens"])
    sample = {"net_input": {"src_tokens": torch.from_numpy(g["feats"]).to(dev), "src_lengths": lt.to(dev), "src_lengths_cpu": lt},
              "target": torch.from_numpy(g["target"]).to(dev)}
    # buckets equal to the batch's own shape: the graph's static buffers hold exactly this batch
    tr = Trainer(m, CtcLossCriterion(DP._Task(50)), NoamLRScheduler(0.0, 5, 64, 0.0), use_cuda_graphs=True,
                 bucket_frames=g["feats"].shape[1], bucket_tokens=g["target"].shape[1])
    tr._reduce_and_update = lambda: None  # keep the parameters fixed: compare raw gradient buffers
    n = m.flat.numel
    tr.train_step([sample])               # first sight of the shape: eager step (device seed of update 1)
    torch.cuda.synchronize()
    g_first = m.flat.g32[:n].clone()
    tr.train_step([sample])               # capture + replay (device seed of update 2)
    torch.cuda.synchronize()
    assert len(tr._graphs) == 1
    g_graph = m.flat.g32[:n].clone()
    seed_val = int(tr._seed.item())
    assert seed_val == 2 * 1000003
    tr._fwd_bwd([sample])                 # eager, same device-seed value
    torch.cuda.synchronize()
    g_eager = m.flat.g32[:n].clone()
    denom = g_eager.abs().max().item()
    err = (g_graph - g_eager).abs().max().item() / denom
    fresh = (g_graph - g_first).abs().max().item() / denom
    print("graph replay vs eager at dropout 0.1: %.2e (vs the previous update's masks: %.2e)" % (err, fresh))
    assert err < 2e-2, err
    assert fresh > 0.1, fresh             # a replay draws new masks, not the captured step's
