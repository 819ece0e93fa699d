"""Cost of fairseq's search options in the native beam search at bench.py's decode shape: the 12 + 6 layer Transformer
(d 256, 4 heads) with the 6 x 512 Transformer LM, beam 5, lm-weight 0.47, eos-factor 1.5, max-len-a 0.08, 50 synthetic 10 s
utterances per batch.  Prints one JSON line: for plain beam search, --no-repeat-ngram-size 3, a forced 2-token prefix,
--diverse-beam-groups 5, --diversity-rate 0.5 and --sampling --sampling-topp 0.9, the milliseconds per batch (CUDA events around generate(), CUDA-graph
replay after two warm-up calls, the options taken in rotating order batch by batch) and the kernel launches per search
step of an eager run, with the card's name and power limit read in the same run.

    python profiles/search_strategy_cost.py [--batches 6]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import _Dict, _Task, synth_wave  # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still reported, without the power limit
        q = "unavailable (%s)" % e
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=6)
    args = ap.parse_args()
    from espresso_b200 import lib
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerModelBase
    from espresso_b200.models.transformer_lm import TransformerLanguageModel
    from espresso_b200.sequence_generator import SequenceGenerator


    dev = torch.device("cuda:0")
    torch.manual_seed(5)
    cfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, layernorm_embedding=False, max_target_positions=1024,
        encoder=dict(embed_dim=256, ffn_embed_dim=1024, layers=12, attention_heads=4, normalize_before=True,
                     learned_pos=False, relative_positional_embeddings=True, layer_type="transformer"),
        decoder=dict(embed_dim=256, ffn_embed_dim=1024, layers=6, attention_heads=4, normalize_before=True,
                     learned_pos=False, relative_positional_embeddings=False, input_dim=256, output_dim=256)))
    model = SpeechTransformerModelBase.build_model(cfg, _Task()).finalize_(dev)
    model.frontend = OnTheFlyFbank(np.full(80, 15.0), np.full(80, 4.0))
    model.eval()
    lm = TransformerLanguageModel(_Dict(), embed_dim=512, ffn_embed_dim=2048, layers=6, attention_heads=8,
                                  max_target_positions=1024).finalize_(dev)
    kw = dict(beam_size=5, max_len_a=0.08, max_len_b=0, lm_model=lm, lm_weight=0.47, eos_factor=1.5)
    per_batch, n = 50, 160000
    rs = np.random.RandomState(3)
    waves = [torch.from_numpy(np.stack([synth_wave(rs, n) for _ in range(per_batch)]).astype(np.float32)).to(dev) for _ in range(2)]
    lens = torch.full((per_batch,), n, dtype=torch.int32, device=dev)
    sample = lambda i: {"net_input": {"src_tokens": waves[i % 2], "src_lengths": lens,  # noqa: E731
                                      "src_lengths_cpu": torch.full((per_batch,), n, dtype=torch.long)}}
    options = {"plain": {}, "ngram3": dict(no_repeat_ngram_size=3), "prefix2": {},
               "groups5": dict(diverse_beam_groups=5, diverse_beam_strength=0.5), "siblings": dict(diversity_rate=0.5),
               "sampling_topp": dict(sampling=True, sampling_topp=0.9)}
    prefix = torch.randint(4, 5000, (per_batch, 2), device=dev)
    pkw = lambda name: {"prefix_tokens": prefix} if name == "prefix2" else {}  # noqa: E731
    gens = {k: SequenceGenerator([model], _Dict(), **kw, **o) for k, o in options.items()}

    # launches per step, eager
    per_step = {}
    steps = {"n": 0}
    orig = model.decode_step

    def counting(*a, **k):
        steps["n"] += 1
        return orig(*a, **k)

    for name, o in options.items():
        g = SequenceGenerator([model], _Dict(), use_cuda_graphs=False, **kw, **o)
        g.generate([model], sample(0), **pkw(name))
        torch.cuda.synchronize()
        model.decode_step = counting
        steps["n"] = 0
        l0 = lib.launch_count()
        g.generate([model], sample(0), **pkw(name))
        torch.cuda.synchronize()
        per_step[name] = (lib.launch_count() - l0) / max(steps["n"], 1)
        model.decode_step = orig

    for name in options:  # eager, capture
        for i in range(2):
            gens[name].generate([model], sample(i), **pkw(name))
    torch.cuda.synchronize()
    names = list(options)
    ms = {k: [] for k in names}
    for i in range(args.batches):
        for name in names[i % len(names):] + names[: i % len(names)]:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            gens[name].generate([model], sample(i), **pkw(name))
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1))
    name, q = _card()
    print(json.dumps({
        "shape": "beam 5, 50 x 10 s utterances, Transformer 12+6 x 256 + 6 x 512 LM, lm_weight 0.47, eos_factor 1.5",
        "ms_per_batch": {k: float(np.median(v)) for k, v in ms.items()}, "ms_all": ms,
        "launches_per_step": per_step, "gpu": name, "power_limit_and_max_sm_clock": q}))


if __name__ == "__main__":
    main()
