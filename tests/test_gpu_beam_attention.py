"""GPU: encoder attention of the beam search (`print_alignment`) through the C ABI.

esp_decode_cross_attn_weights: context bit-identical to esp_decode_cross_attn, head-averaged weights against the fp32
restatement (oracle/beam_attention.py), rows summing to 1, padded keys exactly 0, H in {4, 8}, Tk up to the 1280 limit.
esp_beam_bookkeep_attn: a bitwise copy of a host walk of the ancestry table, every other output bitwise that of
esp_beam_bookkeep.  End to end on the fixture model in bf16 against the REAL reference (tests/golden/beam_attention.npz)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import beam_attention as OA  # noqa: E402

DEV = torch.device("cuda:0")


@pytest.mark.parametrize("H", [4, 8])
@pytest.mark.parametrize("Tk", [1, 250, 875, 1280])
def test_cross_attn_weights_kernel(H, Tk):
    from espresso_b200 import ops

    torch.manual_seed(H * 10000 + Tk)
    bsz, beam, hd = 3, 4, 64
    N, d = bsz * beam, H * hd
    q = (torch.randn(N, d) * 0.5).bfloat16().to(DEV)
    kv = torch.randn(bsz, Tk, 2 * d).bfloat16().to(DEV)
    for lens in (torch.tensor([Tk, max(1, Tk // 2), max(1, Tk - 7)], dtype=torch.int32), None):
        ln = None if lens is None else lens.to(DEV)
        w = torch.full((N, Tk), float("nan"), device=DEV)
        ctx = ops.decode_cross_attn_weights(q, kv, ln, beam, H, hd ** -0.5, w)
        assert torch.equal(ctx, ops.decode_cross_attn(q, kv, ln, beam, H, hd ** -0.5))  # bit-identical context
        wr = torch.empty(N, Tk)
        OA.decode_cross_attn_weights(q.cpu(), kv.cpu(), lens, beam, H, hd ** -0.5, wr)
        w = w.cpu()
        assert (w - wr).abs().max().item() < 1e-5
        assert (w.sum(-1) - 1).abs().max().item() < 1e-5
        if lens is not None:
            valid = torch.arange(Tk)[None, :] < lens.long()[torch.arange(N) // beam][:, None]
            assert torch.all(w[~valid] == 0)


def test_cross_attn_weights_refuses_more_than_1280_keys():
    from espresso_b200 import ops
    from espresso_b200.lib import EspressoB200Error

    q = torch.zeros(4, 256, dtype=torch.bfloat16, device=DEV)
    kv = torch.zeros(2, 1281, 512, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(EspressoB200Error, match="Tk=1281"):
        ops.decode_cross_attn_weights(q, kv, None, 2, 4, 0.125, torch.empty(4, 1281, device=DEV))


class _St:
    pass


def _state(bsz, beam, L, Tk, dev, seed):
    g = torch.Generator().manual_seed(seed)
    N = bsz * beam
    st = _St()
    st.tokens = torch.randint(4, 20, (N, L), generator=g, dtype=torch.int32)
    st.tokens_alt = torch.zeros_like(st.tokens)
    st.scores = -torch.rand(N, L - 1, generator=g).cumsum(1)
    st.scores_alt = torch.zeros_like(st.scores)
    st.ignore = (torch.rand(N, generator=g) < 0.2).to(torch.uint8)
    st.finished = torch.zeros(bsz, dtype=torch.uint8)
    st.finished[-1] = 1
    st.nfin = torch.randint(0, beam, (bsz,), generator=g, dtype=torch.int32)
    st.fin_tokens = torch.full((bsz, beam, L - 1), 1, dtype=torch.int32)
    st.fin_len = torch.zeros(bsz, beam, dtype=torch.int32)
    st.fin_score = torch.zeros(bsz, beam)
    st.fin_pos = torch.zeros(bsz, beam, L - 1)
    st.fin_attn = torch.zeros(bsz, beam, L - 1, Tk)
    st.new_order = torch.zeros(N, dtype=torch.int32)
    st.n_unfinished = torch.tensor([bsz - 1], dtype=torch.int32)
    for k, v in list(vars(st).items()):
        setattr(st, k, v.to(dev))
    return st


@pytest.mark.parametrize("step", [0, 5, 11])
def test_bookkeep_attn_is_a_bitwise_walk_of_the_ancestry_table(step):
    """Step 0, a middle step and the forced-eos step at max_len (11): the finalised attention columns are exact copies of
    att[t][anc[t][row]] (host walk in oracle/beam_attention.py), everything else is what esp_beam_bookkeep writes."""
    from espresso_b200 import ops

    bsz, beam, max_len, Tk, eos = 5, 4, 11, 37, 2
    L, N = max_len + 2, bsz * beam
    K = 2 * beam
    g = torch.Generator().manual_seed(step)
    cs = -torch.rand(bsz, K, generator=g).cumsum(1)
    ct = torch.randint(4, 20, (bsz, K), generator=g, dtype=torch.int32)
    ct[torch.rand(bsz, K, generator=g) < 0.4] = eos
    ct[0, :beam] = eos  # a sentence that fills its slots this step
    cb = torch.randint(0, beam, (bsz, K), generator=g, dtype=torch.int32)
    T_max = max_len + 3
    att = torch.rand(T_max, N, Tk, generator=g)
    anc = torch.randint(0, N, (T_max, N), generator=g, dtype=torch.int32)
    anc[step] = torch.arange(N, dtype=torch.int32)
    a, b, h = (_state(bsz, beam, L, Tk, d_, 7) for d_ in (DEV, DEV, "cpu"))
    args = (step, max_len, bsz, beam, K, eos, 1, True, 1.0)
    ops.beam_bookkeep_attn(*args, cs.to(DEV), ct.to(DEV), cb.to(DEV), a, att.to(DEV), anc.to(DEV))
    ops.beam_bookkeep(*args, cs.to(DEV), ct.to(DEV), cb.to(DEV), b)
    OA.beam_bookkeep_attn(*args, cs, ct, cb, h, att, anc)
    for k in ("tokens", "tokens_alt", "scores", "scores_alt", "ignore", "finished", "nfin", "fin_tokens", "fin_len", "fin_score",
              "fin_pos", "new_order", "n_unfinished"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert int((a.nfin.cpu() - _state(bsz, beam, L, Tk, "cpu", 7).nfin).sum()) > 0  # something was finalised
    assert torch.equal(a.fin_attn.cpu(), h.fin_attn)


# ---------------------------------------------------------------------------------------------------------------------
# end to end on the fixture model (bf16) against the REAL reference generator
# ---------------------------------------------------------------------------------------------------------------------
class _Npz:
    def __init__(self, sd, base):
        self.d = {"sd." + k: v for k, v in sd.items()}
        self.base = base
        self.files = list(self.d)

    def __getitem__(self, k):
        return self.d[k] if k in self.d else self.base[k]


class _Dict:
    def __len__(self):
        return 50

    def pad(self):
        return 1

    def eos(self):
        return 2

    def unk(self):
        return 3


GEN_KW = {"beam4": dict(beam_size=4, max_len_a=0.0, max_len_b=40), "ensemble": dict(beam_size=4, max_len_a=0.0, max_len_b=40),
          "maxlen": dict(beam_size=4, max_len_a=0.0, max_len_b=3)}
ATT_BOUND = 0.04   # |bf16 attention - fp32|, abs; queries scaled up to 80x (search_model) amplify the bf16 error
# Token identity with the reference is asserted only for sentences whose recorded decision margin (the smallest gap at the
# beam cuts over their search, oracle/pin_beam_attention.py) exceeds MARGIN: below it, bf16 score errors can flip a
# decision.  Every hypothesis the reference also found (any rank) is compared with the reference's matrix; every
# hypothesis at all is compared with the fp32 model teacher-forced along its own tokens.
MARGIN = 0.05


def _models(golden_dir, n):
    from test_host_orchestration import _build_encdec

    e = np.load(os.path.join(golden_dir, "encdec_transformer.npz"))
    sd1 = OA.search_model({k[3:]: e[k] for k in e.files if k.startswith("sd.")})
    sds = [sd1, OA.perturbed(sd1)][:n]
    ms = []
    for sd in sds:
        m = _build_encdec(_Npz(sd, e)).finalize_(DEV)
        m.eval()
        ms.append(m)
    return ms, sds


@pytest.mark.parametrize("case", sorted(GEN_KW))
def test_end_to_end_attention_vs_reference(case, golden_dir, parity):
    from espresso_b200.sequence_generator import SequenceGenerator

    g = np.load(os.path.join(golden_dir, "beam_attention.npz"))
    ms, sds = _models(golden_dir, 2 if case == "ensemble" else 1)
    sample = {"net_input": {"src_tokens": torch.from_numpy(g["feats"]).to(DEV), "src_lengths": torch.from_numpy(g["lens"]).to(DEV)}}
    got = SequenceGenerator(ms, _Dict(), print_alignment=True, **GEN_KW[case]).generate(ms, sample)
    oracles = [OA.Fp32EncDec(sd) for sd in sds]
    encs = [o.forward_encoder({"src_tokens": torch.from_numpy(g["feats"]), "src_lengths": torch.from_numpy(g["lens"])}) for o in oracles]
    worst_own, worst_ref, compared = 0.0, 0.0, 0
    for b, hyps in enumerate(got):
        assert len(hyps) == int(g["%s_b%d_n" % (case, b)])
        for h in hyps:  # every hypothesis: its attention vs the fp32 model teacher-forced along its own tokens
            att = h["attention"]
            prefix = torch.cat([torch.tensor([2]), h["tokens"]])
            for t in range(len(h["tokens"])):
                rows = [OA.decoder_step(o.sd, prefix[None, : t + 1], e["enc"][b:b + 1], None if e["pad"] is None else e["pad"][b:b + 1])[1][0]
                        for o, e in zip(oracles, encs)]
                worst_own = max(worst_own, (att[:, t] - sum(rows) / len(rows)).abs().max().item())
        refs = {tuple(g["%s_b%d_k%d_tokens" % (case, b, k)].tolist()): g["%s_b%d_k%d_attention" % (case, b, k)]
                for k in range(len(hyps))}
        if float(g["%s_b%d_margin" % (case, b)]) > MARGIN:
            assert [h["tokens"].tolist() for h in hyps] == [g["%s_b%d_k%d_tokens" % (case, b, k)].tolist() for k in range(len(hyps))]
        for h in hyps:
            r = refs.get(tuple(h["tokens"].tolist()))
            if r is not None:
                worst_ref = max(worst_ref, (h["attention"] - torch.from_numpy(r)).abs().max().item())
                compared += 1
    if case == "maxlen":  # short hypotheses: most of the reference's n-best is found again in bf16
        assert compared >= 4, compared
    parity("beam attention %s: |att - fp32 along own tokens|" % case, worst_own, ATT_BOUND)
    parity("beam attention %s: |att - reference| (%d hyps in its n-best)" % (case, compared), worst_ref, ATT_BOUND)


def test_alignments_do_not_change_hypotheses_and_graphs_replay_bitwise(golden_dir):
    from espresso_b200.sequence_generator import SequenceGenerator

    g = np.load(os.path.join(golden_dir, "beam_attention.npz"))
    (m,), _ = _models(golden_dir, 1)
    feats, lens = torch.from_numpy(g["feats"]).to(DEV), torch.from_numpy(g["lens"]).to(DEV)
    kw = dict(beam_size=4, max_len_a=0.0, max_len_b=20)
    gen_on = SequenceGenerator([m], _Dict(), print_alignment=True, **kw)
    gen_off = SequenceGenerator([m], _Dict(), **kw)
    eager = SequenceGenerator([m], _Dict(), print_alignment=True, use_cuda_graphs=False, **kw)
    torch.manual_seed(11)
    inputs = [feats, feats.roll(1, dims=0) + 0.3 * torch.randn_like(feats), feats]
    for call, x in enumerate(inputs):  # call 0 eager, 1 capture, 2 replay only
        smp = {"net_input": {"src_tokens": x, "src_lengths": lens}}
        on, off, ref = gen_on.generate([m], smp), gen_off.generate([m], smp), eager.generate([m], smp)
        for a, b, c in zip(on, off, ref):
            assert len(a) == len(b) == len(c)
            for x_, y_, z_ in zip(a, b, c):
                assert torch.equal(x_["tokens"], y_["tokens"]) and torch.equal(x_["score"], y_["score"]), call
                assert torch.equal(x_["positional_scores"], y_["positional_scores"]) and y_["attention"] is None
                assert torch.equal(x_["tokens"], z_["tokens"]) and torch.equal(x_["score"], z_["score"]), call
                assert torch.equal(x_["attention"], z_["attention"]), call
    assert len(next(iter(gen_on._graph_cache.values()))["graphs"]) > 0
