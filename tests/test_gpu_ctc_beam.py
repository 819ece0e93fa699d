"""GPU: the CTC prefix beam search kernels (esp_ctc_beam_frames / _search / _finalize) against oracle/ctc_beam.py run in
float64 on the same bf16 logits.  Hypothesis tokens must match exactly wherever the oracle's score margin to the
neighbouring ranks exceeds MARGIN (closer hypotheses may legitimately swap under fp32 rounding); scores must agree within
1e-4 relative.  An LSTM LM is run in fp32 on the device and in float64 (teacher forced) by the oracle.  Every case records
the error it reached next to its bound through the `parity` fixture (tests/conftest.py)."""
import math

import numpy as np
import pytest
import torch

from oracle import ctc_beam as O
from test_ctc_beam_search import _FakeCTC, _dict, _lstm_lm, lm_oracle_fn

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
MARGIN = 1e-3
SCORE_TOL = 1e-4


def _x(B, T, V, seed, scale=1.0, ld=None, quant=None):
    rs = np.random.RandomState(seed)
    x = rs.randn(B, T, ld or (V + 7) // 8 * 8) * scale
    if quant:
        x = np.round(x * quant) / quant  # many exact ties
    return torch.from_numpy(x).float().bfloat16()


def _repeat_heavy(B, T, V, seed, blank=0, peak=4.0):
    """Peaked logits whose argmax runs repeat the same token over several frames, often as token-blank-token (a
    repeated label): many merges."""
    rs = np.random.RandomState(seed)
    x = rs.randn(B, T, (V + 7) // 8 * 8)
    for b in range(B):
        t, prev = 0, None
        while t < T:
            if prev is not None and prev != blank and rs.rand() < 0.5:
                seq = [blank, prev]
            else:
                seq = [blank if rs.rand() < 0.3 else rs.randint(4, V)]
            for v in seq:
                n = rs.randint(1, 4)
                x[b, t:t + n, v] += peak
                t += n
                prev = v
    return torch.from_numpy(x).float().bfloat16()


# ---- frames --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,K,excl,case", [(2, 2, (-1, -1, -1), "dense"), (7, 4, (1, 2, 3), "dense"), (7, 7, (1, 2, 3), "ties"),
                                           (5004, 60, (1, 2, 3), "dense"), (5004, 128, (1, 2, -1), "slice"),
                                           (8200, 16, (1, 2, 3), "ties"), (8200, 10, (1, 2, 3), "slice")])
def test_frames_top_tokens_and_lp(V, K, excl, case, parity):
    from espresso_b200 import ops

    B, T = 3, 37
    if case == "slice":  # a time and column slice of a larger buffer: unaligned rows, scalar loads
        big = _x(B, T + 9, V + 24, seed=V + K)
        x = big[:, 4:T + 4, 3:3 + V]
    else:
        x = _x(B, T, V, seed=V + K, quant=(2 if case == "ties" else None), scale=(3.0 if case == "ties" else 1.0))
    lens = torch.tensor([T, 20, 1], dtype=torch.int32)
    blank = 0
    lse, lpb, tok, lp = ops.ctc_beam_frames(x.to(DEV) if case != "slice" else big.to(DEV)[:, 4:T + 4, 3:3 + V], V, lens.to(DEV), K,
                                            blank, *excl)
    lse, lpb, tok, lp = (a.cpu() for a in (lse, lpb, tok, lp))
    err = 0.0
    for b in range(B):
        n = int(lens[b])
        x64 = x[b, :n, :V].double().numpy()
        l64 = O.log_softmax(x64)
        ref_tok = O.topk_tokens(x64, K, blank, excl)
        assert np.array_equal(tok[b, :n].numpy(), ref_tok), (b, tok[b, :n], ref_tok)
        lse64 = x64.max(-1) + np.log(np.exp(x64 - x64.max(-1, keepdims=True)).sum(-1))
        err = max(err, np.abs(lse[b, :n].numpy() - lse64).max(), np.abs(lpb[b, :n].numpy() - l64[:, blank]).max())
        ok = ref_tok >= 0
        ref_lp = np.where(ok, np.take_along_axis(l64, np.maximum(ref_tok, 0), -1), -np.inf)
        assert np.array_equal(np.isinf(lp[b, :n].numpy()), ~ok)
        err = max(err, np.abs(lp[b, :n].numpy()[ok] - ref_lp[ok]).max() if ok.any() else 0.0)
    parity("ctc_beam_frames V=%d K=%d %s: |lse|, |lp| abs err" % (V, K, case), err, 2e-5 * max(1.0, math.log(V)))


def test_beam_above_the_maximum_is_refused():
    from espresso_b200 import lib, ops

    x = _x(1, 4, 16, seed=0).to(DEV)
    lens = torch.tensor([4], dtype=torch.int32, device=DEV)
    with pytest.raises(lib.EspressoB200Error, match="beam_size_token"):
        ops.ctc_beam_frames(x, 16, lens, 129, 0)
    fr = ops.ctc_beam_frames(x, 16, lens, 8, 0)
    with pytest.raises(lib.EspressoB200Error, match="beam_size 129"):
        ops.ctc_beam_search(x, 16, lens, fr, 129, 10.0, 0, 4, ops.ctc_beam_workspace(1, 4, 129, DEV))
    ops.ctc_beam_search(x, 16, lens, fr, 128, 10.0, 0, 4, ops.ctc_beam_workspace(1, 4, 128, DEV))  # the maximum works
    torch.cuda.synchronize()


# ---- search ---------------------------------------------------------------------------------------------------------
def _compare(parity, name, dec, x, lens, V, lm_fn=None, check=None):
    """Kernels (through CTCDecoder.search) vs the oracle per sentence: tokens / frames exact where the margins allow,
    scores within SCORE_TOL relative."""
    tokens, L, S, Fr = dec.search(x.to(DEV), V, lens.to(DEV))
    excl = (dec.pad, dec.eos, -1 if dec.allow_unk else dec.unk)
    K = dec.beam_size_token if dec.beam_size_token is not None else min(dec.beam_size, V)
    thr = dec.beam_threshold if dec.beam_threshold is not None else float(min(dec.beam_size, V))
    err, n_exact = 0.0, 0
    for b in (check if check is not None else range(x.shape[0])):
        n = int(lens[b])
        ref = O.search(x[b, :n, :V].double().numpy(), dec.beam_size, K, dec.blank, excl, thr, lm_fn,
                       dec.lm_weight if lm_fn else 0.0, dec.word_score, dec.eos)
        sc = [r[1] for r in ref]
        for r in range(dec.nbest):
            if r >= len(ref):
                assert S[b, r] == -math.inf
                continue
            gap = min(sc[r - 1] - sc[r] if r > 0 else math.inf, sc[r] - sc[r + 1] if r + 1 < len(sc) else math.inf)
            m = int(L[b, r])
            got = tuple(tokens[b, r, :m].tolist())
            if gap > MARGIN:
                assert got == ref[r][0], (name, b, r)
                err = max(err, abs(float(S[b, r]) - sc[r]) / max(1.0, abs(sc[r])))
                if Fr is not None:
                    assert tuple(Fr[b, r, :m].tolist()) == ref[r][2]
                n_exact += 1
            else:  # a near-tie may swap ranks: the hypothesis must still be one of the oracle's, at its score
                alt = [h for h in ref if h[0] == got]
                if alt:
                    err = max(err, abs(float(S[b, r]) - alt[0][1]) / max(1.0, abs(alt[0][1])))
            if r == 0 and n == 0:
                assert int(L[b, 0]) == 0
    assert n_exact > 0
    parity(name + ": score rel err", err, SCORE_TOL)
    return tokens, L, S, Fr


def _decoder(V, beam, blank=0, lm=None, **kw):
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    return CTCDecoder(_dict(n_sym=V - 4), blank_idx=blank, beam_size=beam, lm_model=lm, **kw)


@pytest.mark.parametrize("beam", [1, 4, 16, 60])
def test_search_no_lm_ragged(beam, parity):
    V, B, T = 40, 4, 50
    x = _x(B, T, V, seed=beam, scale=2.0)
    lens = torch.tensor([50, 33, 1, 0])
    dec = _decoder(V, beam, nbest=min(beam, 3), print_alignment=True, word_score=0.25)
    from espresso_b200 import lib

    c0 = lib.launch_count()
    _compare(parity, "ctc beam no LM beam=%d ragged" % beam, dec, x, lens, V)
    assert lib.launch_count() - c0 == 3  # frames, one search launch for all frames, finalize


@pytest.mark.parametrize("beam,K,thr,blank", [(16, 5, None, 0), (16, 16, 2.0, 0), (8, 8, None, 7), (60, 12, 4.0, 5)])
def test_search_no_lm_options(beam, K, thr, blank, parity):
    V, B, T = 48, 3, 40
    x = _x(B, T, V, seed=beam + K + blank, scale=2.5)
    lens = torch.tensor([40, 17, 29])
    dec = _decoder(V, beam, blank=blank, beam_size_token=K, beam_threshold=thr, nbest=3)
    _compare(parity, "ctc beam no LM beam=%d K=%d thr=%s blank=%d" % (beam, K, thr, blank), dec, x, lens, V)


@pytest.mark.parametrize("beam", [4, 16])
def test_search_repeat_heavy_merges(beam, parity):
    V, B, T = 24, 4, 60
    x = _repeat_heavy(B, T, V, seed=beam)
    lens = torch.tensor([60, 59, 31, 2])
    dec = _decoder(V, beam, nbest=2, print_alignment=True)
    tokens, L, _, _ = _compare(parity, "ctc beam repeat-heavy beam=%d" % beam, dec, x, lens, V)
    assert any(a == b for bb in range(B) for a, b in zip(tokens[bb, 0, :int(L[bb, 0])].tolist(),
                                                            tokens[bb, 0, 1:int(L[bb, 0])].tolist()))


def test_search_recipe_shape(parity):
    """T' = 875 (35 s of audio at 40 ms per encoder frame, the longest LibriSpeech utterances), V = 5004, bsz 24; the
    oracle checks a subset of the sentences."""
    V, B, T = 5004, 24, 875
    x = _repeat_heavy(B, T, V, seed=11, peak=6.0)  # peaked like a trained model's posteriors
    lens = torch.tensor([T - 13 * b for b in range(B)])
    dec = _decoder(V, 10, nbest=2)
    _compare(parity, "ctc beam no LM T'=875 V=5004 bsz=24 beam=10", dec, x, lens, V, check=[0, 7, 23])


# ---- LM fusion ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beam,lm_blank", [(4, False), (16, True), (60, False)])
def test_search_lstm_lm_fusion(beam, lm_blank, parity):
    V, B, T = 36, 3, 30
    d_lm = _dict(n_sym=V - 4, bos=not lm_blank)
    lm = _lstm_lm(d_lm, seed=beam, hidden=32).finalize_(DEV, dtype=torch.float32)
    x = _x(B, T, V, seed=100 + beam, scale=2.0)
    lens = torch.tensor([30, 21, 0])
    dec = _decoder(V, beam, lm=lm, lm_weight=0.47, word_score=0.6, nbest=3, print_alignment=True)
    assert dec.lm_blank == (0 if lm_blank else -1)
    lm_fn = lm_oracle_fn(lm.cpu(), V, dec.eos, dec.lm_blank)
    lm.to(DEV)
    _compare(parity, "ctc beam + LSTM LM beam=%d lm_blank=%s" % (beam, lm_blank), dec, x, lens, V, lm_fn=lm_fn)


# ---- the real fixture model -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_lm", [False, True])
def test_fixture_conformer_beam_decode(with_lm, golden_dir, parity):
    import os

    from test_gpu_encoder import _build, _sample

    g = np.load(os.path.join(golden_dir, "encoder_conformer.npz"))
    m = _build("conformer", g)
    m.eval()
    sample = _sample(g, DEV)
    with torch.no_grad():
        net = m(**sample["net_input"])
    V = net["encoder_out"][0].size(-1)
    x = net["b200_out"].cpu()
    lens = net["src_lengths"][0].cpu()
    lm = _lstm_lm(_dict(n_sym=V - 4), seed=9, hidden=32).finalize_(DEV, dtype=torch.float32) if with_lm else None
    dec = _decoder(V, 8, lm=lm, lm_weight=0.47, word_score=0.2, nbest=2)
    lm_fn = None
    if with_lm:
        lm_fn = lm_oracle_fn(lm.cpu(), V, dec.eos, -1)
        lm.to(DEV)
    _compare(parity, "ctc beam fixture conformer LM=%s" % with_lm, dec, x, lens, V, lm_fn=lm_fn)
    # the model path: decode() / generate() on the same sample
    tok, sc, al = dec.decode([m], sample)
    hy = dec.generate([m], sample)
    assert al is None and len(hy) == x.shape[0]
    for b, h in enumerate(hy):
        assert torch.equal(h[0]["tokens"], tok[b, : h[0]["tokens"].numel()]) and h[0]["score"] == float(sc[b])


def test_decode_generate_structure_and_alignment(parity):
    V, B, T = 30, 3, 25
    x = _repeat_heavy(B, T, V, seed=3)
    lens = torch.tensor([25, 12, 0])
    dec = _decoder(V, 6, nbest=4, print_alignment=True)
    model = _FakeCTC(x.to(DEV), lens.to(DEV), V)
    hy = dec.generate([model], {"net_input": {}})
    tok, sc, al = dec.decode([model], {"net_input": {}})
    assert len(hy) == B and tok.shape[0] == B and al.shape == tok.shape
    for b, hs in enumerate(hy):
        n = int(lens[b])
        ref = O.search(x[b, :n, :V].double().numpy(), 6, 6, 0, (1, 2, 3), 6.0, eos=2)
        assert 1 <= len(hs) <= 4 and len(hs) == min(4, len(ref))
        for r, h in enumerate(hs):
            assert set(h) == {"tokens", "score", "attention", "alignment", "positional_scores"}
            t, a = h["tokens"], h["alignment"]
            assert t.dtype == torch.int64 and a.shape == t.shape
            assert not any(v in (0, 1, 2) for v in t.tolist())  # no blank, pad or eos
            assert all(0 <= f < n for f in a.tolist()) and a.tolist() == sorted(set(a.tolist()))
            if r == 0:
                assert tuple(t.tolist()) == ref[0][0] and tuple(a.tolist()) == ref[0][2]
                assert tok[b, : t.numel()].tolist() == t.tolist() and al[b, : t.numel()].tolist() == a.tolist()
        assert [h["score"] for h in hs] == sorted((h["score"] for h in hs), reverse=True)
    assert hy[2][0]["tokens"].numel() == 0 and hy[2][0]["score"] == 0.0  # in_len 0: the empty hypothesis, log 1
