"""Oracle: plain-PyTorch / numpy statement of the CTC beam search ops in espresso_b200/ops.py (ctc_beam_frames,
ctc_beam_workspace, ctc_beam_search, ctc_beam_finalize), same signatures, fp32 arithmetic.

TEST INFRASTRUCTURE ONLY.  CPU tests monkeypatch these in for `espresso_b200.ops` (next to oracle/ops_ref.py) to run the
host orchestration of espresso_b200/tools/ctc_decoder.py without a GPU.  The search itself is oracle/ctc_beam.py's
statement run in float32; the workspace is a dict holding each sentence's hypotheses.  The product never imports this
module."""
import numpy as np
import torch


def ctc_beam_frames(logits, V, in_lens, K, blank, pad=-1, eos=-1, unk=-1):
    """fp32 log-normaliser, lp[blank] and the K best allowed tokens by (logit desc, id asc); rows past in_lens are 0 / -1."""
    from oracle import ctc_beam as O

    B, T, _ = logits.shape
    x = logits[..., :V].float()
    lse = torch.logsumexp(x, dim=-1)
    lpb = x[..., blank] - lse
    tok = torch.from_numpy(O.topk_tokens(x.numpy(), K, blank, (pad, eos, unk))).to(torch.int32)
    lp = torch.where(tok >= 0, x.gather(-1, tok.clamp(min=0).long()) - lse[..., None], torch.full(tok.shape, float("-inf")))
    live = (torch.arange(T)[None, :] < in_lens.long()[:, None])
    z = lambda v, fill: torch.where(live.view(B, T, *([1] * (v.dim() - 2))), v, torch.full_like(v, fill))  # noqa: E731
    return z(lse, 0.0), z(lpb, 0.0), z(tok, -1), z(lp, float("-inf"))


def ctc_beam_workspace(B, T, beam, device):
    return {"B": B, "T": T, "beam": beam, "hyps": None, "new_order": None}


def _lm_fn(lm, V_lm, lm_blank, rows):
    """Prefix -> fp32 LM log-probs over the CTC vocabulary for the slots `rows` ({prefix: row})."""
    lp = torch.log_softmax(lm[:, :V_lm].float(), dim=-1)
    if lm_blank >= 0:  # the LM has no blank column: give it one (never read)
        lp = torch.cat([lp[:, :lm_blank], torch.zeros(lp.shape[0], 1), lp[:, lm_blank:]], dim=1)
    lp = lp.numpy()
    return lambda y: lp[rows[y]]


def ctc_beam_search(logits, V, in_lens, frames, beam, beam_threshold, t0, t1, workspace, lm=None, V_lm=0, lm_blank=-1,
                    lm_weight=0.0, word_score=0.0, eos=2, want_order=False):
    """oracle/ctc_beam.py's step in fp32 over frames [t0, t1) of every sentence (the workspace holds the hypotheses)."""
    from oracle import ctc_beam as O

    B, T, _ = logits.shape
    lse, lpb, tok, _ = frames
    dt = np.float32
    if t0 == 0:
        workspace["hyps"] = [O.initial(dt) for _ in range(B)]
    col = lambda v: v - 1 if (lm_blank >= 0 and v > lm_blank) else v  # noqa: E731
    order = torch.arange(B * beam, dtype=torch.int32)
    grown = torch.zeros(B * beam, dtype=torch.int32)
    fed = torch.full((B * beam,), col(eos), dtype=torch.int32)
    x = logits[..., :V].float().numpy()
    for b in range(B):
        tend = min(t1, int(in_lens[b]))
        for t in range(t0, tend):
            hyps = workspace["hyps"][b]
            lm_fn = None
            if lm is not None:
                lm_fn = _lm_fn(lm, V_lm, lm_blank, {h.y: b * beam + i for i, h in enumerate(hyps)})
            lp = (x[b, t] - lse[b, t].numpy()).astype(dt)
            hyps, src = O.step(hyps, t, lp, lpb[b, t].numpy(), tok[b, t].numpy(), beam, dt(beam_threshold), lm_fn, lm_weight,
                               word_score, dt)
            workspace["hyps"][b] = hyps
            if t + 1 == tend:
                for k, (h, v) in enumerate(src):
                    order[b * beam + k] = b * beam + h
                    grown[b * beam + k] = int(v >= 0)
                    fed[b * beam + k] = col(v if v >= 0 else eos)
    return (order, grown, fed) if want_order else None


def ctc_beam_finalize(in_lens, T, V, beam, nbest, workspace, lm=None, V_lm=0, lm_blank=-1, lm_weight=0.0, eos=2, pad=1,
                      want_frames=False):
    from oracle import ctc_beam as O

    B = in_lens.numel()
    tokens = torch.full((B, nbest, T), pad, dtype=torch.int32)
    frames = torch.full((B, nbest, T), -1, dtype=torch.int32)
    lens = torch.zeros(B, nbest, dtype=torch.int32)
    scores = torch.full((B, nbest), float("-inf"))
    for b in range(B):
        hyps = workspace["hyps"][b]
        lm_fn = None if lm is None else _lm_fn(lm, V_lm, lm_blank, {h.y: b * beam + i for i, h in enumerate(hyps)})
        for r, (y, s, fr) in enumerate(O.finish(hyps, lm_fn, lm_weight, eos, np.float32)[:nbest]):
            tokens[b, r, :len(y)] = torch.tensor(y, dtype=torch.int32)
            frames[b, r, :len(y)] = torch.tensor(fr, dtype=torch.int32)
            lens[b, r] = len(y)
            scores[b, r] = s
    return tokens, lens, scores, (frames if want_frames else None)
