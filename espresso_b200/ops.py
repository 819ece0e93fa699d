"""Thin torch-tensor wrappers over the C ABI (include/espresso_b200.h).

PyTorch is used only for device memory and the current CUDA stream; all arithmetic happens in the
hand-written sm_90a kernels.  Every wrapper requires CUDA tensors and raises otherwise.
"""
import ctypes as C

import torch

from . import lib as _lib
from .lib import ACT_NONE, ACT_RELU, ACT_RELU_BWD, ACT_SILU, ACT_SILU_BWD, EspGemm  # noqa: F401


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


# Device-resident seed increment (uint64/int64 tensor of 1 element) added to every op's seed inside the
# kernels.  The trainer bumps it once per update; because the kernels read it from memory, a captured CUDA
# graph of the whole step replays with fresh dropout masks.
_SEED_T = None


def set_seed_tensor(t):
    global _SEED_T
    _SEED_T = t


def _seed_ptr():
    return None if _SEED_T is None else C.c_void_p(_SEED_T.data_ptr())


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.EspressoB200Error("espresso_b200 ops need CUDA tensors (no CPU fallback)")


# ----------------------------------------------------------------------------------------------
# dense contraction
# ----------------------------------------------------------------------------------------------
def gemm(A, B, C_out, M, N, K, lda, ldb, ldc, *, a_kmajor=True, b_kmajor=True, nb1=1, nb2=1,
         sA=(0, 0), sB=(0, 0), sC=(0, 0), bias=None, act=ACT_NONE, aux=None, ld_aux=0, sAux=(0, 0),
         R=None, ldr=0, sR=(0, 0), alpha=1.0, beta=1.0, C2=None, drop_p=0.0, drop_mode=0, seed=0,
         skew_r=0, tile_n=0, accumulate=False, rowsum_a=None, rowsum_scale=1.0):
    """C = epilogue(op(A) @ op(B)^T); see EspGemm in include/espresso_b200.h.  Strides in elements."""
    _need_cuda(A, B, C_out, bias, aux, R, C2)
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
    g = EspGemm()
    g.A, g.B, g.C = A.data_ptr(), B.data_ptr(), C_out.data_ptr()
    g.C2 = C2.data_ptr() if C2 is not None else None
    g.bias = bias.data_ptr() if bias is not None else None
    g.aux = aux.data_ptr() if aux is not None else None
    g.R = R.data_ptr() if R is not None else None
    if bias is not None:
        assert bias.dtype == torch.bfloat16
    if aux is not None:
        assert aux.dtype == torch.bfloat16
    g.M, g.N, g.K = M, N, K
    g.lda, g.ldb, g.ldc, g.ld_aux, g.ldr = lda, ldb, ldc, ld_aux, ldr
    g.sA1, g.sA2 = sA
    g.sB1, g.sB2 = sB
    g.sC1, g.sC2 = sC
    g.sAux1, g.sAux2 = sAux
    g.sR1, g.sR2 = sR
    g.a_kmajor, g.b_kmajor = int(a_kmajor), int(b_kmajor)
    g.nb1, g.nb2 = nb1, nb2
    g.c_f32 = int(C_out.dtype == torch.float32)
    g.r_f32 = int(R is not None and R.dtype == torch.float32)
    g.act, g.drop_mode, g.skew_r, g.tile_n = act, drop_mode, skew_r, tile_n
    g.accumulate = int(accumulate)
    g.alpha, g.beta, g.drop_p = alpha, beta, drop_p
    g.seed = seed
    g.seed_ptr = _SEED_T.data_ptr() if (_SEED_T is not None and drop_p > 0) else None
    if rowsum_a is not None:
        assert rowsum_a.dtype == torch.float32 and rowsum_a.is_cuda and rowsum_a.numel() >= M and rowsum_a.stride(-1) == 1
        g.rowsum_a, g.rowsum_scale = rowsum_a.data_ptr(), rowsum_scale
    _lib.check(_lib.load().esp_gemm_bf16(C.byref(g), _stream()))
    return C_out


def linear(x, W, bias=None, *, act=ACT_NONE, out=None, out_dtype=torch.bfloat16, **kw):
    """y[M,N] = epi(x[M,K] @ W[N,K]^T + bias); x, W contiguous 2-D (row strides may exceed K)."""
    M, K = x.shape
    N = W.shape[0]
    if out is None:
        out = torch.empty(M, N, device=x.device, dtype=out_dtype)
    return gemm(x, W, out, M, N, K, x.stride(0), W.stride(0), out.stride(0), bias=bias, act=act, **kw)


def linear_dgrad(dy, W, out=None, **kw):
    """Input gradient of `linear`: dx[M,K] = epi(dy[M,N] @ W[N,K]); out: bf16 [M,K] destination (new if None)."""
    M, N = dy.shape
    K = W.shape[1]
    if out is None:
        out = torch.empty(M, K, device=dy.device, dtype=torch.bfloat16)
    return gemm(dy, W, out, M, K, N, dy.stride(0), W.stride(0), out.stride(0), b_kmajor=False, **kw)


def linear_wgrad(dy, x, gW, gb=None):
    """Parameter gradients of `linear`: gW[N,K] += dy[M,N]^T @ x[M,K] (fp32 accumulate, e.g. into the flat gradient
    buffer); with `gb` the bias gradient gb[N] += sum_m dy[m, :] comes out of the same GEMM (row sums of its A operand)."""
    M, N = dy.shape
    K = x.shape[1]
    gW2 = gW.view(N, K)
    gemm(dy, x, gW2, N, K, M, dy.stride(0), x.stride(0), K, a_kmajor=False, b_kmajor=False, accumulate=True,
         rowsum_a=gb)


# ----------------------------------------------------------------------------------------------
# front end
# ----------------------------------------------------------------------------------------------
def num_frames(n_samples):
    """Fbank frames of n 16 kHz samples as `frontend_fbank` frames them: snip_edges, 400-sample (25 ms) window,
    160-sample (10 ms) hop (espresso/tools/utils.py:457-486).  An int, or an integer tensor element-wise."""
    if torch.is_tensor(n_samples):
        return torch.where(n_samples >= 400, 1 + torch.div(n_samples - 400, 160, rounding_mode="floor"),
                           torch.zeros_like(n_samples))
    return 1 + (n_samples - 400) // 160 if n_samples >= 400 else 0


def frontend_fbank(wave, n_samples, cmvn_mean=None, cmvn_std=None, freq_masks=None, time_masks=None,
                   t_max=None, out_dtype=torch.bfloat16, workspace=None):
    """Fused fbank -> CMVN -> SpecAugment.  wave [B, N] fp32/int16 (int16 value range), n_samples int32 [B].

    Returns (feats [B, t_max, 80], lengths int32 [B]).
    """
    _need_cuda(wave, n_samples, cmvn_mean, cmvn_std, freq_masks, time_masks)
    assert wave.dim() == 2 and wave.stride(1) == 1
    assert wave.dtype in (torch.float32, torch.int16)
    assert n_samples.dtype == torch.int32
    B = wave.shape[0]
    if t_max is None:
        t_max = num_frames(wave.shape[1])
    out = torch.empty(B, t_max, 80, device=wave.device, dtype=out_dtype)
    lens = torch.empty(B, device=wave.device, dtype=torch.int32)
    if workspace is None:
        workspace = torch.zeros(max(1, B) * 16, device=wave.device, dtype=torch.uint8)
    nf = 0 if freq_masks is None else freq_masks.shape[1]
    nt = 0 if time_masks is None else time_masks.shape[1]
    for m in (freq_masks, time_masks):
        if m is not None:
            assert m.dtype == torch.int32 and m.is_contiguous() and m.shape[0] == B and m.shape[2] == 2
    for s in (cmvn_mean, cmvn_std):
        if s is not None:
            assert s.dtype == torch.float32 and s.numel() == 80
    _lib.check(_lib.load().esp_frontend_fbank(
        _ptr(wave), int(wave.dtype == torch.int16), wave.stride(0), _ptr(n_samples), B, _ptr(cmvn_mean),
        _ptr(cmvn_std), _ptr(freq_masks), nf, _ptr(time_masks), nt, _ptr(out),
        int(out_dtype == torch.float32), t_max, _ptr(lens), _ptr(workspace), _stream()))
    return out, lens


def specaug_features(x, lens, time_warp=None, freq_masks=None, time_masks=None, out_dtype=None):
    """Adaptive SpecAugment on right-padded features: time warp, then frequency and time masks filled with the
    utterance's mean before the warp.  x [B, T, F] fp32/bf16, lens int32 [B] frames, time_warp int32 [B, 2] = (w0, w),
    masks int32 [B, N, 2] = (start, width), each optional.  Returns a new [B, T, F] tensor of out_dtype (default x.dtype)
    whose frames beyond lens are zero."""
    _need_cuda(x, lens, time_warp, freq_masks, time_masks)
    assert x.dim() == 3 and x.dtype in (torch.float32, torch.bfloat16)
    assert lens.dtype == torch.int32 and lens.numel() == x.shape[0]
    out_dtype = x.dtype if out_dtype is None else out_dtype
    assert out_dtype in (torch.float32, torch.bfloat16)
    x = x.contiguous()
    B, T, F = x.shape
    if time_warp is not None:
        assert time_warp.dtype == torch.int32 and time_warp.is_contiguous() and tuple(time_warp.shape) == (B, 2)
    for m in (freq_masks, time_masks):
        if m is not None:
            assert m.dtype == torch.int32 and m.is_contiguous() and m.dim() == 3 and m.shape[0] == B and m.shape[2] == 2
    nf = 0 if freq_masks is None else freq_masks.shape[1]
    nt = 0 if time_masks is None else time_masks.shape[1]
    out = torch.empty(B, T, F, device=x.device, dtype=out_dtype)
    L = _lib.load()
    ws = None
    if nf > 0 or nt > 0:
        ws = torch.empty(max(1, int(L.esp_specaug_workspace_bytes(B, T))), device=x.device, dtype=torch.uint8)
    _lib.check(L.esp_specaug_features(
        _ptr(x), int(x.dtype == torch.float32), _ptr(out), int(out_dtype == torch.float32), B, T, F, _ptr(lens),
        _ptr(time_warp), _ptr(freq_masks), nf, _ptr(time_masks), nt, _ptr(ws), _stream()))
    return out


# ----------------------------------------------------------------------------------------------
# FLAC decoding
# ----------------------------------------------------------------------------------------------
FLAC_STATUS = {0: "ok", 1: "unsupported stream parameters", 2: "no valid frame where the previous frame ended",
               3: "frame sample numbers out of sequence", 4: "frame CRC-16 mismatch", 5: "reserved or invalid code",
               6: "negative LPC shift", 7: "a frame runs past the end of the stream"}


def flac_decode(data, offsets, params, ld, max_channels, names=None, check=True):
    """Decode a batch of FLAC streams (esp_flac_decode): data uint8 [n_bytes] holds stream b's frames in
    [offsets[b], offsets[b+1]) (int64 [B+1]); params int64 [B, 5] = (total samples, sample rate, channels, bps, max block
    size).  Returns (out float32 [B, ld] in int16 range, zeros past each stream's total, status int32 [B]).  With check,
    reads the status back (one synchronisation) and raises naming the first failing utterance (`names[b]`, else its
    index)."""
    _need_cuda(data, offsets, params)
    assert data.dtype == torch.uint8 and data.is_contiguous()
    assert offsets.dtype == torch.int64 and params.dtype == torch.int64 and params.dim() == 2 and params.shape[1] == 5
    B = params.shape[0]
    assert offsets.numel() == B + 1
    out = torch.empty(B, ld, device=data.device, dtype=torch.float32)
    status = torch.empty(B, device=data.device, dtype=torch.int32)
    L = _lib.load()
    ws = torch.empty(max(1, int(L.esp_flac_decode_workspace_bytes(B, data.numel(), max_channels, ld))), device=data.device,
                     dtype=torch.uint8)
    _lib.check(L.esp_flac_decode(_ptr(data), data.numel(), _ptr(offsets), _ptr(params.contiguous()), B, max_channels,
                                 _ptr(out), ld, _ptr(status), _ptr(ws), _stream()))
    if check:
        bad = status.cpu().nonzero().flatten().tolist()
        if bad:
            b = bad[0]
            code = int(status[b])
            raise _lib.EspressoB200Error("FLAC decoding failed for utterance %s: status %d (%s)%s" % (
                names[b] if names is not None else b, code, FLAC_STATUS.get(code, "?"),
                "" if len(bad) == 1 else "; %d utterances failed" % len(bad)))
    return out, status


# ----------------------------------------------------------------------------------------------
# CTC
# ----------------------------------------------------------------------------------------------
def _grad_with_strides(logits, V):
    """Uninitialised bf16 gradient with exactly the strides of `logits` (a possibly non-dense view such as a time or
    column slice of a larger buffer).  The loss kernels address the gradient with the logits' strides and may write
    each row up to ceil8(V) columns (include/espresso_b200.h), so the storage covers that much past the last row;
    torch.empty_like would return a dense tensor with different strides for a non-dense view."""
    if logits.numel() == 0:
        return torch.empty_like(logits)
    last = sum((n - 1) * s for n, s in zip(logits.shape[:-1], logits.stride()[:-1]))
    n = last + max(logits.shape[-1], (V + 7) // 8 * 8)
    return torch.empty(n, device=logits.device, dtype=logits.dtype).as_strided(logits.shape, logits.stride())


def ctc_loss(logits, V, in_lens, targets, tgt_lens, blank, zero_infinity=True, grad_scale=1.0, want_grad=True):
    """logits bf16 [B, T, ld] (ld >= V, batch-major, any strides with unit column stride, e.g. a time or column slice
    of a larger buffer); returns (loss fp32 [B], grad bf16 or None).  grad has the logits' exact strides."""
    _need_cuda(logits, in_lens, targets, tgt_lens)
    assert logits.dtype == torch.bfloat16 and logits.dim() == 3 and logits.stride(2) == 1 and logits.shape[2] >= V
    assert min(logits.stride()) >= 0
    assert in_lens.dtype == torch.int32 and tgt_lens.dtype == torch.int32 and targets.dtype == torch.int32
    B, T, _ = logits.shape
    u_max = targets.shape[1] if targets.dim() == 2 else 0
    L = _lib.load()
    ws = torch.empty(int(L.esp_ctc_workspace_bytes(B, T, u_max)), device=logits.device, dtype=torch.uint8)
    loss = torch.empty(B, device=logits.device, dtype=torch.float32)
    grad = _grad_with_strides(logits, V) if want_grad else None
    _lib.check(L.esp_ctc_loss(_ptr(logits), logits.stride(0), logits.stride(1), V, B, T, _ptr(in_lens),
                              _ptr(targets.contiguous()), u_max, _ptr(tgt_lens), blank, int(zero_infinity),
                              float(grad_scale), _ptr(loss), _ptr(grad), _ptr(ws), _stream()))
    return loss, grad


# ----------------------------------------------------------------------------------------------
# CTC prefix beam search (include/espresso_b200.h: esp_ctc_beam_*)
# ----------------------------------------------------------------------------------------------
def ctc_beam_frames(logits, V, in_lens, K, blank, pad=-1, eos=-1, unk=-1):
    """logits bf16 [B, T, ld] (addressed like ctc_loss) -> (lse fp32 [B, T], lp_blank fp32 [B, T], top_tok int32 [B, T, K],
    top_lp fp32 [B, T, K]): per frame the K best tokens other than blank / pad / eos / unk (-1 allows one), ranked by
    (logit desc, token id asc); rows t >= in_lens[b] are not written."""
    _need_cuda(logits, in_lens)
    assert logits.dtype == torch.bfloat16 and logits.dim() == 3 and logits.stride(2) == 1 and logits.shape[2] >= V
    assert in_lens.dtype == torch.int32
    B, T, _ = logits.shape
    dev = logits.device
    lse = torch.empty(B, T, device=dev, dtype=torch.float32)
    lpb = torch.empty(B, T, device=dev, dtype=torch.float32)
    tok = torch.empty(B, T, K, device=dev, dtype=torch.int32)
    lp = torch.empty(B, T, K, device=dev, dtype=torch.float32)
    _lib.check(_lib.load().esp_ctc_beam_frames(_ptr(logits), logits.stride(0), logits.stride(1), V, B, T, _ptr(in_lens), K, blank,
                                               pad, eos, unk, _ptr(lse), _ptr(lpb), _ptr(tok), _ptr(lp), _stream()))
    return lse, lpb, tok, lp


def ctc_beam_workspace(B, T, beam, device):
    """Search state + parent table, carried from ctc_beam_search to ctc_beam_finalize (opaque)."""
    return torch.empty(int(_lib.load().esp_ctc_beam_workspace_bytes(B, T, beam)), device=device, dtype=torch.uint8)


def ctc_beam_search(logits, V, in_lens, frames, beam, beam_threshold, t0, t1, workspace, lm=None, V_lm=0, lm_blank=-1,
                    lm_weight=0.0, word_score=0.0, eos=2, want_order=False):
    """Frames [t0, t1) of the prefix beam search (t0 == 0 starts it).  frames: ctc_beam_frames' output; lm: LM logits
    [B * beam, ld] (bf16 / fp32) of every slot's prefix.  With want_order returns (new_order, grown, fed) int32
    [B * beam] of the last frame: source row, 1 when a token was appended, the LM input token (eos when not)."""
    _need_cuda(logits, in_lens, workspace, lm)
    assert logits.dtype == torch.bfloat16 and logits.dim() == 3 and logits.stride(2) == 1 and in_lens.dtype == torch.int32
    assert lm is None or (lm.dim() == 2 and lm.stride(1) == 1 and lm.dtype in (torch.bfloat16, torch.float32))
    B, T, _ = logits.shape
    lse, lpb, tok, lp = frames
    K = tok.shape[-1]
    order = [torch.empty(B * beam, device=logits.device, dtype=torch.int32) for _ in range(3)] if want_order else [None] * 3
    _lib.check(_lib.load().esp_ctc_beam_search(
        _ptr(logits), logits.stride(0), logits.stride(1), V, B, T, _ptr(in_lens), _ptr(lse), _ptr(lpb), _ptr(tok), _ptr(lp), K, beam,
        float(beam_threshold), t0, t1, _ptr(lm), int(lm is not None and lm.dtype == torch.float32),
        0 if lm is None else lm.stride(0), V_lm, lm_blank, float(lm_weight), float(word_score), eos, _ptr(order[0]), _ptr(order[1]),
        _ptr(order[2]), _ptr(workspace), _stream()))
    return tuple(order) if want_order else None


def ctc_beam_finalize(in_lens, T, V, beam, nbest, workspace, lm=None, V_lm=0, lm_blank=-1, lm_weight=0.0, eos=2, pad=1,
                      want_frames=False):
    """-> (tokens int32 [B, nbest, T] pad-filled, lengths int32 [B, nbest], scores fp32 [B, nbest] (natural log, -inf where
    the beam held fewer hypotheses), frames int32 [B, nbest, T] or None)."""
    _need_cuda(in_lens, workspace, lm)
    assert lm is None or (lm.dim() == 2 and lm.stride(1) == 1 and lm.dtype in (torch.bfloat16, torch.float32))
    B = in_lens.numel()
    dev = in_lens.device
    tokens = torch.empty(B, nbest, T, device=dev, dtype=torch.int32)
    lens = torch.empty(B, nbest, device=dev, dtype=torch.int32)
    scores = torch.empty(B, nbest, device=dev, dtype=torch.float32)
    frames = torch.empty(B, nbest, T, device=dev, dtype=torch.int32) if want_frames else None
    _lib.check(_lib.load().esp_ctc_beam_finalize(
        B, T, _ptr(in_lens), V, beam, nbest, _ptr(lm), int(lm is not None and lm.dtype == torch.float32), 0 if lm is None else lm.stride(0),
        V_lm, lm_blank, float(lm_weight), eos, pad, _ptr(workspace), _ptr(tokens), _ptr(lens), _ptr(scores), _ptr(frames), _stream()))
    return tokens, lens, scores, frames


# ----------------------------------------------------------------------------------------------
# n-gram LMs and the CTC prefix beam search fused with them (include/espresso_b200.h: esp_ngram_*, esp_ctc_ngram_*)
# ----------------------------------------------------------------------------------------------
def ngram_score(lm, states, words):
    """lm: NgramLanguageModel; states, words int32 [n] (device) -> (log10 P(word | state) fp32 [n], next state int32 [n])."""
    _need_cuda(states, words)
    assert states.dtype == torch.int32 and words.dtype == torch.int32 and states.shape == words.shape
    g = lm.to(states.device)
    logp = torch.empty(states.shape, device=states.device, dtype=torch.float32)
    nxt = torch.empty(states.shape, device=states.device, dtype=torch.int32)
    _lib.check(_lib.load().esp_ngram_score(C.byref(g["struct"]), states.numel(), _ptr(states.contiguous()), _ptr(words.contiguous()),
                                           _ptr(logp), _ptr(nxt), _stream()))
    return logp, nxt


def ctc_ngram_workspace(B, T, beam, device):
    """Search state (with the n-gram state, trie node and look-ahead per slot) + parent table (opaque)."""
    return torch.empty(int(_lib.load().esp_ctc_ngram_workspace_bytes(B, T, beam)), device=device, dtype=torch.uint8)


def ctc_ngram_search(logits, V, in_lens, frames, beam, beam_threshold, workspace, lm, tok_word=None, lexicon=None,
                     lm_weight=0.0, word_score=0.0):
    """Every frame of the prefix beam search fused with the n-gram `lm` (NgramLanguageModel), in one launch.
    Lexicon-free: tok_word int32 [V] maps CTC tokens to n-gram word ids.  With `lexicon` (LexiconTrie) the search
    follows the trie and scores whole words."""
    _need_cuda(logits, in_lens, workspace, tok_word)
    assert logits.dtype == torch.bfloat16 and logits.dim() == 3 and logits.stride(2) == 1 and in_lens.dtype == torch.int32
    assert (lexicon is None) != (tok_word is None)
    B, T, _ = logits.shape
    lse, lpb, tok, lp = frames
    dev = logits.device
    g = lm.to(dev)
    lx = lexicon.to(dev, lm)["struct"] if lexicon is not None else None
    _lib.check(_lib.load().esp_ctc_ngram_search(
        _ptr(logits), logits.stride(0), logits.stride(1), V, B, T, _ptr(in_lens), _ptr(lse), _ptr(lpb), _ptr(tok), _ptr(lp),
        tok.shape[-1], beam, float(beam_threshold), C.byref(g["struct"]), _ptr(tok_word), 0 if tok_word is None else tok_word.numel(),
        None if lx is None else C.byref(lx),
        float(lm_weight), float(word_score), _ptr(workspace), _stream()))


def ctc_ngram_finalize(in_lens, T, V, beam, nbest, workspace, lm, lexicon=None, lm_weight=0.0, pad=1, want_frames=False):
    """+ lm_weight * log10 P(</s> | y) (root slots only with a lexicon) -> as ctc_beam_finalize."""
    _need_cuda(in_lens, workspace)
    B = in_lens.numel()
    dev = in_lens.device
    g = lm.to(dev)
    lx = lexicon.to(dev, lm)["struct"] if lexicon is not None else None
    tokens = torch.empty(B, nbest, T, device=dev, dtype=torch.int32)
    lens = torch.empty(B, nbest, device=dev, dtype=torch.int32)
    scores = torch.empty(B, nbest, device=dev, dtype=torch.float32)
    frames = torch.empty(B, nbest, T, device=dev, dtype=torch.int32) if want_frames else None
    _lib.check(_lib.load().esp_ctc_ngram_finalize(
        B, T, _ptr(in_lens), V, beam, nbest, C.byref(g["struct"]), None if lx is None else C.byref(lx), float(lm_weight), pad,
        _ptr(workspace), _ptr(tokens), _ptr(lens), _ptr(scores), _ptr(frames), _stream()))
    return tokens, lens, scores, frames


# ----------------------------------------------------------------------------------------------
# HBM-bound block kernels.  Conventions: activations bf16, row-major [rows, channels]; "acc" outputs are
# fp32 tensors that the kernel ACCUMULATES into (they are views of the flat gradient buffer).
# ----------------------------------------------------------------------------------------------
def _bf(*ts):
    for t in ts:
        assert t is None or t.dtype == torch.bfloat16


def layer_norm_fwd(x, gamma, beta, eps=1e-5, lens=None, T=0, drop_p=0.0, seed=0):
    """x [R, d] contiguous.  Returns (y, mean[R], rstd[R]).  lens/T: zero rows t >= lens[b] (rows are [B,T])."""
    _need_cuda(x, gamma, beta, lens)
    _bf(x, gamma, beta)
    assert x.is_contiguous()
    R, d = x.shape
    y = torch.empty_like(x)
    mean = torch.empty(R, device=x.device, dtype=torch.float32)
    rstd = torch.empty(R, device=x.device, dtype=torch.float32)
    _lib.check(_lib.load().esp_layer_norm_fwd(_ptr(x), _ptr(gamma), _ptr(beta), eps, R, d, _ptr(y), _ptr(mean), _ptr(rstd),
                                              _ptr(lens), T, drop_p, seed, _seed_ptr(), _stream()))
    return y, mean, rstd


def layer_norm_bwd(dy, x, mean, rstd, gamma, dgamma_acc, dbeta_acc, dres=None, lens=None, T=0, drop_p=0.0, seed=0, next_drop=None):
    """next_drop = (p, seed, scale): additionally return dropout_p(dx, seed) * scale -- the masked gradient the next module's
    backward starts with -- as a second tensor (same values as ops.dropout(dx, p, seed, scale))."""
    _need_cuda(dy, x, gamma, dres)
    _bf(dy, x, gamma, dres)
    assert dy.is_contiguous() and x.is_contiguous() and (dres is None or dres.is_contiguous())
    assert dgamma_acc.dtype == torch.float32 and dbeta_acc.dtype == torch.float32
    R, d = x.shape
    dx = torch.empty_like(x)
    if next_drop is None:
        _lib.check(_lib.load().esp_layer_norm_bwd(_ptr(dy), _ptr(x), _ptr(mean), _ptr(rstd), _ptr(gamma), _ptr(dres), R, d,
                                                  _ptr(dx), _ptr(dgamma_acc), _ptr(dbeta_acc), _ptr(lens), T, drop_p, seed,
                                                  _seed_ptr(), _stream()))
        return dx
    p2, seed2, scale2 = next_drop
    dx2 = torch.empty_like(x)
    _lib.check(_lib.load().esp_layer_norm_bwd2(_ptr(dy), _ptr(x), _ptr(mean), _ptr(rstd), _ptr(gamma), _ptr(dres), R, d,
                                               _ptr(dx), _ptr(dgamma_acc), _ptr(dbeta_acc), _ptr(lens), T, drop_p, seed,
                                               _seed_ptr(), _ptr(dx2), p2, seed2, scale2, _stream()))
    return dx, dx2


def colsum(x, out_acc, scale=1.0):
    """out_acc[n] += scale * sum_r x[r, n]; x may be a column-slice view (row stride = x.stride(0))."""
    _need_cuda(x, out_acc)
    _bf(x)
    assert out_acc.dtype == torch.float32 and x.stride(1) == 1
    R, N = x.shape
    _lib.check(_lib.load().esp_colsum(_ptr(x), R, N, x.stride(0), scale, _ptr(out_acc), _stream()))


def dropout(x, p, seed, scale=1.0, out=None):
    """y = dropout_p(x) * scale with the GEMM-epilogue RNG (index r*N+n)."""
    _need_cuda(x)
    _bf(x)
    assert x.stride(1) == 1
    R, N = x.shape
    if out is None:
        out = torch.empty(R, N, device=x.device, dtype=torch.bfloat16)
    _lib.check(_lib.load().esp_dropout(_ptr(x), R, N, x.stride(0), out.stride(0), scale, p, seed, _seed_ptr(), _ptr(out), _stream()))
    return out


def mask_rows_(x, lens):
    """In place: zero x[b, t >= lens[b], :] for x [B, T, N]."""
    _need_cuda(x, lens)
    _bf(x)
    assert x.is_contiguous()
    B, T, N = x.shape
    _lib.check(_lib.load().esp_mask_rows(_ptr(x), _ptr(lens), B, T, N, _stream()))
    return x


def qprep_fwd(q, u, v, scale):
    """q [R, d] view (row stride q.stride(0)); returns (q_u, q_v) = ((q+u)*s, (q+v)*s), contiguous."""
    _need_cuda(q, u, v)
    _bf(q, u, v)
    R, d = q.shape
    qu = torch.empty(R, d, device=q.device, dtype=torch.bfloat16)
    qv = torch.empty(R, d, device=q.device, dtype=torch.bfloat16)
    _lib.check(_lib.load().esp_qprep_fwd(_ptr(q), q.stride(0), _ptr(u), _ptr(v), scale, R, d, _ptr(qu), _ptr(qv), _stream()))
    return qu, qv


def qprep_bwd(dqu, dqv, scale, dq_out):
    """dq_out[R, d] view (row stride) = scale * (dqu + dqv)."""
    _need_cuda(dqu, dqv, dq_out)
    _bf(dqu, dqv, dq_out)
    R, d = dqu.shape
    _lib.check(_lib.load().esp_qprep_bwd(_ptr(dqu), _ptr(dqv), scale, R, d, _ptr(dq_out), dq_out.stride(0), _stream()))


def attn_softmax_fwd(scores, T, lens, drop_p=0.0, seed=0, causal=False):
    """scores [H, B, Tq, ld] bf16 over T keys -> (p, p_drop) same shape; p_drop is p when drop_p == 0.
    lens: int32 [B] valid keys per batch entry or None; causal: key j visible to query i iff j <= i."""
    _need_cuda(scores, lens)
    _bf(scores)
    H, B, Tq, ld = scores.shape
    assert scores.is_contiguous()
    p = torch.empty_like(scores)
    pd = torch.empty_like(scores) if drop_p > 0 else None
    _lib.check(_lib.load().esp_attn_softmax_fwd(_ptr(scores), H, B, Tq, T, ld, _ptr(lens), int(causal), _ptr(p), _ptr(pd), drop_p,
                                                seed, _seed_ptr(), _stream()))
    return p, (pd if pd is not None else p)


def attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens, drop_p=0.0, seed=0, save_probs=True, pos_hstride=None, key_bounds=None):
    """Fused relative-position attention forward (esp_attn_fused_fwd): qu, qv [B*T, d]; k, v [B*T, d] views with a common
    row stride (the fused q/k/v buffer); pos [2T-1, E] projected positions (E == d: head h at column h*hd; E == hd: one
    table for all heads); key_bounds: optional (lo, hi) int32 [T] device vectors, query row i attends keys lo[i] <= j < hi[i].
    pos None: plain scaled dot-product attention softmax(qu k^T) v (qu = q * scaling; qv is ignored and may be None).
    Returns (ctx [B*T, d], p, p_drop) with p / p_drop [H, B, T, ld] bf16 or None."""
    if pos is None:
        qv = qu
    _need_cuda(qu, qv, k, v, pos, lens)
    klo, khi = key_bounds if key_bounds is not None else (None, None)
    if klo is not None:
        _need_cuda(klo, khi)
        assert klo.dtype == torch.int32 and khi.dtype == torch.int32 and klo.numel() == T and khi.numel() == T
    _bf(qu, qv, k, v, pos)
    R, d = qu.shape
    hd = d // H
    assert R == B * T and qv.shape == qu.shape and qu.stride(0) == qv.stride(0) and qu.stride(1) == 1
    assert k.stride(0) == v.stride(0) and k.stride(1) == 1 and v.stride(1) == 1 and (pos is None or pos.stride(1) == 1)
    assert lens is None or lens.dtype == torch.int32
    if pos is None:
        pos_hstride = 0
    elif pos_hstride is None:
        pos_hstride = hd if pos.shape[1] == d else 0
    ld = (T + 7) // 8 * 8
    ctx = torch.empty(R, d, device=qu.device, dtype=torch.bfloat16)
    p = torch.empty(H, B, T, ld, device=qu.device, dtype=torch.bfloat16) if save_probs else None
    pd = torch.empty_like(p) if (save_probs and drop_p > 0) else None
    _lib.check(_lib.load().esp_attn_fused_fwd(_ptr(qu), _ptr(qv), qu.stride(0), _ptr(k), _ptr(v), k.stride(0), _ptr(pos),
                                              pos.stride(0) if pos is not None else 0, pos_hstride, B, T, H, hd, _ptr(lens), _ptr(klo), _ptr(khi), _ptr(ctx), d, _ptr(p),
                                              _ptr(pd), ld, drop_p, seed, _seed_ptr(), _stream()))
    return ctx, p, (pd if pd is not None else p)


def attn_fused_bwd(dctx, ctx, qu, v, p, pd, B, T, H, ldp, dk_out, dv_out, drop_p=0.0, seed=0):
    """Score side of the relative-position attention backward (esp_attn_fused_bwd): dctx, ctx, qu [B*T, d]; v [B*T, d] view;
    p / pd [H, B, T, ld] as saved by attn_fused_fwd; dk_out / dv_out [B*T, d] views (same row stride) that receive
    dS^T qu and P_drop^T dctx.  Returns (dS [H,B,T,ld], dBD [H,B,T,ldp] skewed); ldp None (attention without positions):
    no skewed copy, dBD is None."""
    _need_cuda(dctx, ctx, qu, v, p, pd, dk_out, dv_out)
    _bf(dctx, ctx, qu, v, p, pd, dk_out, dv_out)
    R, d = dctx.shape
    hd = d // H
    assert R == B * T and ctx.shape == dctx.shape and dctx.stride(0) == ctx.stride(0) and dctx.stride(1) == 1
    assert p.is_contiguous() and pd.is_contiguous() and p.shape == pd.shape and p.shape[:3] == (H, B, T)
    assert dk_out.stride(0) == dv_out.stride(0) and dk_out.stride(1) == 1 and dv_out.stride(1) == 1 and v.stride(1) == 1
    ld = p.shape[-1]
    ds = torch.empty_like(p)
    dbd = torch.empty(H, B, T, ldp, device=p.device, dtype=torch.bfloat16) if ldp is not None else None
    ws = torch.empty(H * B * T, device=p.device, dtype=torch.float32)
    _lib.check(_lib.load().esp_attn_fused_bwd(_ptr(dctx), _ptr(ctx), dctx.stride(0), _ptr(qu), qu.stride(0), _ptr(v), v.stride(0),
                                              _ptr(p), _ptr(pd), ld, B, T, H, hd, drop_p, seed, _seed_ptr(), _ptr(ws), _ptr(ds),
                                              _ptr(dbd), ldp or 0, _ptr(dk_out), _ptr(dv_out), dk_out.stride(0), _stream()))
    return ds, dbd


def attn_softmax_relaxed_fwd(scores, T, lens, relax_w, drop_p=0.0, seed=0):
    """Relaxed attention probabilities (esp_attn_softmax_relaxed_fwd): scores [H, B, Tq, ld] over T keys -> (p, p_drop):
    p the plain softmax, p_drop = dropout((1 - relax_w) p + relax_w / T), T the padded key count."""
    _need_cuda(scores, lens)
    _bf(scores)
    H, B, Tq, ld = scores.shape
    assert scores.is_contiguous()
    p = torch.empty_like(scores)
    pd = torch.empty_like(scores)
    _lib.check(_lib.load().esp_attn_softmax_relaxed_fwd(_ptr(scores), H, B, Tq, T, ld, _ptr(lens), _ptr(p), _ptr(pd),
                                                        float(relax_w), drop_p, seed, _seed_ptr(), _stream()))
    return p, pd


def attn_softmax_bwd(p, dp_drop, T, ldp, drop_p=0.0, seed=0, want_dbd=True):
    """Returns (dS [H,B,Tq,ld], dBD [H,B,T,ldp] in skewed relative-position layout or None)."""
    _need_cuda(p, dp_drop)
    _bf(p, dp_drop)
    H, B, Tq, ld = p.shape
    ds = torch.empty_like(p)
    dbd = torch.empty(H, B, T, ldp, device=p.device, dtype=torch.bfloat16) if want_dbd else None
    _lib.check(_lib.load().esp_attn_softmax_bwd(_ptr(p), _ptr(dp_drop), H, B, Tq, T, ld, _ptr(ds), _ptr(dbd), ldp, drop_p, seed,
                                                _seed_ptr(), _stream()))
    return ds, dbd


def glu_dwconv_fwd(g, w):
    """g [B, T, 2C], w [C, k] -> (y [B, T, C], stats double [2, C] = per-channel sum / sum of squares of y)."""
    _need_cuda(g, w)
    _bf(g, w)
    assert g.is_contiguous() and w.is_contiguous()
    B, T, C2 = g.shape
    Cn, k = w.shape
    assert C2 == 2 * Cn
    y = torch.empty(B, T, Cn, device=g.device, dtype=torch.bfloat16)
    stats = torch.zeros(2, Cn, device=g.device, dtype=torch.float64)
    _lib.check(_lib.load().esp_glu_dwconv_fwd(_ptr(g), _ptr(w), B, T, Cn, k, _ptr(y), _ptr(stats), _stream()))
    return y, stats


def glu_dwconv_bwd(dy, g, w, dw_acc):
    """Returns dg [B, T, 2C]; accumulates dw into dw_acc fp32 [C, k]."""
    _need_cuda(dy, g, w, dw_acc)
    _bf(dy, g, w)
    assert dy.is_contiguous() and g.is_contiguous() and dw_acc.dtype == torch.float32
    B, T, C2 = g.shape
    Cn, k = w.shape
    dg = torch.empty_like(g)
    _lib.check(_lib.load().esp_glu_dwconv_bwd(_ptr(dy), _ptr(g), _ptr(w), B, T, Cn, k, _ptr(dg), _ptr(dw_acc), _stream()))
    return dg


def bn_finalize(stats, R, C_, eps, momentum, run_mean, run_var, training):
    """-> mr fp32 [2, C] (mean, rstd); in training also updates the fp32 running stats in place."""
    _need_cuda(stats, run_mean, run_var)
    dev = stats.device if stats is not None else run_mean.device
    mr = torch.empty(2, C_, device=dev, dtype=torch.float32)
    _lib.check(_lib.load().esp_bn_finalize(_ptr(stats), R, C_, eps, momentum, _ptr(run_mean), _ptr(run_var), int(training),
                                           _ptr(mr), _stream()))
    return mr


BN_ACT_SILU, BN_ACT_RELU = 1, 2


def conv3x3_fwd(x, w, stride):
    """3x3 convolution, zero padding 1, no bias: x [B, T, F, Cin] (Cin = 1: [B, T, F]) bf16 channels-last, w [Cout, 3, 3, Cin]
    -> y [B, ceil(T/st), ceil(F/sf), Cout]."""
    _need_cuda(x, w)
    _bf(x, w)
    assert x.is_contiguous() and w.is_contiguous()
    st, sf = stride
    Cout = w.shape[0]
    if x.dim() == 3:
        B, T, F_ = x.shape
        y = torch.empty(B, (T + st - 1) // st, (F_ + sf - 1) // sf, Cout, device=x.device, dtype=torch.bfloat16)
        _lib.check(_lib.load().esp_conv3x3_c1_fwd(_ptr(x), _ptr(w), _ptr(y), B, T, F_, Cout, st, sf, _stream()))
        return y
    B, T, F_, Cin = x.shape
    y = torch.empty(B, (T + st - 1) // st, (F_ + sf - 1) // sf, Cout, device=x.device, dtype=torch.bfloat16)
    _lib.check(_lib.load().esp_conv3x3_fwd(_ptr(x), _ptr(w), _ptr(y), B, T, F_, Cin, Cout, st, sf, _stream()))
    return y


def conv3x3_dgrad(dy, w, in_shape, stride):
    """Input gradient of conv3x3_fwd: dy [B, To, Fo, Cout] -> dx [B, T, F, Cin] (in_shape)."""
    _need_cuda(dy, w)
    _bf(dy, w)
    assert dy.is_contiguous() and w.is_contiguous()
    B, T, F_, Cin = in_shape
    dx = torch.empty(B, T, F_, Cin, device=dy.device, dtype=torch.bfloat16)
    _lib.check(_lib.load().esp_conv3x3_dgrad(_ptr(dy), _ptr(w), _ptr(dx), B, T, F_, Cin, w.shape[0], stride[0], stride[1], _stream()))
    return dx


def conv3x3_wgrad(dy, x, dw_acc, stride):
    """Weight gradient of conv3x3_fwd accumulated (fp32, +=) into dw_acc [Cout, 3, 3, Cin] (Cin = 1: x is [B, T, F])."""
    _need_cuda(dy, x, dw_acc)
    _bf(dy, x)
    assert dy.is_contiguous() and x.is_contiguous() and dw_acc.is_contiguous() and dw_acc.dtype == torch.float32
    Cout = dy.shape[-1]
    if x.dim() == 3:
        B, T, F_ = x.shape
        _lib.check(_lib.load().esp_conv3x3_c1_wgrad(_ptr(dy), _ptr(x), _ptr(dw_acc), B, T, F_, Cout, stride[0], stride[1], _stream()))
        return
    B, T, F_, Cin = x.shape
    _lib.check(_lib.load().esp_conv3x3_wgrad(_ptr(dy), _ptr(x), _ptr(dw_acc), B, T, F_, Cin, Cout, stride[0], stride[1], _stream()))


def bn_stats(x, C_, pre_bias=None):
    """Per-channel (sum, sum of squares) of channels-last x [..., C] (+ pre_bias[c], rounded to bf16) -> double [2, C]."""
    _need_cuda(x, pre_bias)
    _bf(x, pre_bias)
    assert x.is_contiguous() and x.shape[-1] == C_
    stats = torch.zeros(2, C_, device=x.device, dtype=torch.float64)
    _lib.check(_lib.load().esp_bn_stats(_ptr(x), _ptr(pre_bias), x.numel() // C_, C_, _ptr(stats), _stream()))
    return stats


def bn_act_fwd(y, mr, gamma, beta, act=BN_ACT_SILU, pre_bias=None):
    _need_cuda(y, mr, gamma, beta, pre_bias)
    _bf(y, gamma, beta, pre_bias)
    assert y.is_contiguous()
    Cn = y.shape[-1]
    z = torch.empty_like(y)
    _lib.check(_lib.load().esp_bn_act_fwd(_ptr(y), _ptr(pre_bias), y.numel() // Cn, Cn, _ptr(mr), _ptr(gamma), _ptr(beta), act,
                                          _ptr(z), _stream()))
    return z


def bn_act_bwd(dz, y, mr, gamma, beta, dgamma_acc, dbeta_acc, act=BN_ACT_SILU, pre_bias=None):
    _need_cuda(dz, y, mr, gamma, beta, pre_bias)
    _bf(dz, y, gamma, beta, pre_bias)
    assert dz.is_contiguous() and y.is_contiguous()
    Cn = y.shape[-1]
    sums = torch.empty(3, Cn, device=y.device, dtype=torch.float64)  # 2C double sums + 2C float coefficients
    dy = torch.empty_like(y)
    _lib.check(_lib.load().esp_bn_act_bwd(_ptr(dz), _ptr(y), _ptr(pre_bias), y.numel() // Cn, Cn, _ptr(mr), _ptr(gamma), _ptr(beta), act,
                                          _ptr(sums), _ptr(dy), _ptr(dgamma_acc), _ptr(dbeta_acc), _stream()))
    return dy


def bn_silu_fwd(y, mr, gamma, beta):
    return bn_act_fwd(y, mr, gamma, beta, BN_ACT_SILU)


def bn_silu_bwd(dz, y, mr, gamma, beta, dgamma_acc, dbeta_acc):
    return bn_act_bwd(dz, y, mr, gamma, beta, dgamma_acc, dbeta_acc, BN_ACT_SILU)


# ----------------------------------------------------------------------------------------------
# optimizer
# ----------------------------------------------------------------------------------------------
def sumsq(g, out):
    _need_cuda(g, out)
    assert g.dtype == torch.float32 and out.dtype == torch.float32
    _lib.check(_lib.load().esp_sumsq_f32(_ptr(g), g.numel(), _ptr(out), _stream()))
    return out


def adam_step(p32, m, v, g, p16, lr, beta1, beta2, eps, weight_decay, step, sumsq_t, denom_dev=None, denom_const=1.0,
              clip_norm=0.0, gnorm_out=None, hyper_dev=None):
    _need_cuda(p32, m, v, g, p16, sumsq_t, denom_dev, gnorm_out)
    assert p32.dtype == m.dtype == v.dtype == g.dtype == torch.float32 and p16.dtype == torch.bfloat16
    n = p32.numel()
    assert m.numel() == n and v.numel() == n and p16.numel() == n and g.numel() >= n
    _lib.check(_lib.load().esp_adam_step(_ptr(p32), _ptr(m), _ptr(v), _ptr(g), _ptr(p16), n, lr, beta1, beta2, eps, weight_decay,
                                         step, _ptr(sumsq_t), _ptr(denom_dev), denom_const, clip_norm, _ptr(gnorm_out),
                                         _ptr(hyper_dev), _stream()))


def cast_f32_bf16(x, y):
    _need_cuda(x, y)
    _lib.check(_lib.load().esp_cast_f32_bf16(_ptr(x), x.numel(), _ptr(y), _stream()))


def cast_bf16_f32(x, y):
    _need_cuda(x, y)
    _lib.check(_lib.load().esp_cast_bf16_f32(_ptr(x), x.numel(), _ptr(y), _stream()))


# ----------------------------------------------------------------------------------------------
# decoder-side kernels
# ----------------------------------------------------------------------------------------------
SMOOTH_UNIFORM, SMOOTH_UNIGRAM, SMOOTH_TEMPORAL = 0, 1, 2


def lsce_loss(logits, V, targets, pad_idx, eps, grad_scale=1.0, want_grad=True, smoothing=SMOOTH_UNIFORM, unigram=None, U=0):
    """logits bf16 [R, >=V] with row stride ld (a multiple of 8; a row or column slice of a larger buffer is fine) and a
    16-byte aligned base; targets int32 [R] -> (loss fp32 [R], nll fp32 [R], grad bf16 or None).  grad has the
    logits' exact strides.  smoothing: uniform | unigram (unigram fp32 [V]) | temporal (rows are [B, U])."""
    _need_cuda(logits, targets, unigram)
    assert unigram is None or (unigram.dtype == torch.float32 and unigram.numel() >= V and unigram.is_contiguous())
    _bf(logits)
    assert logits.dim() == 2 and logits.stride(1) == 1 and logits.shape[1] >= V and targets.dtype == torch.int32
    R, ld = logits.shape[0], logits.stride(0)
    loss = torch.empty(R, device=logits.device, dtype=torch.float32)
    nll = torch.empty(R, device=logits.device, dtype=torch.float32)
    grad = _grad_with_strides(logits, V) if want_grad else None
    _lib.check(_lib.load().esp_lsce_loss(_ptr(logits), ld, V, R, _ptr(targets), pad_idx, eps, smoothing, _ptr(unigram), U,
                                         grad_scale, _ptr(loss), _ptr(nll), _ptr(grad), _stream()))
    return loss, nll, grad


def embed_fwd(tokens, E, pos, U, scale, pad_idx, drop_p=0.0, seed=0):
    """tokens int32 [R] (R = B*U), E bf16 [V, d], pos bf16 [>=U, d] or None -> x bf16 [R, d]."""
    _need_cuda(tokens, E, pos)
    _bf(E, pos)
    assert tokens.dtype == torch.int32
    R, d = tokens.numel(), E.shape[1]
    x = torch.empty(R, d, device=E.device, dtype=torch.bfloat16)
    _lib.check(_lib.load().esp_embed_fwd(_ptr(tokens), _ptr(E), _ptr(pos), U, d, scale, R, pad_idx, _ptr(x), drop_p, seed,
                                         _seed_ptr(), _stream()))
    return x


def embed_bwd(tokens, dx, dE_acc, scale, pad_idx, drop_p=0.0, seed=0):
    _need_cuda(tokens, dx, dE_acc)
    _bf(dx)
    assert dE_acc.dtype == torch.float32 and dx.is_contiguous()
    R, d = dx.shape
    _lib.check(_lib.load().esp_embed_bwd(_ptr(tokens), _ptr(dx), d, scale, R, pad_idx, _ptr(dE_acc), drop_p, seed, _seed_ptr(),
                                         _stream()))


def argmax_rows(x, V):
    """x bf16 [R, ld] -> int32 [R] argmax over the first V columns."""
    _need_cuda(x)
    _bf(x)
    R = x.shape[0]
    out = torch.empty(R, device=x.device, dtype=torch.int32)
    _lib.check(_lib.load().esp_argmax_rows(_ptr(x), x.stride(0), V, R, _ptr(out), _stream()))
    return out


# ----------------------------------------------------------------------------------------------
# beam search step
# ----------------------------------------------------------------------------------------------
def beam_merge(x, V, x_is_logits, out, prev_scores=None, temperature=1.0, lm=None, lm_is_logits=True, lm_weight=0.0,
               pad=1, unk=3, unk_penalty=0.0, eos=2, force_eos=False, eos_factor=None, ban_eos=False):
    """x [N, ld] (bf16 logits or fp32 log-probs) -> out fp32 [N, V] masked candidate scores (+ prev_scores[n])."""
    _need_cuda(x, out, prev_scores, lm)
    assert x.stride(1) == 1 and out.is_contiguous() and out.dtype == torch.float32
    N = x.shape[0]
    _lib.check(_lib.load().esp_beam_merge(
        _ptr(x), int(x.dtype == torch.float32), x.stride(0), int(x_is_logits), temperature, _ptr(lm),
        int(lm is not None and lm.dtype == torch.float32), 0 if lm is None else lm.stride(0), int(lm_is_logits), lm_weight, N, V,
        _ptr(prev_scores), pad, unk, unk_penalty, eos, int(force_eos), int(eos_factor is not None),
        0.0 if eos_factor is None else float(eos_factor), int(ban_eos), _ptr(out), _stream()))
    return out


def beam_topk(cand, bsz, sent_stride, n_cand, K, V):
    """cand fp32; per sentence top-K of n_cand candidates -> (scores [bsz,K], tokens int32, beams int32)."""
    _need_cuda(cand)
    s = torch.empty(bsz, K, device=cand.device, dtype=torch.float32)
    t = torch.empty(bsz, K, device=cand.device, dtype=torch.int32)
    b = torch.empty(bsz, K, device=cand.device, dtype=torch.int32)
    _lib.check(_lib.load().esp_beam_topk(_ptr(cand), sent_stride, bsz, n_cand, K, V, _ptr(s), _ptr(t), _ptr(b), _stream()))
    return s, t, b


def beam_bookkeep(step, max_len, bsz, beam, K, eos, pad, normalize, len_penalty, cs, ct, cb, st):
    """st: SearchState-like object with tokens/scores ping-pong buffers and finalisation slots (see
    espresso_b200/sequence_generator.py).  Swaps the ping-pong halves."""
    _lib.check(_lib.load().esp_beam_bookkeep(
        step, max_len, bsz, beam, K, eos, pad, int(normalize), len_penalty, _ptr(cs), _ptr(ct), _ptr(cb), _ptr(st.tokens),
        _ptr(st.tokens_alt), _ptr(st.scores), _ptr(st.scores_alt), _ptr(st.ignore), _ptr(st.finished), _ptr(st.nfin),
        _ptr(st.fin_tokens), _ptr(st.fin_len), _ptr(st.fin_score), _ptr(st.fin_pos), _ptr(st.new_order), _ptr(st.n_unfinished),
        _stream()))
    st.tokens, st.tokens_alt = st.tokens_alt, st.tokens
    st.scores, st.scores_alt = st.scores_alt, st.scores


def beam_bookkeep_attn(step, max_len, bsz, beam, K, eos, pad, normalize, len_penalty, cs, ct, cb, st, att, anc):
    """beam_bookkeep that also copies every finalised hypothesis's encoder-attention rows att[t][anc[t][row]], t = 0..step,
    into st.fin_attn fp32 [bsz, beam, max_len + 1, Tk]; att fp32 [T_max, N, Tk], anc int32 [T_max, N] (this step's table),
    N = bsz * beam, T_max > step."""
    _need_cuda(att, anc, st.fin_attn)
    N = bsz * beam
    if not (att.dtype == torch.float32 and att.is_contiguous() and att.dim() == 3 and att.shape[1] == N and att.shape[0] > step):
        raise _lib.EspressoB200Error("beam_bookkeep_attn: att must be contiguous fp32 [T_max > step, bsz*beam, Tk], got %s %s"
                                     % (att.dtype, tuple(att.shape)))
    if not (anc.dtype == torch.int32 and anc.is_contiguous() and tuple(anc.shape) == tuple(att.shape[:2])):
        raise _lib.EspressoB200Error("beam_bookkeep_attn: anc must be contiguous int32 %s, got %s %s"
                                     % (tuple(att.shape[:2]), anc.dtype, tuple(anc.shape)))
    if not (st.fin_attn.is_contiguous() and tuple(st.fin_attn.shape) == (bsz, beam, max_len + 1, att.shape[2])):
        raise _lib.EspressoB200Error("beam_bookkeep_attn: fin_attn must be contiguous [bsz, beam, max_len + 1, Tk]")
    _lib.check(_lib.load().esp_beam_bookkeep_attn(
        step, max_len, bsz, beam, K, eos, pad, int(normalize), len_penalty, _ptr(cs), _ptr(ct), _ptr(cb), _ptr(st.tokens),
        _ptr(st.tokens_alt), _ptr(st.scores), _ptr(st.scores_alt), _ptr(st.ignore), _ptr(st.finished), _ptr(st.nfin),
        _ptr(st.fin_tokens), _ptr(st.fin_len), _ptr(st.fin_score), _ptr(st.fin_pos), _ptr(st.new_order), _ptr(st.n_unfinished),
        _ptr(att), _ptr(anc), att.shape[2], _ptr(st.fin_attn), _stream()))
    st.tokens, st.tokens_alt = st.tokens_alt, st.tokens
    st.scores, st.scores_alt = st.scores_alt, st.scores


def beam_block_ngrams(tokens, step, n, lprobs, V):
    """--no-repeat-ngram-size: lprobs fp32 [N, >= V] (in place) = -inf for every token that would repeat an n-gram of the
    int32 token buffer tokens [N, >= step+1] (see include/espresso_b200.h: esp_beam_block_ngrams)."""
    _need_cuda(tokens, lprobs)
    assert tokens.dtype == torch.int32 and tokens.stride(1) == 1 and lprobs.dtype == torch.float32 and lprobs.stride(1) == 1
    _lib.check(_lib.load().esp_beam_block_ngrams(_ptr(tokens), tokens.stride(0), tokens.shape[0], step, n, _ptr(lprobs),
                                                 lprobs.stride(0), V, _stream()))
    return lprobs


def beam_prefix(prefix, step, beam, pad, eos, cand, V, st):
    """--prefix-size at `step`: prefix int32 [bsz, P > step]; cand fp32 [bsz*beam, V] (in place); st.tokens / st.scores are
    the search's current token and score rows (beam 0 copied into every beam where the prefix token is eos)."""
    _need_cuda(prefix, cand)
    assert prefix.dtype == torch.int32 and prefix.stride(1) == 1 and cand.is_contiguous()
    assert st.tokens.is_contiguous() and st.scores.is_contiguous() and st.scores.shape[1] == st.tokens.shape[1] - 1
    _lib.check(_lib.load().esp_beam_prefix(_ptr(prefix), prefix.stride(0), prefix.shape[0], beam, step, pad, eos, _ptr(cand), V,
                                           _ptr(st.tokens), st.tokens.shape[1], _ptr(st.scores), _stream()))
    return cand


def beam_diverse_groups(lprobs, prev_scores, bsz, beam, V, groups, Kg, strength):
    """--diverse-beam-groups: lprobs fp32 [bsz*beam, V] without cumulative scores, prev_scores fp32 [bsz*beam] or None at
    step 0 -> (scores [bsz, Kg*groups], tokens int32, beams int32), interleaved by group."""
    _need_cuda(lprobs, prev_scores)
    assert lprobs.is_contiguous() and lprobs.dtype == torch.float32
    K = Kg * groups
    s = torch.empty(bsz, K, device=lprobs.device, dtype=torch.float32)
    t = torch.empty(bsz, K, device=lprobs.device, dtype=torch.int32)
    b = torch.empty(bsz, K, device=lprobs.device, dtype=torch.int32)
    _lib.check(_lib.load().esp_beam_diverse_groups(_ptr(lprobs), _ptr(prev_scores), bsz, beam, V, groups, Kg, float(strength),
                                                   _ptr(s), _ptr(t), _ptr(b), _stream()))
    return s, t, b


def beam_sibling_topk(cand, bsz, beam, V, k, rate):
    """--diversity-rate at step > 0: cand fp32 [bsz*beam, V] with cumulative scores -> (scores [bsz, k], tokens int32,
    beams int32)."""
    _need_cuda(cand)
    assert cand.is_contiguous() and cand.dtype == torch.float32
    dev = cand.device
    ws = torch.empty(bsz * beam * k, device=dev, dtype=torch.float32)
    wt = torch.empty(bsz * beam * k, device=dev, dtype=torch.int32)
    wb = torch.empty(bsz * beam * k, device=dev, dtype=torch.int32)
    s = torch.empty(bsz, k, device=dev, dtype=torch.float32)
    t = torch.empty(bsz, k, device=dev, dtype=torch.int32)
    b = torch.empty(bsz, k, device=dev, dtype=torch.int32)
    _lib.check(_lib.load().esp_beam_sibling_topk(_ptr(cand), bsz, beam, V, k, float(rate), _ptr(ws), _ptr(wt), _ptr(wb), _ptr(s),
                                                 _ptr(t), _ptr(b), _stream()))
    return s, t, b


def beam_sample(lprobs, prev_scores, bsz, beam, V, topk, topp, seed, step):
    """--sampling: lprobs fp32 [bsz*beam, V] without cumulative scores, prev_scores fp32 [bsz*beam] or None at step 0, seed
    int64 [1] on the device -> (scores [bsz, beam], tokens int32, beams int32); see esp_beam_sample."""
    _need_cuda(lprobs, prev_scores, seed)
    assert lprobs.is_contiguous() and lprobs.dtype == torch.float32 and seed.dtype == torch.int64
    s = torch.empty(bsz, beam, device=lprobs.device, dtype=torch.float32)
    t = torch.empty(bsz, beam, device=lprobs.device, dtype=torch.int32)
    b = torch.empty(bsz, beam, device=lprobs.device, dtype=torch.int32)
    _lib.check(_lib.load().esp_beam_sample(_ptr(lprobs), _ptr(prev_scores), bsz, beam, V, int(topk), float(topp), _ptr(seed), step,
                                           _ptr(s), _ptr(t), _ptr(b), _stream()))
    return s, t, b


def lookahead_words(nodes_in, new_order, node_word, word_unk, nodes_out, words):
    """Look-ahead LM fusion, part 1: nodes_out = nodes_in[new_order]; words = word completed at each node (or <unk>)."""
    _need_cuda(nodes_in, node_word, nodes_out, words)
    _lib.check(_lib.load().esp_lookahead_words(_ptr(nodes_in), _ptr(new_order) if new_order is not None else None, _ptr(node_word),
                                               word_unk, nodes_in.numel(), _ptr(nodes_out), _ptr(words), _stream()))


def wordlm_cumsum(logits, Vw, prev_tokens, tok_stride, space_idx, first, cum_in, new_order, cum_out, eos_logprob, word_eos,
                  log_mode=False):
    """Part 2: rows after a <space> (all rows if first) get cumsum(softmax(logits[:, :Vw])) -- or log_softmax with
    log_mode -- the rest inherit cum_in[new_order].  logits bf16 / fp32 [N, >= Vw]; prev_tokens: int32 view with element
    stride tok_stride."""
    _need_cuda(logits, cum_in, cum_out, eos_logprob)
    assert logits.dtype in (torch.bfloat16, torch.float32) and logits.stride(1) == 1 and prev_tokens.dtype == torch.int32
    assert cum_out.is_contiguous() and cum_in.is_contiguous() and cum_out.shape[1] == Vw
    _lib.check(_lib.load().esp_wordlm_cumsum(
        _ptr(logits), int(logits.dtype == torch.float32), logits.stride(0), logits.shape[0], Vw, _ptr(prev_tokens), tok_stride,
        space_idx, int(first), _ptr(cum_in), _ptr(new_order) if new_order is not None else None, _ptr(cum_out), _ptr(eos_logprob),
        word_eos, int(log_mode), _stream()))


def lookahead_step(prev_tokens, tok_stride, first, nodes_in, nodes_out, cum, Vw, eos_logprob, tree, space_idx, eos_idx, pad_idx,
                   word_unk, oov_penalty, open_vocab, zero, out, Vs):
    """Part 3: prefix-tree transition and the fp32 subword log-probability rows out[:, :Vs] (tree: dict of device int32
    arrays from TensorizedPrefixTree.to)."""
    _need_cuda(nodes_in, nodes_out, cum, out)
    assert out.dtype == torch.float32 and out.stride(1) == 1 and cum.is_contiguous()
    _lib.check(_lib.load().esp_lookahead_step(
        _ptr(prev_tokens), tok_stride, nodes_in.numel(), int(first), _ptr(nodes_in), _ptr(nodes_out), _ptr(cum), Vw, _ptr(eos_logprob),
        _ptr(tree["child_off"]), _ptr(tree["child_tok"]), _ptr(tree["child_node"]), _ptr(tree["node_word"]), _ptr(tree["node_lo"]),
        _ptr(tree["node_hi"]), space_idx, eos_idx, pad_idx, word_unk, oov_penalty, int(open_vocab), zero, _ptr(out), out.stride(0), Vs,
        _stream()))


def multilevel_step(prev_tokens, tok_stride, first, nodes_in, nodes_out, new_order, wlp, Vw, sub, sub_is_logits, sub_weight, out_prev,
                    cumlp_in, cumlp_out, tree, space_idx, eos_idx, word_unk, word_eos, log_oov_penalty, open_vocab, logzero, out, Vs):
    """Multi-level (subword + word) LM step: see esp_multilevel_step in include/espresso_b200.h."""
    _need_cuda(nodes_in, nodes_out, wlp, sub, out)
    assert sub.dtype in (torch.bfloat16, torch.float32) and sub.stride(1) == 1 and out.dtype == torch.float32 and wlp.is_contiguous()
    assert out_prev.stride() == out.stride()
    _lib.check(_lib.load().esp_multilevel_step(
        _ptr(prev_tokens), tok_stride, nodes_in.numel(), int(first), _ptr(nodes_in), _ptr(nodes_out),
        _ptr(new_order) if new_order is not None else None, _ptr(wlp), Vw, _ptr(sub), int(sub.dtype == torch.float32), sub.stride(0),
        int(sub_is_logits), sub_weight, _ptr(out_prev), _ptr(cumlp_in), _ptr(cumlp_out), _ptr(tree["child_off"]),
        _ptr(tree["child_tok"]), _ptr(tree["child_node"]), _ptr(tree["node_word"]), space_idx, eos_idx, word_unk, word_eos,
        log_oov_penalty, int(open_vocab), logzero, _ptr(out), out.stride(0), Vs, _stream()))


def gather_rows(src, idx, out=None):
    """out[i] = src[idx[i]] along dim 0 (rows must be multiples of 16 bytes)."""
    _need_cuda(src, idx)
    assert src.is_contiguous() and idx.dtype == torch.int32
    if out is None:
        out = torch.empty((idx.numel(),) + tuple(src.shape[1:]), device=src.device, dtype=src.dtype)
    row_bytes = src[0].numel() * src.element_size()
    _lib.check(_lib.load().esp_gather_rows(_ptr(src), _ptr(idx), row_bytes, idx.numel(), _ptr(out), _stream()))
    return out


# ----------------------------------------------------------------------------------------------
# incremental decoding
# ----------------------------------------------------------------------------------------------
def decode_self_attn(q, kv_cache, anc, T, H, scale):
    """q bf16 [N, d]; kv_cache bf16 [T_max, N, 2d]; anc int32 [T_max, N]; attends over times 0..T-1 -> [N, d]."""
    _need_cuda(q, kv_cache, anc)
    _bf(q, kv_cache)
    N, d = q.shape
    out = torch.empty_like(q)
    _lib.check(_lib.load().esp_decode_self_attn(_ptr(q), _ptr(kv_cache), _ptr(anc), N, H, d // H, T, scale, _ptr(out), _stream()))
    return out


def decode_cross_attn(q, kv, lens, beam, H, scale):
    """q bf16 [N, d]; kv bf16 [bsz, Tk, 2d]; lens int32 [bsz] or None -> [N, d]."""
    _need_cuda(q, kv, lens)
    _bf(q, kv)
    N, d = q.shape
    out = torch.empty_like(q)
    _lib.check(_lib.load().esp_decode_cross_attn(_ptr(q), _ptr(kv), _ptr(lens), N, beam, H, d // H, kv.shape[1], scale, _ptr(out),
                                                 _stream()))
    return out


def decode_cross_attn_weights(q, kv, lens, beam, H, scale, weights):
    """decode_cross_attn (bit-identical context) that also writes weights fp32 [N, Tk] = the head-averaged fp32 softmax
    probabilities of every hypothesis (padded keys 0).  weights may be a row block of a larger history, e.g. att[step]."""
    _need_cuda(q, kv, lens, weights)
    _bf(q, kv)
    N, d = q.shape
    assert weights.dtype == torch.float32 and weights.is_contiguous() and weights.shape == (N, kv.shape[1])
    out = torch.empty_like(q)
    _lib.check(_lib.load().esp_decode_cross_attn_weights(_ptr(q), _ptr(kv), _ptr(lens), N, beam, H, d // H, kv.shape[1], scale,
                                                         _ptr(out), _ptr(weights), _stream()))
    return out


def decode_update_ancestry(anc_in, anc_out, new_order, step):
    _need_cuda(anc_in, anc_out, new_order)
    N = anc_in.shape[1]
    _lib.check(_lib.load().esp_decode_update_ancestry(_ptr(anc_in), _ptr(anc_out), _ptr(new_order), N, step, _stream()))


def decode_update_paths(cells_in, len_in, cells_out, len_out, new_order, grown, slot, pos_out=None):
    """Path tables of the frame-slot cache (include/espresso_b200.h): cells int32 [S, N], len int32 [N]; new_order, grown
    int32 [N]; pos_out int32 [N] or None receives len_in[new_order]."""
    _need_cuda(cells_in, len_in, cells_out, len_out, new_order, grown, pos_out)
    assert all(t.dtype == torch.int32 and t.is_contiguous() for t in (cells_in, len_in, cells_out, len_out, new_order, grown))
    assert 0 <= slot < cells_in.shape[0] and cells_out.shape == cells_in.shape
    N = cells_in.shape[1]
    _lib.check(_lib.load().esp_decode_update_paths(_ptr(cells_in), _ptr(len_in), _ptr(cells_out), _ptr(len_out), _ptr(pos_out),
                                                   _ptr(new_order), _ptr(grown), slot, N, _stream()))


def decode_self_attn_paths(q, kv_cache, cells, lens, H, scale):
    """q bf16 [N, d]; kv_cache bf16 [S, N, 2d] by frame slot; cells int32 [S, N], lens int32 [N] (the path tables) ->
    [N, d], hypothesis n attending over its lens[n] keys."""
    _need_cuda(q, kv_cache, cells, lens)
    _bf(q, kv_cache)
    assert cells.dtype == torch.int32 and lens.dtype == torch.int32 and cells.shape == kv_cache.shape[:2]
    N, d = q.shape
    out = torch.empty_like(q)
    _lib.check(_lib.load().esp_decode_self_attn_paths(_ptr(q), _ptr(kv_cache), _ptr(cells), _ptr(lens), kv_cache.shape[0], N, H,
                                                      d // H, scale, _ptr(out), _stream()))
    return out


# ----------------------------------------------------------------------------------------------
# transducer
# ----------------------------------------------------------------------------------------------
def joint_fwd(enc, dec):
    """enc bf16 [B, T, J], dec bf16 [B, U1, J] -> relu(enc[:, :, None] + dec[:, None]) [B, T, U1, J]."""
    _need_cuda(enc, dec)
    _bf(enc, dec)
    assert enc.is_contiguous() and dec.is_contiguous()
    B, T, J = enc.shape
    U1 = dec.shape[1]
    out = torch.empty(B, T, U1, J, device=enc.device, dtype=torch.bfloat16)
    _lib.check(_lib.load().esp_joint_fwd(_ptr(enc), _ptr(dec), B, T, U1, J, _ptr(out), _stream()))
    return out


def joint_bwd(df, f):
    """-> (denc bf16 [B, T, J], ddec fp32 [B, U1, J])."""
    _need_cuda(df, f)
    _bf(df, f)
    assert df.is_contiguous() and f.is_contiguous()
    B, T, U1, J = f.shape
    denc = torch.empty(B, T, J, device=f.device, dtype=torch.bfloat16)
    ddec = torch.zeros(B, U1, J, device=f.device, dtype=torch.float32)
    _lib.check(_lib.load().esp_joint_bwd(_ptr(df), _ptr(f), B, T, U1, J, _ptr(denc), _ptr(ddec), _stream()))
    return denc, ddec


def rnnt_loss(logits, V, t_lens, u_lens, targets, blank, grad_scale=1.0, want_grad=True):
    """logits bf16 [B, T, U1, ld]; targets int32 [B, u_max]; -> (loss fp32 [B], grad bf16 like logits or None)."""
    _need_cuda(logits, t_lens, u_lens, targets)
    _bf(logits)
    assert logits.is_contiguous() and targets.dtype == torch.int32 and t_lens.dtype == torch.int32 and u_lens.dtype == torch.int32
    B, T, U1, ld = logits.shape
    L = _lib.load()
    ws = torch.empty(int(L.esp_rnnt_workspace_bytes(B, T, U1)), device=logits.device, dtype=torch.uint8)
    loss = torch.empty(B, device=logits.device, dtype=torch.float32)
    grad = torch.empty_like(logits) if want_grad else None
    tg = targets.contiguous()
    _lib.check(L.esp_rnnt_loss(_ptr(logits), ld, V, B, T, U1, _ptr(t_lens), _ptr(u_lens), _ptr(tg), tg.shape[1], blank, grad_scale,
                               _ptr(loss), _ptr(grad), _ptr(ws), _stream()))
    return loss, grad


# ---- transducer beam search (csrc/transducer_beam.cu) ------------------------------------------------------------------
def _rnnt_beam_struct(st):
    """The EspRnntBeam view of a search-state dict (tools/transducer_beam_search_decoder.py: beam_state), built once."""
    s = st.get("_struct")
    if s is None:
        for n in _lib.EspRnntBeam.TABLES:
            t = st[n]
            _need_cuda(t)
            assert t.is_contiguous() and t.dtype == (torch.float32 if n in ("score", "a_score") else
                                                     torch.int64 if n == "p_hash" else torch.int32), n
        s = _lib.EspRnntBeam(*[int(st[n]) for n in _lib.EspRnntBeam.DIMS], *[st[n].data_ptr() for n in _lib.EspRnntBeam.TABLES])
        st["_struct"] = s
    return s


def _lm_rows(lm_logits, n):
    if lm_logits is None:
        return None, 0, 0
    _need_cuda(lm_logits)
    assert lm_logits.dim() == 2 and lm_logits.size(0) == n and lm_logits.stride(1) == 1
    assert lm_logits.dtype in (torch.float32, torch.bfloat16)
    return lm_logits, lm_logits.stride(0), int(lm_logits.dtype == torch.float32)


def rnnt_beam_lprobs(logits, V, scores, k, blank, temperature=1.0, eos=-1, fold_eos=False, lm_logits=None, lm_weight=0.0,
                     no_blank_in_lm=False):
    """Per joint row: top k of log_softmax(logits / temperature) (LM-fused, eos folded into blank) + scores[row] as
    (values fp32 [n, k], tokens int32 [n, k]), and the row's raw blank log-prob fp32 [n]."""
    _need_cuda(logits, scores)
    _bf(logits)
    assert logits.dim() == 2 and logits.stride(1) == 1 and logits.size(1) >= V
    n = logits.size(0)
    assert scores.dtype == torch.float32 and scores.is_contiguous() and scores.numel() >= n
    lm, ld_lm, lm_f32 = _lm_rows(lm_logits, n)
    val = torch.empty(n, k, device=logits.device, dtype=torch.float32)
    tok = torch.empty(n, k, device=logits.device, dtype=torch.int32)
    lpb = torch.empty(n, device=logits.device, dtype=torch.float32)
    _lib.check(_lib.load().esp_rnnt_beam_lprobs(_ptr(logits), logits.stride(0), V, n, _ptr(scores), k, blank, temperature, eos,
                                                int(fold_eos), _ptr(lm), ld_lm, lm_f32, lm_weight, int(no_blank_in_lm), _ptr(val),
                                                _ptr(tok), _ptr(lpb), _stream()))
    return val, tok, lpb


def rnnt_beam_prefix_merge(st, t, alpha):
    """Frame t's length sort and prefix pairs of every utterance still inside its frames (lists m_pair / m_ring / m_tok)."""
    assert alpha == st["alpha"]
    _lib.check(_lib.load().esp_rnnt_beam_prefix_merge(C.byref(_rnnt_beam_struct(st)), t, _stream()))


def rnnt_beam_merge_scores(logits, V, st, temperature=1.0, blank=0, lm_logits=None, lm_weight=0.0, no_blank_in_lm=False):
    """Log-adds each listed pair's path score into its longer hypothesis; logits bf16 [B * S, ld] of the path steps."""
    _need_cuda(logits)
    _bf(logits)
    assert logits.dim() == 2 and logits.stride(1) == 1 and logits.size(0) == st["B"] * st["S"] and logits.size(1) >= V
    lm, ld_lm, lm_f32 = _lm_rows(lm_logits, logits.size(0))
    _lib.check(_lib.load().esp_rnnt_beam_merge_scores(_ptr(logits), logits.stride(0), V, C.byref(_rnnt_beam_struct(st)),
                                                      temperature, blank, _ptr(lm), ld_lm, lm_f32, lm_weight, int(no_blank_in_lm),
                                                      _stream()))


def rnnt_beam_select(val, tok, lpb, st, rnd, beam, blank, gamma=None, normalize=True, final=False):
    """One expansion round (or, final, the frame's last combination) of every utterance with live rows."""
    _need_cuda(val, tok, lpb)
    BK = st["B"] * st["K"]
    assert val.dtype == torch.float32 and tok.dtype == torch.int32 and lpb.dtype == torch.float32
    assert val.shape == tok.shape and val.size(0) == BK and lpb.numel() == BK and val.is_contiguous() and tok.is_contiguous()
    assert gamma is None or gamma > 0
    _lib.check(_lib.load().esp_rnnt_beam_select(_ptr(val), _ptr(tok), val.size(1), _ptr(lpb), C.byref(_rnnt_beam_struct(st)), rnd,
                                                beam, blank, -1.0 if gamma is None else gamma, int(normalize), int(final),
                                                _stream()))


def rnnt_beam_finalize(st, pad):
    """(tokens int64 [B, K, L] pad-filled, scores fp32 [B, K] = score / (len - 1) best first, lens int32 [B, K]);
    L = the longest row (one host read of the lengths)."""
    B, K = st["B"], st["K"]
    dev = st["len"].device
    L = max(int(st["len"].max()) - 1, 1)
    tokens = torch.empty(B, K, L, device=dev, dtype=torch.int64)
    scores = torch.empty(B, K, device=dev, dtype=torch.float32)
    lens = torch.empty(B, K, device=dev, dtype=torch.int32)
    _lib.check(_lib.load().esp_rnnt_beam_finalize(C.byref(_rnnt_beam_struct(st)), L, pad, _ptr(tokens), _ptr(scores), _ptr(lens),
                                                  _stream()))
    return tokens, scores, lens
