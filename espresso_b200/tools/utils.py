"""Self-attention visibility for streaming / limited-context encoders, as per-row key RANGES; attention plots.

The reference builds [T, T] boolean masks (`chunk_streaming_mask`, espresso/tools/utils.py:131-194, and the
`transformer_context` band mask, espresso/models/transformer/speech_transformer_encoder.py:232-263) and adds -1e8 to the
masked scores (fairseq/modules/multihead_attention.py:835-839).  Both masks are contiguous per query row, so the fused
attention kernel takes two int32 vectors instead: row i may attend keys lo[i] <= j < hi[i] (csrc/attn_fused.cu)."""
import os

import numpy as np


def chunk_streaming_bounds(max_len, chunk_size, left_window=0, right_window=0, always_partial_in_last=False):
    """(lo, hi) int32 [max_len] with the reference's chunk layout, including its coin flip (np.random.rand() > 0.5, drawn
    under numpy_seed(num_updates) by the caller) between a partial FIRST and a partial LAST chunk during training."""
    starts = np.arange(0, max_len, chunk_size, dtype=np.int64)                  # e.g. [0, 18, 36, 54]
    if not always_partial_in_last and np.random.rand() > 0.5:
        starts = (max_len - starts)[::-1][:-1]
        starts = np.concatenate([[0], starts])
    start_pad = np.concatenate([[0], starts])                                   # [0, 0, 18, 36, 54]
    end_pad = np.concatenate([starts, [max_len]])                               # [0, 18, 36, 54, max_len]
    seq = np.arange(max_len)
    idx = np.nonzero((seq[:, None] >= start_pad[None]) & (seq[:, None] < end_pad[None]))[1]
    il = np.maximum(idx - left_window, 0)
    ir = np.minimum(idx + right_window, len(starts))
    return start_pad[il].astype(np.int32), end_pad[ir].astype(np.int32)


def context_bounds(max_len, left_context=None, right_context=None):
    """`transformer_context` = (left, right): row i sees keys i - left .. i + right (None = unlimited)."""
    i = np.arange(max_len)
    lo = np.zeros(max_len, dtype=np.int64) if left_context is None else np.maximum(i - left_context, 0)
    hi = np.full(max_len, max_len, dtype=np.int64) if right_context is None else np.minimum(i + right_context + 1, max_len)
    return lo.astype(np.int32), hi.astype(np.int32)


def plot_attention(attention, hypo_sent, utt_id, save_dir):
    """Save `attention` [src_len, tgt_len] as a matrix image titled with the hypothesis to <save_dir>/<utt_id>.pdf -- the
    decode script's attention plot (espresso/tools/utils.py:240-262), with the same message when matplotlib is missing."""
    try:
        import matplotlib

        matplotlib.use("Agg")  # files only, no display
        from matplotlib import pyplot
    except ImportError:
        raise ImportError("This function requires matplotlib.\nPlease install it to generate plots, or unset --print-alignment.\n"
                          "If you are on a cluster where you do not have admin rights you could try using virtualenv.")
    pyplot.matshow(attention.detach().cpu().numpy())
    pyplot.title(hypo_sent, fontsize=8)
    pyplot.savefig(os.path.join(save_dir, utt_id + ".pdf"), bbox_inches="tight")
    pyplot.close()


def bounds_to_mask(lo, hi):
    """[T, T] bool, True = visible (the reference's chunk_streaming_mask orientation)."""
    j = np.arange(len(lo))[None, :]
    return (j >= np.asarray(lo)[:, None]) & (j < np.asarray(hi)[:, None])
