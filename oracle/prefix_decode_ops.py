"""Oracle: plain-PyTorch statement of the prefix-decoding ops in espresso_b200/ops.py (decode_update_paths,
decode_self_attn_paths), same signatures, fp32 arithmetic.

TEST INFRASTRUCTURE ONLY.  GPU tests compare the kernels with these; CPU tests monkeypatch them in for
`espresso_b200.ops` (next to oracle/ops_ref.py) to run the frame-slot KV cache of IncrementalDecoder and the CTC decoder's
Transformer-LM loop without a GPU.  The statement is the one in include/espresso_b200.h: a cache indexed by frame slot,
and per hypothesis the flat cells slot * N + row of its keys."""
import torch

BF = torch.bfloat16


def decode_update_paths(cells_in, len_in, cells_out, len_out, new_order, grown, slot, pos_out=None):
    """p = new_order[n]: cells_out[i][n] = cells_in[i][p] for i < len_in[p]; cells_out[len_in[p]][n] = slot * N + n when
    grown[n]; len_out[n] = len_in[p] + grown[n]; pos_out[n] = len_in[p].  Cells at and past len_out[n] are not written."""
    N = cells_in.shape[1]
    p = new_order.long()
    L = len_in.long()[p]
    g = (grown != 0).long()
    copy = torch.arange(slot + 1)[:, None] < L[None, :]
    cells_out[: slot + 1] = torch.where(copy, cells_in[: slot + 1][:, p], cells_out[: slot + 1])
    rows = torch.arange(N)[g.bool()]
    cells_out[L[rows], rows] = (slot * N + rows).to(cells_out.dtype)
    len_out.copy_((L + g).to(len_out.dtype))
    if pos_out is not None:
        pos_out.copy_(L.to(pos_out.dtype))


def decode_self_attn_paths(q, kv_cache, cells, lens, H, scale):
    """Hypothesis n attends over the K/V at flat cells cells[:lens[n], n] of kv_cache [S, N, 2d] (softmax in fp32, the
    probabilities rounded to bf16 before P.V, as esp_decode_self_attn); lens[n] = 0 gives zeros."""
    N, d = q.shape
    hd = d // H
    flat = kv_cache.float().reshape(-1, 2 * d)
    out = torch.zeros(N, d)
    for n in range(N):
        L = int(lens[n])
        if L == 0:
            continue
        kvs = flat[cells[:L, n].long()]  # [L, 2d]
        k = kvs[:, :d].reshape(L, H, hd)
        v = kvs[:, d:].reshape(L, H, hd)
        s = torch.einsum("hc,thc->ht", q[n].float().reshape(H, hd), k) * scale
        p = torch.softmax(s, dim=-1).to(BF).float()
        out[n] = torch.einsum("ht,thc->hc", p, v).reshape(d)
    return out.to(BF)
