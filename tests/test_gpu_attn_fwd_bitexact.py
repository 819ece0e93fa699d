"""GPU: the fused relative-position attention forward (csrc/attn_fused.cu) reproduces pinned outputs bit for bit.

The kernel's arithmetic per output element is fixed by its wgmma shapes, the order of its sums and its rounding points,
so a rework of its schedule must not move a single bit of ctx, P or Pd (the padding columns [T, ld) of P / Pd
included).  Inputs come from CPU generators, so the digests do not depend on the GPU's RNG; each case hashes the bytes
of ctx, P and Pd with SHA-256.  The digests were recorded with the kernel as it was before its Hopper rework (288
threads, W halves recomputed per key tile) and were stable across repeated runs."""
import hashlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# name: (B, T, H, lens, key bounds (chunk, left, right) or None, shared position table, dropout, device seed, save_probs)
CASES = {
    "bench_15x431": (15, 431, 8, "ragged", None, False, 0.0, None, True),
    "bench_15x431_drop": (15, 431, 8, "ragged", None, False, 0.1, None, True),
    "bench_24x250": (24, 250, 8, "ragged", None, False, 0.0, None, True),
    "bench_24x250_drop": (24, 250, 8, "ragged", None, False, 0.1, None, True),
    "bench_8x754": (8, 754, 8, "ragged", None, False, 0.0, None, True),
    "bench_8x754_drop": (8, 754, 8, "ragged", None, False, 0.1, None, True),
    "t1": (3, 1, 2, None, None, False, 0.0, None, True),
    "t127": (3, 127, 2, "ragged", None, False, 0.0, None, True),
    "t128": (3, 128, 2, "ragged", None, False, 0.0, None, True),
    "t129": (3, 129, 2, "ragged", None, False, 0.0, None, True),
    "t300": (3, 300, 4, "ragged", None, False, 0.0, None, True),
    "chunks_203": (2, 203, 2, "ragged", (16, 1, 0), False, 0.0, None, True),
    "chunks_407": (3, 407, 2, "ragged", (40, 2, 1), False, 0.0, None, True),
    "chunks_90_padded_rows": (2, 90, 2, "ragged", (30, 0, 0), False, 0.0, None, True),
    "shared_pos_200": (2, 200, 4, "ragged", None, True, 0.0, None, True),
    "drop_device_seed_300": (2, 300, 8, "ragged", None, False, 0.1, 2 ** 64 - 5, True),
    "drop_chunks_407": (3, 407, 2, "ragged", (40, 2, 1), False, 0.1, 12345, True),
    "inference_431": (15, 431, 8, "ragged", None, False, 0.0, None, False),
    "inference_drop_300": (2, 300, 8, "ragged", None, False, 0.1, None, False),
}

DIGESTS = {
    "bench_15x431": ("0b96b7f56c6659df16a57600dbdf7f83a77c99ad7bd3c0a69570089a5846207e",
        "eeccf3f06fc9302c63632817f0e8ad7165565c3ca364d5279fec5a3610c99b30",
        "-"),
    "bench_15x431_drop": ("5bbf553aeb071c71a17399c8ee0451277aa75427f8fca2a8a095326a8744aa61",
        "eeccf3f06fc9302c63632817f0e8ad7165565c3ca364d5279fec5a3610c99b30",
        "425a3dc29fc08880e19dd0c655339195a85e64de831fafb351549c138e94cad1"),
    "bench_24x250": ("cf9df7bf963bbfc612e919be2fabbab3ff6bd169ba5379c5c25f3ad94989be25",
        "d220aca9ce5564f7d2769b59edec2dafd9799bdf794d65931ba06e6131c5bcad",
        "-"),
    "bench_24x250_drop": ("1ed209ca33a2ef333d02702fa8649a1f8507be32291808d0878215731e4c88a1",
        "d220aca9ce5564f7d2769b59edec2dafd9799bdf794d65931ba06e6131c5bcad",
        "9385d32898a7f661ff311b07a1f0f25643444cf991f148ef7f9cd02492a751ad"),
    "bench_8x754": ("47dce41780a8bbea09aeaced3e0d09dc22fc137372cd28f707f8b563298afd3a",
        "678735466a46aec978281cd1b340724fbc91f9aac20f212f29301b96ecd71061",
        "-"),
    "bench_8x754_drop": ("4f6a804de0ce0f5c6b094670473dcbaca4a347fc0a95bcd06708b9e53e57c564",
        "678735466a46aec978281cd1b340724fbc91f9aac20f212f29301b96ecd71061",
        "ad752a9732988a3b81c7131b5950846d4d68f12b550fa689a51abd57f36b999e"),
    "chunks_203": ("b80fe6362a15c7519457a46b065a6f00b651c69b1a34f5c574dea0607220f924",
        "728ca72766cad835b064db0da195422b5806b5c1de065a74ef64aec02203cf6f",
        "-"),
    "chunks_407": ("a4a3f96d218f67c14502d2c154bafeaddcd88520ae5cc7df313f726880ad2099",
        "84270aad2ca813307400c6709fc687c80193f4bdf24b86c3b58a44dac3e8def2",
        "-"),
    "chunks_90_padded_rows": ("f904521f2665c0268f22eb8b97c6fa6bc4c4bdcbae2aecce7b1d8b5b9206ea72",
        "3c499b4315b8dfb53e01c06f2997529f0d4aec040da41f29ab6d371c4be0488a",
        "-"),
    "drop_chunks_407": ("836d05c45b7aaf44235ba23ae040a938499dc84dd0119c24bd8da262b5d87dbd",
        "84270aad2ca813307400c6709fc687c80193f4bdf24b86c3b58a44dac3e8def2",
        "bf63ea985d44a39ad6f301f271f31533cb488c272bb09a55976ff0f7405a8a75"),
    "drop_device_seed_300": ("61d8b83986dde421f4edf148e2e6d00965bdc934657e3e248e27b128ebe051ef",
        "746cc921ad1abb36750774e500285f77417427f9f455d3419456bdf1d82316bb",
        "08b9d89813834d588e74b4f4e0cbc0b8e884884861148c56f7cb91cdc754b411"),
    "inference_431": ("0b96b7f56c6659df16a57600dbdf7f83a77c99ad7bd3c0a69570089a5846207e",
        "-",
        "-"),
    "inference_drop_300": ("14fdcf1780b9304ba299988ccfa618f2d859d451dab75f89f6b20a532ed63f03",
        "-",
        "-"),
    "shared_pos_200": ("d8f4e8bf63c130d2130a8d885541b2ac82f51b2c2f87335b3ef5f6bcd3975888",
        "481aead584b1c94a32521b5294056653245cf9aa294972b6ba787254e04a15af",
        "-"),
    "t1": ("a18bb0928300fd182551c26990bb87f4e0cba111ce55df2b6493ab72242fe1a6",
        "9651d66e0f905325f44cad139e86820df53e88f37e16d39fefc99810d7aa974d",
        "-"),
    "t127": ("5e2f0aad81db21c841f7f0aae8281d05d9620f35f24b16d136efdb3bc275099a",
        "03489fedb024c357de2d12e60924ec8425c55182cfabc585b7aafbc4d36d796a",
        "-"),
    "t128": ("bb5b61dfca9415605649253e99cafa33d9ca5fbac66a21b36afdd476a3138600",
        "b4c44e395ef53e7e61fbfbbdd8afea0af1f20c6affa2681b782087fd581239a6",
        "-"),
    "t129": ("95cb8f5cbb6941b2ccb2f13b789b708f79ce6bb49fb1cb9f3ecdc8223cb7d8c8",
        "34f1c3b97e762462f469af84911d68734a5624d0c68c6db980d9e1038dbc6bdf",
        "-"),
    "t300": ("bf5c171f5cba70475917e01804aeec0159a74d54eabaf010959ca943cf4d0104",
        "2be4c8297ba0c9e50f97e6549999a977d19a53e3bfcbca43fd5266f31668bc21",
        "-"),
}


def _bytes(t):
    return t.contiguous().view(torch.int16).cpu().numpy().tobytes()


def run_case(name, dev):
    """SHA-256 hex digests of (ctx, P, Pd) for case `name` ("-" for an output the case does not produce)."""
    from espresso_b200 import ops
    from espresso_b200.tools.utils import chunk_streaming_bounds

    B, T, H, lens, kb, shared, drop, dseed, save = CASES[name]
    d = H * 64
    g = torch.Generator(device="cpu").manual_seed(1000 * T + B)
    qkv = (torch.randn(B * T, 3 * d, generator=g) * 0.7).bfloat16()
    qu = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16()
    qv = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16()
    pos = (torch.randn(2 * T - 1, 64 if shared else d, generator=g) * 0.7).bfloat16()
    lens_t = None
    if lens == "ragged":
        ln = torch.randint(max(1, T // 3), T + 1, (B,), generator=g, dtype=torch.int32)
        ln[0] = T
        lens_t = ln.to(dev)
    bounds = None
    if kb is not None:
        lo, hi = chunk_streaming_bounds(T, *kb, always_partial_in_last=True)
        bounds = (torch.from_numpy(lo.astype(np.int32)).to(dev), torch.from_numpy(hi.astype(np.int32)).to(dev))
    qkv = qkv.to(dev)
    ops.set_seed_tensor(None if dseed is None else
                        torch.tensor([dseed - 2 ** 64 if dseed >= 2 ** 63 else dseed], dtype=torch.int64, device=dev))
    try:
        ctx, p, pd = ops.attn_fused_fwd(qu.to(dev), qv.to(dev), qkv[:, d:2 * d], qkv[:, 2 * d:], pos.to(dev), B, T, H,
                                        lens_t, drop_p=drop, seed=777, save_probs=save, key_bounds=bounds)
        torch.cuda.synchronize()
    finally:
        ops.set_seed_tensor(None)
    out = [hashlib.sha256(_bytes(ctx)).hexdigest()]
    out.append(hashlib.sha256(_bytes(p)).hexdigest() if p is not None else "-")
    out.append(hashlib.sha256(_bytes(pd)).hexdigest() if (pd is not None and drop > 0) else "-")
    return tuple(out)


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.mark.parametrize("name", sorted(CASES))
def test_attn_fused_fwd_bitexact(dev, name):
    assert run_case(name, dev) == DIGESTS[name]
