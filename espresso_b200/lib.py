"""ctypes binding of libespresso_b200.so (the C ABI in include/espresso_b200.h).

The product path fails loudly when the CUDA extension is missing: there is no fallback.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libespresso_b200.so")


class EspressoB200Error(RuntimeError):
    pass


class EspGemm(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("B", C.c_void_p), ("C", C.c_void_p), ("C2", C.c_void_p),
        ("bias", C.c_void_p), ("aux", C.c_void_p), ("R", C.c_void_p),
        ("M", C.c_int64), ("N", C.c_int64), ("K", C.c_int64),
        ("lda", C.c_int64), ("ldb", C.c_int64), ("ldc", C.c_int64), ("ld_aux", C.c_int64), ("ldr", C.c_int64),
        ("sA1", C.c_int64), ("sA2", C.c_int64), ("sB1", C.c_int64), ("sB2", C.c_int64),
        ("sC1", C.c_int64), ("sC2", C.c_int64), ("sAux1", C.c_int64), ("sAux2", C.c_int64),
        ("sR1", C.c_int64), ("sR2", C.c_int64),
        ("a_kmajor", C.c_int32), ("b_kmajor", C.c_int32), ("nb1", C.c_int32), ("nb2", C.c_int32),
        ("c_f32", C.c_int32), ("r_f32", C.c_int32), ("act", C.c_int32), ("drop_mode", C.c_int32),
        ("skew_r", C.c_int32), ("tile_n", C.c_int32), ("accumulate", C.c_int32),
        ("alpha", C.c_float), ("beta", C.c_float), ("drop_p", C.c_float),
        ("seed", C.c_uint64),
        ("seed_ptr", C.c_void_p),
        ("rowsum_a", C.c_void_p), ("rowsum_scale", C.c_float),
    ]


class EspNgram(C.Structure):
    _fields_ = [
        ("word", C.c_void_p), ("prob", C.c_void_p), ("backoff", C.c_void_p), ("child_lo", C.c_void_p),
        ("child_hi", C.c_void_p), ("suffix", C.c_void_p), ("order", C.c_int32), ("order_off", C.c_int32 * 7),
        ("start", C.c_int32), ("eos", C.c_int32), ("unk", C.c_int32),
    ]


class EspArpaTables(C.Structure):
    _fields_ = [
        ("order", C.c_int32), ("count", C.c_int64 * 6), ("vocab_bytes", C.c_int64), ("unk_added", C.c_int32),
        ("word", C.c_void_p), ("prob", C.c_void_p), ("backoff", C.c_void_p), ("child_lo", C.c_void_p),
        ("child_hi", C.c_void_p), ("suffix", C.c_void_p), ("vocab", C.c_void_p),
        ("start", C.c_int32), ("eos", C.c_int32), ("unk", C.c_int32),
    ]


class EspLexicon(C.Structure):
    _fields_ = [
        ("child_off", C.c_void_p), ("child_tok", C.c_void_p), ("child_node", C.c_void_p), ("word_off", C.c_void_p),
        ("words", C.c_void_p), ("word_lm", C.c_void_p), ("smear", C.c_void_p),
        ("num_nodes", C.c_int32), ("max_words", C.c_int32),
    ]


class EspRnntBeam(C.Structure):
    DIMS = ("B", "K", "E", "A", "P", "Pm", "S", "alpha", "ring_stride")
    TABLES = ("score", "nemit", "len", "node", "srow", "fsrc", "parent", "prev", "nrow", "nlive", "nframes", "a_score",
              "a_nemit", "a_len", "a_node", "a_src", "na", "p_parent", "p_tok", "p_len", "p_hash", "npool", "m_pair",
              "m_ring", "m_tok", "m_npair")
    _fields_ = [(n, C.c_int32) for n in DIMS] + [(n, C.c_void_p) for n in TABLES]


ACT_NONE, ACT_RELU, ACT_SILU, ACT_RELU_BWD, ACT_SILU_BWD = 0, 1, 2, 3, 4

_vp, _i32, _i64, _f32, _u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_uint64

# name -> (restype, argtypes); every symbol declared in include/espresso_b200.h must appear here
SIGNATURES = {
    "esp_last_error": (C.c_char_p, []),
    "esp_version": (C.c_int, []),
    "esp_launch_count": (_i64, []),
    "esp_batch_by_size": (_i64, [_vp, _i64, _i64, _i64, _i32, _vp]),
    "esp_note_graph_replay": (None, [_i64]),
    "esp_gemm_bf16": (C.c_int, [C.POINTER(EspGemm), _vp]),
    "esp_frontend_fbank": (C.c_int, [_vp, _i32, _i64, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _i32, _vp, _i32, _i32,
                                     _vp, _vp, _vp]),
    "esp_frontend_workspace_bytes": (_i64, [_i32]),
    "esp_specaug_features": (C.c_int, [_vp, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _vp, _i32, _vp, _vp]),
    "esp_specaug_workspace_bytes": (_i64, [_i32, _i32]),
    "esp_flac_decode": (C.c_int, [_vp, _i64, _vp, _vp, _i32, _i32, _vp, _i64, _vp, _vp, _vp]),
    "esp_flac_decode_workspace_bytes": (_i64, [_i32, _i64, _i32, _i64]),
    "esp_ctc_workspace_bytes": (_i64, [_i32, _i32, _i32]),
    "esp_ctc_loss": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _f32, _vp, _vp,
                               _vp, _vp]),
    "esp_ctc_beam_workspace_bytes": (_i64, [_i32, _i32, _i32]),
    "esp_ctc_beam_frames": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp,
                                      _vp]),
    "esp_ctc_beam_search": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _f32, _i32, _i32,
                                      _vp, _i32, _i64, _i32, _i32, _f32, _f32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "esp_ctc_beam_finalize": (C.c_int, [_i32, _i32, _vp, _i32, _i32, _i32, _vp, _i32, _i64, _i32, _i32, _f32, _i32, _i32, _vp,
                                        _vp, _vp, _vp, _vp, _vp]),
    "esp_ngram_build": (C.c_int, [C.c_char_p, _i64, C.POINTER(EspArpaTables)]),
    "esp_ngram_score": (C.c_int, [C.POINTER(EspNgram), _i32, _vp, _vp, _vp, _vp, _vp]),
    "esp_ctc_ngram_workspace_bytes": (_i64, [_i32, _i32, _i32]),
    "esp_ctc_ngram_search": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _f32,
                                       C.POINTER(EspNgram), _vp, _i32, C.POINTER(EspLexicon), _f32, _f32, _vp, _vp]),
    "esp_ctc_ngram_finalize": (C.c_int, [_i32, _i32, _vp, _i32, _i32, _i32, C.POINTER(EspNgram), C.POINTER(EspLexicon), _f32,
                                         _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "esp_layer_norm_fwd": (C.c_int, [_vp, _vp, _vp, _f32, _i64, _i32, _vp, _vp, _vp, _vp, _i32, _f32, _u64, _vp, _vp]),
    "esp_layer_norm_bwd": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _i32, _f32, _u64, _vp, _vp]),
    "esp_layer_norm_bwd2": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _i32, _f32, _u64, _vp, _vp, _f32, _u64,
                                      _f32, _vp]),
    "esp_colsum": (C.c_int, [_vp, _i64, _i32, _i64, _f32, _vp, _vp]),
    "esp_dropout": (C.c_int, [_vp, _i64, _i32, _i64, _i64, _f32, _f32, _u64, _vp, _vp, _vp]),
    "esp_mask_rows": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp]),
    "esp_qprep_fwd": (C.c_int, [_vp, _i64, _vp, _vp, _f32, _i64, _i32, _vp, _vp, _vp]),
    "esp_qprep_bwd": (C.c_int, [_vp, _vp, _f32, _i64, _i32, _vp, _i64, _vp]),
    "esp_attn_fused_fwd": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp,
                                     _i64, _vp, _vp, _i32, _f32, _u64, _vp, _vp]),
    "esp_attn_fused_bwd": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _u64, _vp,
                                     _vp, _vp, _vp, _i32, _vp, _vp, _i64, _vp]),
    "esp_attn_softmax_fwd": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _i32, _vp, _i32, _vp, _vp, _f32, _u64, _vp, _vp]),
    "esp_attn_softmax_relaxed_fwd": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, C.c_double, _f32, _u64, _vp,
                                               _vp]),
    "esp_attn_softmax_bwd": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _f32, _u64, _vp, _vp]),
    "esp_glu_dwconv_fwd": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "esp_glu_dwconv_bwd": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "esp_bn_finalize": (C.c_int, [_vp, _i64, _i32, _f32, _f32, _vp, _vp, _i32, _vp, _vp]),
    "esp_bn_stats": (C.c_int, [_vp, _vp, _i64, _i32, _vp, _vp]),
    "esp_bn_act_fwd": (C.c_int, [_vp, _vp, _i64, _i32, _vp, _vp, _vp, _i32, _vp, _vp]),
    "esp_bn_act_bwd": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "esp_conv3x3_fwd": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "esp_conv3x3_dgrad": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "esp_conv3x3_wgrad": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "esp_conv3x3_c1_fwd": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "esp_conv3x3_c1_wgrad": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "esp_lsce_loss": (C.c_int, [_vp, _i64, _i32, _i64, _vp, _i32, _f32, _i32, _vp, _i32, _f32, _vp, _vp, _vp, _vp]),
    "esp_embed_fwd": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _f32, _i64, _i32, _vp, _f32, _u64, _vp, _vp]),
    "esp_embed_bwd": (C.c_int, [_vp, _vp, _i32, _f32, _i64, _i32, _vp, _f32, _u64, _vp, _vp]),
    "esp_argmax_rows": (C.c_int, [_vp, _i64, _i32, _i64, _vp, _vp]),
    "esp_beam_merge": (C.c_int, [_vp, _i32, _i64, _i32, _f32, _vp, _i32, _i64, _i32, _f32, _i32, _i32, _vp, _i32, _i32, _f32, _i32,
                                 _i32, _i32, _f32, _i32, _vp, _vp]),
    "esp_beam_topk": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "esp_beam_bookkeep": (C.c_int, [_i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _f32] + [_vp] * 17),
    "esp_beam_bookkeep_attn": (C.c_int, [_i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _f32] + [_vp] * 18 + [_i32, _vp, _vp]),
    "esp_gather_rows": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp]),
    "esp_beam_block_ngrams": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _vp, _i64, _i32, _vp]),
    "esp_beam_prefix": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _i32, _vp, _i32, _vp, _vp]),
    "esp_beam_diverse_groups": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp]),
    "esp_beam_sibling_topk": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "esp_beam_sample": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _i32, _vp, _vp, _vp, _vp]),
    "esp_lookahead_words": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "esp_wordlm_cumsum": (C.c_int, [_vp, _i32, _i64, _i32, _i32, _vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _i32, _vp]),
    "esp_multilevel_step": (C.c_int, [_vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _i32, _i64, _i32, _f32, _vp, _vp, _vp,
                                      _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _i32, _f32, _vp, _i64, _i32, _vp]),
    "esp_lookahead_step": (C.c_int, [_vp, _i64, _i32, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32,
                                     _i32, _f32, _i32, _f32, _vp, _i64, _i32, _vp]),
    "esp_decode_self_attn": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _vp]),
    "esp_decode_cross_attn": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp, _vp]),
    "esp_decode_cross_attn_weights": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _vp, _vp, _vp]),
    "esp_decode_update_ancestry": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _vp]),
    "esp_decode_update_paths": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp]),
    "esp_decode_self_attn_paths": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _vp]),
    "esp_rnnt_beam_lprobs": (C.c_int, [_vp, _i64, _i32, _i32, _vp, _i32, _i32, _f32, _i32, _i32, _vp, _i64, _i32, _f32, _i32, _vp,
                                       _vp, _vp, _vp]),
    "esp_rnnt_beam_prefix_merge": (C.c_int, [C.POINTER(EspRnntBeam), _i32, _vp]),
    "esp_rnnt_beam_merge_scores": (C.c_int, [_vp, _i64, _i32, C.POINTER(EspRnntBeam), _f32, _i32, _vp, _i64, _i32, _f32, _i32,
                                             _vp]),
    "esp_rnnt_beam_select": (C.c_int, [_vp, _vp, _i32, _vp, C.POINTER(EspRnntBeam), _i32, _i32, _i32, _f32, _i32, _i32, _vp]),
    "esp_rnnt_beam_finalize": (C.c_int, [C.POINTER(EspRnntBeam), _i32, _i32, _vp, _vp, _vp, _vp]),
    "esp_joint_fwd": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "esp_joint_bwd": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "esp_rnnt_workspace_bytes": (_i64, [_i32, _i32, _i32]),
    "esp_rnnt_loss": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp]),
    "esp_sumsq_f32": (C.c_int, [_vp, _i64, _vp, _vp]),
    "esp_adam_step": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _f32, _f32, _i32, _vp, _vp, _f32, _f32,
                                _vp, _vp, _vp]),
    "esp_cast_f32_bf16": (C.c_int, [_vp, _i64, _vp, _vp]),
    "esp_cast_bf16_f32": (C.c_int, [_vp, _i64, _vp, _vp]),
}

_lib = None


def load():
    """Load libespresso_b200.so and bind every entry point.  Raises if the library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EspressoB200Error(
            "libespresso_b200.so not found at %s -- build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (or `make -C espresso_b200/csrc`).  There is no CPU fallback." % LIB_PATH
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError => header/library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise EspressoB200Error("espresso_b200 native call failed (%d): %s" % (rc, load().esp_last_error().decode()))


def launch_count():
    return int(load().esp_launch_count())
