/* espresso_b200 -- C ABI of the H100-native Espresso hot path (libespresso_b200.so).
 *
 * Conventions (SURVEY.md §8b "What the C-ABI replacement exports"):
 *  - plain C: raw DEVICE pointers, explicit sizes/strides (in ELEMENTS unless noted), no torch types;
 *  - the caller owns all memory (the library never allocates or frees device memory);
 *  - every entry point launches asynchronously on `stream` (a cudaStream_t passed as void*);
 *  - return 0 on success, negative on error; esp_last_error() returns a thread-local message;
 *  - no global mutable state apart from cached device attributes / kernel attributes.
 *
 * Each entry point cites the reference call site it replaces (paths relative to the
 * freewym/espresso tree).  The reference reaches native code through pybind11 torch extensions
 * (fairseq/clib/cuda/ngram_repeat_block_cuda.cpp:22-55); INTEGRATION.md shows the ctypes stub a
 * maintainer would add instead.
 */
#ifndef ESPRESSO_B200_H_
#define ESPRESSO_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- library ------------------------------------------------------------------------------ */
const char* esp_last_error(void);
int esp_version(void);
/* number of kernel launches issued through this library since load (for bench gpu_launches) */
int64_t esp_launch_count(void);
/* a CUDA graph captured from this library's launches was replayed: credit the kernels it contains */
void esp_note_graph_replay(int64_t launches);

/* ---- dense contraction: C = epi(op(A) * op(B)^T), bf16 in, fp32 accumulate (wgmma + TMA) -----
 * replaces torch.nn.functional.linear / torch.bmm call sites:
 *   fairseq/modules/conformer_layer.py:134-146,79-101; fairseq/modules/multihead_attention.py:650-653,
 *   788,799-823,897-907; espresso/models/transformer/speech_transformer_encoder.py:341-343;
 *   espresso/models/transformer/speech_transformer_encoder_model.py:207-208.
 * A is logically [M,K]: a_kmajor=1 -> A[m*lda+k]; a_kmajor=0 -> A[k*lda+m].
 * B is logically [N,K]: b_kmajor=1 -> B[n*ldb+k]; b_kmajor=0 -> B[k*ldb+n].
 * Two batch dims (nb1 fastest) with per-operand strides; stride 0 broadcasts the operand.
 * Epilogue, in order: +bias[n]; C2=bf16(pre-activation); dropout(mode 2); activation
 * (ESP_ACT_*; *_BWD multiply by act'(aux)); dropout(mode 1); *alpha; +beta*R (R optionally read with
 * the Transformer-XL skew R[m,(skew_r-1)-m+n]); store bf16 or fp32.  With `accumulate`, the epilogue is
 * C(fp32) += alpha*acc only (atomic, split-K); `rowsum_a` adds the bias gradient of the same layer for free.
 * Dropout is a stateless counter RNG keyed by (seed, logical element index): the backward pass
 * regenerates the forward mask, nothing is stored. */
enum { ESP_ACT_NONE = 0, ESP_ACT_RELU = 1, ESP_ACT_SILU = 2, ESP_ACT_RELU_BWD = 3, ESP_ACT_SILU_BWD = 4 };

typedef struct EspGemm {
  const void* A;
  const void* B;
  void* C;
  void* C2;          /* optional bf16 [M,N] (same ld/strides as C): value before activation */
  const void* bias;  /* optional bf16 [N] */
  const void* aux;   /* bf16, saved pre-activation for *_BWD */
  const void* R;     /* optional residual, bf16 or fp32 (r_f32) */
  int64_t M, N, K;
  int64_t lda, ldb, ldc, ld_aux, ldr;
  int64_t sA1, sA2, sB1, sB2, sC1, sC2, sAux1, sAux2, sR1, sR2;
  int32_t a_kmajor, b_kmajor;
  int32_t nb1, nb2;
  int32_t c_f32, r_f32;
  int32_t act;
  int32_t drop_mode; /* 0 none, 1 after activation (forward), 2 before activation (backward) */
  int32_t skew_r;    /* 0, or T: read R with relative-position skew */
  int32_t tile_n;    /* 0 auto, or 64/128: tile width (other values are refused); 2-CTA clusters follow from the shape */
  int32_t accumulate; /* 1: C (fp32) += alpha*acc with L2 vector reductions; enables split-K (weight gradients) */
  float alpha, beta, drop_p;
  uint64_t seed;
  const uint64_t* seed_ptr; /* optional DEVICE pointer: effective seed = seed + *seed_ptr (CUDA-graph replays) */
  float* rowsum_a;   /* optional fp32 [M] (weight-gradient GEMMs: a_kmajor = 0, accumulate = 1, no batch dims):
                        rowsum_a[m] += rowsum_scale * sum_k A[m, k] -- with A = dy^T this is the BIAS gradient, computed
                        from the operand tiles already staged in shared memory by otherwise idle warps */
  float rowsum_scale;
} EspGemm;

int esp_gemm_bf16(const EspGemm* g, void* stream);

/* ---- fused front end: framing -> DC removal -> pre-emphasis -> Povey window -> 512-pt rFFT ->
 *      power -> 80 mel -> log -> global CMVN -> adaptive SpecAugment, batched on device ---------
 * replaces espresso/data/feat_text_dataset.py:128-161 (per-utterance CPU path):
 *   espresso/tools/utils.py:426-454 -> torchaudio/compliance/kaldi.py:514-646 (fbank defaults),
 *   fairseq/data/audio/feature_transforms/global_cmvn.py:26-29,
 *   espresso/data/feature_transforms/adaptive_specaugment.py:77-136 (mask draws stay on the host
 *   with the reference's NumPy RNG; only the descriptors are uploaded).
 * wave: [B, wave_ld] samples in int16 range (fp32, or int16 if wave_i16), right padded.
 * n_samples[b]: valid samples.  frames m_b = 1 + (n-400)/160 (0 if n < 400).
 * cmvn_mean/cmvn_std: fp32[80] or NULL (no CMVN).
 * freq_masks: int32 [B, n_freq_masks, 2] = (f0, f); time_masks: int32 [B, max_time_masks, 2] = (t0, t);
 *   a mask with width 0 is a no-op.  Fill value = mean of the utterance's CMVN'd features
 *   (adaptive_specaugment.py:83-86).  Pass NULL / 0 for no SpecAugment (validation / decoding).
 * out: [B, t_max, 80] (bf16, or fp32 if out_f32), frames >= m_b are zero (collate pad value 0.0,
 *   espresso/tools/utils.py:97-113).  out_lens: int32[B] = m_b.
 * workspace: >= B*16 bytes, zero-initialised by the caller is NOT required (the kernel resets it). */
int esp_frontend_fbank(const void* wave, int32_t wave_i16, int64_t wave_ld, const int32_t* n_samples,
                       int32_t B, const float* cmvn_mean, const float* cmvn_std,
                       const int32_t* freq_masks, int32_t n_freq_masks, const int32_t* time_masks,
                       int32_t max_time_masks, void* out, int32_t out_f32, int32_t t_max,
                       int32_t* out_lens, void* workspace, void* stream);
int64_t esp_frontend_workspace_bytes(int32_t B);

/* ---- adaptive SpecAugment on features: time warp -> frequency masks -> time masks --------------
 * replaces espresso/data/feature_transforms/adaptive_specaugment.py:77-136 as
 *   espresso/data/feat_text_dataset.py:128-161 applies it to Kaldi features and to computed fbanks alike
 *   (draws stay on the host with the reference's NumPy RNG; only the descriptors are uploaded).
 * in: [B, T, F] (fp32 if in_f32, else bf16), contiguous, right padded; any F >= 1.  lens: int32 [B] frames m_b
 *   (clamped to [0, T]).  out: a separate [B, T, F] buffer (fp32 if out_f32, else bf16); frames >= m_b are zero.
 * time_warp: int32 [B, 2] = (w0, w) or NULL: frames [0, w0) are resized to w0 + w rows and [w0, m) to m - w0 - w rows
 *   along time with cv2.resize's INTER_LINEAR rule (adaptive_specaugment.py:94-109; stated in csrc/specaug.cu).
 *   w = 0 leaves the utterance unchanged, as does a pair without 0 < w0 < m and 0 < w0 + w < m.
 * freq_masks: int32 [B, n_freq_masks, 2] = (f0, f); time_masks: int32 [B, max_time_masks, 2] = (t0, t), applied
 *   after the warp; width 0 is a no-op; at most 64 of each.  Fill value = mean of the utterance's m_b x F input values
 *   before the warp (adaptive_specaugment.py:83-86), summed in double in a fixed order: the result is deterministic.
 * workspace: >= esp_specaug_workspace_bytes(B, T) bytes when masks are given (no initialisation needed), else unused.
 * Launches 1 kernel, or 2 with masks. */
int esp_specaug_features(const void* in, int32_t in_f32, void* out, int32_t out_f32, int32_t B, int32_t T, int32_t F,
                         const int32_t* lens, const int32_t* time_warp, const int32_t* freq_masks,
                         int32_t n_freq_masks, const int32_t* time_masks, int32_t max_time_masks, void* workspace,
                         void* stream);
int64_t esp_specaug_workspace_bytes(int32_t B, int32_t T);

/* ---- FLAC decoding (RFC 9639) of a batch of streams into the front end's waveform layout -----------
 * replaces fairseq/data/audio/audio_utils.py:69-126 get_waveform(normalization=False) on .flac files (libsndfile):
 *   out[b, i] = s / 2^(bps-1) * 2^15 for a mono stream; for C channels each
 *   channel is scaled the same way and the C values are added in channel order and divided by C, all in float32 (the
 *   channel mean of the WAVE path).  Bit depths 4-24, 1-8 channels, every channel assignment, fixed and variable
 *   blocking, block sizes up to 65535, CONSTANT / VERBATIM / FIXED / LPC subframes with wasted bits, Rice and Rice2
 *   residuals with escaped partitions.
 * bytes: the streams' frames, stream b in [offsets[b], offsets[b+1]) starting at its first frame (metadata blocks
 *   stripped); offsets: int64 [B+1], non-decreasing; n_bytes = offsets[B] < 2^31.
 * params: int64 [B, 5] = (total samples, sample rate, channels, bits per sample, max block size) from STREAMINFO.
 * out: float32 [B, ld]: samples [0, total_b) of every decoded stream, zeros after them; a stream whose status is not
 *   ESP_FLAC_OK reads as zeros.  Nothing outside [B, ld] is written.
 * status: int32 [B], one ESP_FLAC_* per stream.  A frame counts only on the chain that starts at the stream's first
 *   byte: each frame begins where the previous one's CRC-16 ends and continues its sample numbers, and the chain covers
 *   exactly `total` samples; a sync code inside frame data never reaches `out`.
 * workspace: >= esp_flac_decode_workspace_bytes(B, n_bytes, max_channels, ld) (no initialisation needed), where
 *   max_channels >= every stream's channel count.  Launches 4 kernels (after one 4-byte memset). */
enum {
  ESP_FLAC_OK = 0,
  ESP_FLAC_BAD_PARAMS = 1,    /* unsupported stream: total 0 or > ld, channels outside [1, max_channels], bps outside [4, 24] */
  ESP_FLAC_NO_FRAME = 2,      /* no frame header (valid CRC-8, matching STREAMINFO) where the previous frame ended */
  ESP_FLAC_BAD_SEQUENCE = 3,  /* a frame's first sample is not where the previous frame ended, or it passes the total */
  ESP_FLAC_CRC16 = 4,         /* frame CRC-16 mismatch */
  ESP_FLAC_RESERVED = 5,      /* reserved or invalid code in a subframe, residual or frame padding */
  ESP_FLAC_LPC_SHIFT = 6,     /* negative LPC quantisation shift */
  ESP_FLAC_TRUNCATED = 7      /* a frame runs past the end of its stream's bytes */
};
int esp_flac_decode(const void* bytes, int64_t n_bytes, const int64_t* offsets, const int64_t* params, int32_t B,
                    int32_t max_channels, float* out, int64_t ld, int32_t* status, void* workspace, void* stream);
int64_t esp_flac_decode_workspace_bytes(int32_t B, int64_t n_bytes, int32_t max_channels, int64_t ld);

/* ---- CTC loss forward+backward fused with the fp32 log-softmax ---------------------------------
 * replaces espresso/criterions/ctc_loss.py:59-103 = get_normalized_probs (fp32 log_softmax,
 *   espresso/models/transformer/speech_transformer_encoder_model.py:141-150) + F.ctc_loss(reduction
 *   ="sum", zero_infinity) with cuDNN disabled, and their autograd backward.
 * logits: bf16 [.., V] addressed as logits[b*stride_b + t*stride_t + v]; in_lens int32[B];
 * targets: int32 [B, u_max] (pad ignored beyond tgt_lens[b]); blank index.
 * loss: fp32[B] per-utterance negative log-likelihood (0 where infinite and zero_infinity);
 * grad: bf16, same addressing as logits; = grad_scale * d(sum_b loss_b)/d logits; rows t>=in_lens[b]
 *   are written as zero.  Columns written per row (b < B, t < t_max): [0, ld_pad), where ld_pad = ceil8(V) when the
 *   row strides of the axes longer than one (both strides when B = t_max = 1) are >= ceil8(V), else V; columns
 *   [V, ld_pad) are zero, nothing else is written.  Any base alignment and strides.  Pass grad=NULL for loss only.
 * workspace: esp_ctc_workspace_bytes(B, t_max, u_max). */
int64_t esp_ctc_workspace_bytes(int32_t B, int32_t t_max, int32_t u_max);
int esp_ctc_loss(const void* logits, int64_t stride_b, int64_t stride_t, int32_t V, int32_t B,
                 int32_t t_max, const int32_t* in_lens, const int32_t* targets, int32_t u_max,
                 const int32_t* tgt_lens, int32_t blank, int32_t zero_infinity, float grad_scale,
                 float* loss, void* grad, void* workspace, void* stream);

/* ---- CTC prefix beam search with optional LSTM-LM shallow fusion ---------------------------------------
 * replaces the beam / LM path of espresso/tools/ctc_decoder.py:18-188 (flashlight LexiconFreeDecoder + KenLM there).
 * Frame-synchronous prefix beam search per sentence over t < in_lens[b], fp32 log space.  A hypothesis holds a prefix y,
 * pb / pnb (log-prob of ending in blank / non-blank) and lm (sum of lm_weight * log P_LM(v | prefix) + word_score per
 * token); score = logaddexp(pb, pnb) + lm.  Per frame (lp = log_softmax(logits[b, t, :V])):
 *   stay:   pb' = lae(pb, pnb) + lp[blank], pnb' = pnb + lp[last(y)] (y non-empty);
 *   extend: with each of the frame's top-K tokens v: ext = (v == last(y) ? pb : lae(pb, pnb)) + lp[v] -> prefix y+v
 *           (pnb = ext, pb = -inf); if y+v is already a live hypothesis, ext is log-added into its stay pnb' instead;
 *   prune:  candidates below best - beam_threshold are dropped, the best `beam` are kept, ordered by (score desc,
 *           candidate index asc), candidate index = h * (K + 1) + j (j = 0 stay of slot h, j = 1..K its extensions in
 *           token-rank order).  Slot k of the next frame holds the k-th kept candidate; slots beyond are dead (-inf).
 * frames: per row (b, t < in_lens[b]): lse = log-normaliser, lp_blank, and the K best tokens other than blank / pad /
 *   eos / unk (pass -1 to allow one) ranked by (logit desc, token id asc), with their lp: top_tok / top_lp [B, t_max, K]
 *   (-1 / -inf where fewer tokens are allowed).  logits addressed like esp_ctc_loss.  V <= 65535.
 * search: frames [t0, t1) of every sentence (t0 == 0 starts from the empty prefix).  lm (optional): per slot the LM
 *   logits [B * beam, ld_lm] (bf16, or fp32 with lm_f32) given the slot's prefix; the kernel log-softmaxes them in
 *   fp32.  lm_blank >= 0 says the LM vocabulary lacks the blank at that index (V_lm = V - 1; LM column = v - (v >
 *   lm_blank)).  Per slot of the last frame: new_order = source row (b * beam + slot), grown = 1 when a token was
 *   appended, fed = that token (else eos) in LM indexing; slots of sentences past their end keep their row.
 *   new_order / grown / fed may be NULL (no LM).  beam, K <= 128.
 * finalize: + lm_weight * log P_LM(eos | y) when lm is given, sort by (score desc, slot asc), then per sentence the
 *   `nbest` best: out_tokens [B, nbest, t_max] (pad-filled), out_len, out_scores (natural log; -inf for missing
 *   hypotheses) and optionally out_frames [B, nbest, t_max] = the frame at which each token entered the prefix.
 * workspace: esp_ctc_beam_workspace_bytes(B, t_max, beam), carried from search to finalize. */
int64_t esp_ctc_beam_workspace_bytes(int32_t B, int32_t t_max, int32_t beam);
int esp_ctc_beam_frames(const void* logits, int64_t stride_b, int64_t stride_t, int32_t V, int32_t B, int32_t t_max,
                        const int32_t* in_lens, int32_t K, int32_t blank, int32_t pad, int32_t eos, int32_t unk, float* lse,
                        float* lp_blank, int32_t* top_tok, float* top_lp, void* stream);
int esp_ctc_beam_search(const void* logits, int64_t stride_b, int64_t stride_t, int32_t V, int32_t B, int32_t t_max,
                        const int32_t* in_lens, const float* lse, const float* lp_blank, const int32_t* top_tok,
                        const float* top_lp, int32_t K, int32_t beam, float beam_threshold, int32_t t0, int32_t t1,
                        const void* lm, int32_t lm_f32, int64_t ld_lm, int32_t V_lm, int32_t lm_blank, float lm_weight,
                        float word_score, int32_t eos, int32_t* new_order, int32_t* grown, int32_t* fed, void* workspace,
                        void* stream);
int esp_ctc_beam_finalize(int32_t B, int32_t t_max, const int32_t* in_lens, int32_t V, int32_t beam, int32_t nbest,
                          const void* lm, int32_t lm_f32, int64_t ld_lm, int32_t V_lm, int32_t lm_blank, float lm_weight,
                          int32_t eos, int32_t pad, void* workspace, int32_t* out_tokens, int32_t* out_len,
                          float* out_scores, int32_t* out_frames, void* stream);

/* ---- ARPA n-gram language models and CTC prefix beam search fused with them ------------------------
 * replaces the KenLM path of espresso/tools/ctc_decoder.py:22-73 (flashlight's LexiconDecoder / LexiconFreeDecoder with
 * a KenLM model).  Scores are log10, KenLM's unit, so lm_weight / word_score tuned with the reference carry over;
 * flashlight's KenLM wrapper passes them on unscaled (that comes from flashlight's source, not in the reference tree).
 *
 * Tables: the entries of order n (1..order) are stored at [order_off[n-1], order_off[n]) sorted by (context entry, word
 * id), so a 1-gram's entry index is its word id.  Per entry: word id, log10 prob, log10 backoff (0 at the highest
 * order), its children [child_lo, child_hi) in the next order (sorted by word id) and suffix = the entry of its longest
 * listed proper suffix (-1: the empty context).  A state is one entry index (-1 = empty context): the longest listed
 * suffix of the word history, of order < `order`.  To score word w from state s: walk s and its suffix links; at each
 * entry look for child w; the first hit c gives log10 p = (sum of the backoffs of the entries passed) + prob(c); at the
 * empty context every word is found (its 1-gram).  Next state = c if order(c) < `order`, else suffix(c).
 * start = the state of "<s>", eos = word id of "</s>", unk = word id of "<unk>". */
typedef struct {
  const int32_t* word;
  const float* prob;
  const float* backoff;
  const int32_t* child_lo;
  const int32_t* child_hi;
  const int32_t* suffix;
  int32_t order;
  int32_t order_off[7];
  int32_t start, eos, unk;
} EspNgram;

/* Host-side ARPA parser (no GPU work).  Call twice on the same text: with t->word == NULL it reads the header and the
 * 1-grams and sets order, count[] (per order, including an added <unk>) and vocab_bytes; then, with every output
 * buffer allocated to those sizes (entries = sum of count), it parses everything and fills them.  vocab receives the
 * words by id, each NUL-terminated.  An ARPA without "<unk>" gets one as the last 1-gram with log10 p = -100 (as KenLM
 * does; unk_added = 1).  Refused with a message naming the cause (and the line for malformed lines): KenLM binary
 * files, orders outside 1..6, positive log-probabilities, counts that disagree with the header, words missing from
 * the 1-grams, duplicated n-grams, an n-gram whose context is not listed one order below, a missing <s> or </s>. */
typedef struct {
  int32_t order;
  int64_t count[6];
  int64_t vocab_bytes;
  int32_t unk_added;
  int32_t* word;
  float* prob;
  float* backoff;
  int32_t* child_lo;
  int32_t* child_hi;
  int32_t* suffix;
  char* vocab;
  int32_t start, eos, unk;
} EspArpaTables;
int esp_ngram_build(const char* text, int64_t len, EspArpaTables* t);

/* n pairs (states[i], words[i]) -> out_logp[i] = log10 P(word | state), out_next[i] = the next state (device). */
int esp_ngram_score(const EspNgram* lm, int32_t n, const int32_t* states, const int32_t* words, float* out_logp,
                    int32_t* out_next, void* stream);

/* Lexicon trie (flashlight's lexicon: a word, then its spelling in CTC units).  CSR edges from node n:
 * [child_off[n], child_off[n+1]) of (child_tok sorted ascending, child_node); node 0 is the root.  Words ending at node
 * n: words[word_off[n] .. word_off[n+1]) in ascending word id; word_lm[word] = its n-gram word id; smear[n] = max over
 * the words below n of log10 P(w | <s>), smear[0] = 0.  max_words = the largest number of words ending at one node. */
typedef struct {
  const int32_t* child_off;
  const int32_t* child_tok;
  const int32_t* child_node;
  const int32_t* word_off;
  const int32_t* words;
  const int32_t* word_lm;
  const float* smear;
  int32_t num_nodes, max_words;
} EspLexicon;

/* CTC prefix beam search with an n-gram LM scored inside the search kernel: one search launch for frames [0, t_max)
 * of every sentence, then finalize.  Same frames, stay / extend / merge / prune / select as esp_ctc_beam_search, and
 * per slot an n-gram state besides.
 * lex == NULL (lexicon-free): token v is n-gram word tok_word[v] (n_tok_word >= V entries); extending with v adds lm_weight * log10 P(v | y) +
 *   word_score; finalize adds lm_weight * log10 P(</s> | y).
 * lex != NULL: a slot also holds a trie node and a look-ahead term; score = lae(pb, pnb) + lm + lookahead.  A slot at
 *   node n extends only with tokens that are children c of n.  Candidates per (slot, token rank): first the in-word
 *   continuation (when c has children; lookahead = lm_weight * smear(c)), then one per word w ending at c in ascending
 *   word id (back to the root, lm += lm_weight * log10 P(w | words) + word_score, lookahead = 0).  Candidate index =
 *   h * (1 + K * (1 + max_words)) + j (j = 0 stay, then 1 + rank * (1 + max_words) + q).  A hypothesis is identified
 *   by its tokens and its word segmentation: merging compares both.  Finalize keeps root slots only and adds
 *   lm_weight * log10 P(</s> | words); a sentence without one returns no hypothesis (score -inf).
 * The candidate scores live in shared memory: a (beam, K, max_words) that does not fit is refused.
 * workspace: esp_ctc_ngram_workspace_bytes(B, t_max, beam), carried from search to finalize.  Outputs as
 * esp_ctc_beam_finalize. */
int64_t esp_ctc_ngram_workspace_bytes(int32_t B, int32_t t_max, int32_t beam);
int esp_ctc_ngram_search(const void* logits, int64_t stride_b, int64_t stride_t, int32_t V, int32_t B, int32_t t_max,
                         const int32_t* in_lens, const float* lse, const float* lp_blank, const int32_t* top_tok,
                         const float* top_lp, int32_t K, int32_t beam, float beam_threshold, const EspNgram* lm,
                         const int32_t* tok_word, int32_t n_tok_word, const EspLexicon* lex, float lm_weight,
                         float word_score,
                         void* workspace, void* stream);
int esp_ctc_ngram_finalize(int32_t B, int32_t t_max, const int32_t* in_lens, int32_t V, int32_t beam, int32_t nbest,
                           const EspNgram* lm, const EspLexicon* lex, float lm_weight, int32_t pad, void* workspace,
                           int32_t* out_tokens, int32_t* out_len, float* out_scores, int32_t* out_frames, void* stream);

/* ---- HBM-bound block kernels (bf16 activations [rows, channels], fp32 statistics) ----------------
 * LayerNorm forward/backward -- torch.nn.LayerNorm call sites: fairseq/modules/conformer_layer.py:79-81,
 *   134-136; espresso/modules/conformer_with_relative_positional_embedding_encoder_layer.py:118,143;
 *   fairseq/modules/transformer_layer.py:163-226; speech_transformer_encoder.py:348-349.
 * Optional fusions: zero rows t >= lens[b] (speech_transformer_encoder.py:354-357; rows are [B,T], so lens needs
 * T >= 1 dividing R) and a
 * trailing dropout (:350).  Backward accumulates dgamma/dbeta (fp32, +=) and adds an optional residual
 * gradient `dres` into dx. */
int esp_layer_norm_fwd(const void* x, const void* gamma, const void* beta, float eps, int64_t R, int32_t d,
                       void* y, float* mean, float* rstd, const int32_t* lens, int32_t T, float drop_p,
                       uint64_t seed, const uint64_t* seed_ptr, void* stream);
int esp_layer_norm_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const void* gamma,
                       const void* dres, int64_t R, int32_t d, void* dx, float* dgamma, float* dbeta,
                       const int32_t* lens, int32_t T, float drop_p, uint64_t seed, const uint64_t* seed_ptr,
                       void* stream);
/* Same, with a second output dx2 = dropout_{drop_p2, seed2}(dx) * scale2 on esp_dropout's counter stream (index r*d + c):
 * the masked residual-stream gradient the NEXT module's backward starts with (fairseq/modules/conformer_layer.py:232-277
 * differentiated: every module output passes through dropout before the residual add), written by this pass instead of by a
 * separate esp_dropout over dx.  dx2 may be NULL. */
int esp_layer_norm_bwd2(const void* dy, const void* x, const float* mean, const float* rstd, const void* gamma,
                        const void* dres, int64_t R, int32_t d, void* dx, float* dgamma, float* dbeta,
                        const int32_t* lens, int32_t T, float drop_p, uint64_t seed, const uint64_t* seed_ptr, void* dx2,
                        float drop_p2, uint64_t seed2, float scale2, void* stream);
/* out[n] += scale * sum_r x[r,n]   (the pos_bias_u / pos_bias_v gradients; Linear bias gradients come out of the
 * weight-gradient GEMM, EspGemm.rowsum_a) */
int esp_colsum(const void* x, int64_t R, int32_t N, int64_t ld, float scale, float* out, void* stream);
/* y = dropout(x) * scale, same counter RNG / indexing (r*N+n) as the GEMM epilogue */
int esp_dropout(const void* x, int64_t R, int32_t N, int64_t ldx, int64_t ldy, float scale, float drop_p,
                uint64_t seed, const uint64_t* seed_ptr, void* y, void* stream);
/* zero rows t >= lens[b] of x [B,T,N] */
int esp_mask_rows(void* x, const int32_t* lens, int32_t B, int32_t T, int32_t N, void* stream);
/* q_u = (q+u)*s, q_v = (q+v)*s  (fairseq/modules/multihead_attention.py:679-688) and the backward sum */
int esp_qprep_fwd(const void* q, int64_t ldq, const void* u, const void* v, float scale, int64_t R, int32_t d,
                  void* qu, void* qv, void* stream);
int esp_qprep_bwd(const void* dqu, const void* dqv, float scale, int64_t R, int32_t d, void* dq, int64_t ld_out,
                  void* stream);
/* attention softmax over keys (scores [H,B,T,ld] bf16): key-padding -> -inf, fp32 softmax, optional dropout
 * copy (fairseq/modules/multihead_attention.py:841-876); Tq x Tk scores (self- or cross-attention), optional
 * causal mask (decoder future mask, fairseq/models/transformer/transformer_decoder.py:404-419); backward also
 * scatters dS into the skewed relative-position layout dBD[., i, (T-1)-i+j] (inverse of :824-830).  A row with no
 * visible key (lens[b] == 0) gets P = 0 (the reference's softmax over all -inf would give NaN). */
int esp_attn_softmax_fwd(const void* scores, int32_t H, int32_t B, int32_t Tq, int32_t Tk, int32_t ld,
                         const int32_t* lens, int32_t causal, void* p, void* p_drop, float drop_p, uint64_t seed,
                         const uint64_t* seed_ptr, void* stream);
int esp_attn_softmax_bwd(const void* p, const void* dp_drop, int32_t H, int32_t B, int32_t Tq, int32_t Tk, int32_t ld,
                         void* ds, void* dbd, int32_t ldp, float drop_p, uint64_t seed, const uint64_t* seed_ptr,
                         void* stream);
/* Relaxed attention probabilities (fairseq/modules/multihead_attention.py:869-872, training only): p = the plain softmax
 * of esp_attn_softmax_fwd (no causal mask), p_drop = dropout((1 - w) p + w / Tk), always written, also at drop_p = 0.  Tk is
 * the PADDED key count, so padded keys receive w / Tk as in the reference; columns [Tk, ld) stay zero.  relax_w in (0, 1].
 * Backward: with g the dropout backward of dP_drop, dS = (1 - w) p (g - sum_j p g) -- esp_attn_softmax_bwd on p and
 * dP_drop, with (1 - w) folded into the alpha of the dq / dk GEMMs. */
int esp_attn_softmax_relaxed_fwd(const void* scores, int32_t H, int32_t B, int32_t Tq, int32_t Tk, int32_t ld,
                                 const int32_t* lens, void* p, void* p_drop, double relax_w, float drop_p, uint64_t seed,
                                 const uint64_t* seed_ptr, void* stream);
/* Fused relative-position self-attention forward (fairseq/modules/multihead_attention.py:788-897, rel-pos branch):
 * ctx = dropout(softmax(qu k^T + skew(qv pos^T) + key-padding mask)) v for every (utterance, head) in one launch.
 * The scores, the 2T-1 relative-position logits and the skew (BD[i,j] = BD_full[i,(T-1)-i+j], :824-830) stay in
 * registers / shared memory.  qu, qv: [B*T, H*64] bf16 (row stride ldq), already (q + pos_bias) * scaling
 * (:679-688); k, v: [B*T, H*64] bf16 with row stride ldkv (views into the fused q/k/v projection buffer); pos:
 * projected positions [2T-1, ldpos] bf16, head h at column h * pos_hstride (pos_hstride = 0: one table for all heads);
 * lens: valid keys per utterance (int32 [B]) or NULL; key_lo / key_hi: optional int32 [T] per-query-row visible key range
 * (chunk-streaming and limited-context masks, espresso/tools/utils.py:131-194, speech_transformer_encoder.py:232-263 --
 * contiguous per row, so two vectors replace the [T,T] mask).  ctx: [B*T, H*64] bf16.  p_out / pd_out: optional
 * [H, B, T, ldp] bf16 probabilities / dropped probabilities for the backward pass (pd_out only when drop_p > 0) --
 * same contents and dropout stream as esp_attn_softmax_fwd; ldp is at most 128 * ceil(T / 128), the columns the key
 * tiles cover.  An utterance with lens[b] == 0 has no visible key: its probabilities and its ctx rows are 0, as in
 * esp_attn_softmax_fwd and esp_decode_cross_attn.
 * pos == NULL: plain scaled dot-product self-attention, ctx = dropout(softmax(qu k^T + key-padding mask)) v, with qu = q *
 * scaling; qv, ldpos and pos_hstride are ignored (qv may be NULL).  A separate kernel instance without the position loads,
 * the W products and the skew; its outputs equal those of a call with an all-zero position table. */
int esp_attn_fused_fwd(const void* qu, const void* qv, int64_t ldq, const void* k, const void* v, int64_t ldkv,
                       const void* pos, int64_t ldpos, int32_t pos_hstride, int32_t B, int32_t T, int32_t H,
                       int32_t head_dim, const int32_t* lens, const int32_t* key_lo, const int32_t* key_hi, void* ctx,
                       int64_t ldctx, void* p_out, void* pd_out, int32_t ldp, float drop_p, uint64_t seed,
                       const uint64_t* seed_ptr, void* stream);
/* Fused relative-position self-attention backward, score side (backward of the call above, :788-897): from dctx and the
 * saved probabilities it produces dS [H,B,T,ldp_probs], its skewed copy dBD[., i, (T-1)-i+j] [H,B,T,ldbd] (zeros elsewhere;
 * inverse of the shift :824-830), dK = dS^T qu and dV = P_drop^T dctx -- replacing the dPd GEMM, esp_attn_softmax_bwd and
 * the dV / dK GEMMs of the unfused chain; dPd lives in registers only, dK / dV accumulate in registers over the query tiles.
 * dctx, ctx: [B*T, H*64] bf16 (row stride ldctx; ctx = the forward output, for the softmax row term sum_j P dP = dctx.ctx);
 * qu: as in the forward; v: [B*T, H*64] view with row stride ldkv; p / pd: what the forward saved (pd == p without dropout;
 * the dropout mask is regenerated from seed / seed_ptr, the forward's stream); rowdot_ws: fp32 [H*B*T] workspace;
 * dk / dv: [B*T, H*64] views with row stride ld_out (slices of the fused dqkv buffer).  The remaining gradients are plain
 * GEMMs: dq_u = dS k, dq_v = dBD pos, dpos = dBD^T q_v.  ldp_probs <= 128 * ceil(T / 128) as in the forward.
 * dbd == NULL (backward of the pos == NULL forward): no skewed copy is written (ldbd is ignored) and T is not limited to
 * the skew kernel's 1024 frames; dq = scaling * dS k. */
int esp_attn_fused_bwd(const void* dctx, const void* ctx, int64_t ldctx, const void* qu, int64_t ldq, const void* v,
                       int64_t ldkv, const void* p, const void* pd, int32_t ldp_probs, int32_t B, int32_t T, int32_t H,
                       int32_t head_dim, float drop_p, uint64_t seed, const uint64_t* seed_ptr, float* rowdot_ws, void* ds,
                       void* dbd, int32_t ldbd, void* dk, void* dv, int64_t ld_out, void* stream);
/* Conformer convolution module body (fairseq/modules/conformer_layer.py:88-96):
 *   y = depthwise_conv_k(GLU(g)) with 'same' zero padding over the padded length T, g [B,T,2C], w [C,k];
 *   stats (double [2,C], +=): per-channel sum and sum of squares of y for BatchNorm1d batch statistics.
 *   bn_finalize: mean / rstd (float [2,C]) from stats (training; also updates running stats with
 *   momentum, unbiased variance; R >= 1) or from the running stats (eval). */
int esp_glu_dwconv_fwd(const void* g, const void* w, int32_t B, int32_t T, int32_t C, int32_t ksz, void* y,
                       double* stats, void* stream);
int esp_glu_dwconv_bwd(const void* dy, const void* g, const void* w, int32_t B, int32_t T, int32_t C, int32_t ksz,
                       void* dg, float* dw, void* stream);
int esp_bn_finalize(const double* stats, int64_t R, int32_t C, float eps, float momentum, float* run_mean,
                    float* run_var, int32_t training, float* mr, void* stream);
/* Channels-last BatchNorm helpers shared by the Conformer conv module (act=1, SiLU; fairseq/modules/
 * conformer_layer.py:95-96) and the conv front end (act=2, ReLU; espresso/modules/speech_convolutions.py:88-90,
 * tensors kept NHWC so rows = B*T*F): per-channel statistics of x [R,C]; z = act(BN(y)); and the two-pass
 * backward (sums = double[3,C] workspace: 2C sums + 2C float coefficients; dgamma/dbeta fp32, +=). */
/* pre_bias (bf16 [C] or NULL): the normalised tensor is bf16(x + pre_bias[c]) without materialising it -- the bias of
 * the convolution in front of the BatchNorm (espresso/modules/speech_convolutions.py:88-90: Conv2d has bias=True),
 * so the convolution itself runs bias-free and no separate bias-add / bias-gradient pass over the activation exists
 * (the bias gradient through a batch-statistics BatchNorm is identically zero). */
int esp_bn_stats(const void* x, const void* pre_bias, int64_t R, int32_t C, double* stats, void* stream);
int esp_bn_act_fwd(const void* y, const void* pre_bias, int64_t R, int32_t C, const float* mr, const void* gamma,
                   const void* beta, int32_t act, void* z, void* stream);
int esp_bn_act_bwd(const void* dz, const void* y, const void* pre_bias, int64_t R, int32_t C, const float* mr,
                   const void* gamma, const void* beta, int32_t act, double* sums, void* dy, float* dgamma,
                   float* dbeta, void* stream);

/* 3x3 convolutions of the conv front end (espresso/modules/speech_convolutions.py:78-102, Convolution2d :104-132: kernel 3x3,
 * zero padding 1, stride (st, sf) in {1, 2}); replaces F.conv2d and its dgrad / wgrad.  Activations are channels-last
 * [B, T, F, C] bf16, weights [Cout, 3, 3, Cin] bf16 (the channels-last storage of the reference's [Cout, Cin, 3, 3]
 * parameter), output positions To = ceil(T / st), Fo = ceil(F / sf).  The bias is NOT added here (see pre_bias above).
 *   esp_conv3x3_fwd / _dgrad / _wgrad: Cin and Cout multiples of 64 -- implicit GEMMs on the wgmma kernel (im2col tiles
 *     are TMA boxes of the activation shifted by the filter tap; nothing is materialised); dw is fp32 [Cout, 3, 3, Cin], +=.
 *   esp_conv3x3_c1_fwd / _c1_wgrad: the first layer, ONE input channel: x [B, T, F] bf16, w [Cout, 3, 3], dw fp32 +=
 *     (no input gradient: the features need none). */
int esp_conv3x3_fwd(const void* x, const void* w, void* y, int32_t B, int32_t T, int32_t F, int32_t Cin, int32_t Cout,
                    int32_t st, int32_t sf, void* stream);
int esp_conv3x3_dgrad(const void* dy, const void* w, void* dx, int32_t B, int32_t T, int32_t F, int32_t Cin, int32_t Cout,
                      int32_t st, int32_t sf, void* stream);
int esp_conv3x3_wgrad(const void* dy, const void* x, float* dw, int32_t B, int32_t T, int32_t F, int32_t Cin, int32_t Cout,
                      int32_t st, int32_t sf, void* stream);
int esp_conv3x3_c1_fwd(const void* x, const void* w, void* y, int32_t B, int32_t T, int32_t F, int32_t Cout, int32_t st,
                       int32_t sf, void* stream);
int esp_conv3x3_c1_wgrad(const void* dy, const void* x, float* dw, int32_t B, int32_t T, int32_t F, int32_t Cout, int32_t st,
                         int32_t sf, void* stream);

/* ---- optimizer on flat buffers (fairseq/optim/fp16_optimizer.py:109-168, fairseq/optim/adam.py:150-239,
 *      fairseq/utils.py:347-397) ---------------------------------------------------------------- */
int esp_sumsq_f32(const float* g, int64_t n, float* out, void* stream);
/* g_eff = g / denom * clip_coef, denom read from device memory if denom_dev != NULL (the all-reduced
 * sample_size in the gradient buffer's tail), else denom_const.  hyper_dev (optional DEVICE float[2] =
 * {lr, step}) overrides the by-value lr/step so a captured CUDA graph can be replayed with a new schedule
 * value.  Writes fp32 master + bf16 model params. */
int esp_adam_step(float* p32, float* m, float* v, const float* g, void* p16, int64_t n, float lr, float beta1,
                  float beta2, float eps, float weight_decay, int32_t step, const float* sumsq,
                  const float* denom_dev, float denom_const, float clip_norm, float* gnorm_out,
                  const float* hyper_dev, void* stream);
int esp_cast_f32_bf16(const float* x, int64_t n, void* y, void* stream);
int esp_cast_bf16_f32(const void* x, int64_t n, float* y, void* stream);

/* ---- decoder-side kernels --------------------------------------------------------------------
 * Label-smoothed cross-entropy fused with the fp32 log-softmax, forward + backward
 * (espresso/criterions/label_smoothed_cross_entropy_v2.py:49-120,216-240).  smoothing_type 0 = uniform:
 *   loss[r] = (1-eps-eps_i)*nll + eps_i*smooth, eps_i = eps/(V-1); 1 = unigram (`unigram` fp32 [V], the smoothed
 *   unigram distribution): (1-eps)*nll - eps*sum_v u[v]*lprobs[v]; 2 = temporal (rows are [B, U]; neighbouring
 *   targets at distance 1 / 2 weighted 5 : 2, normalised, <pad> neighbours dropped).  Rows with target == pad_idx
 *   give 0.  grad = grad_scale * dloss/dlogits (bf16, same row stride; NULL = loss only); each row's columns
 *   [0, ceil8(V)) are written, [V, ceil8(V)) as zero, nothing else.  ld % 8 == 0; logits and grad 16-byte aligned. */
int esp_lsce_loss(const void* logits, int64_t ld, int32_t V, int64_t R, const int32_t* targets, int32_t pad_idx,
                  float eps, int32_t smoothing_type, const float* unigram, int32_t U, float grad_scale, float* loss,
                  float* nll, void* grad, void* stream);
/* x[r] = dropout(bf16(E[tok[r]]*scale) + pos[r % U]) (pos optional; pad tokens get no position), and the
 * scatter-add backward into the fp32 embedding gradient (fairseq/models/transformer/transformer_decoder.py:254-300).
 * E, pos and x 16-byte aligned.  The backward adds fp32(dx * scale) per term, without the reference's bf16 rounding
 * of scale * dx. */
int esp_embed_fwd(const int32_t* tokens, const void* E, const void* pos, int32_t U, int32_t d, float scale, int64_t R,
                  int32_t pad_idx, void* x, float drop_p, uint64_t seed, const uint64_t* seed_ptr, void* stream);
int esp_embed_bwd(const int32_t* tokens, const void* dx, int32_t d, float scale, int64_t R, int32_t pad_idx, float* dE,
                  float drop_p, uint64_t seed, const uint64_t* seed_ptr, void* stream);
/* out[r] = argmax_v x[r, v<V]  (greedy CTC decoding, espresso/tools/ctc_decoder.py:163-188), in torch.argmax's order:
 * the first NaN of a row wins, then the first of equal maxima, so out[r] is in [0, V).  V >= 1, ld >= V. */
int esp_argmax_rows(const void* x, int64_t ld, int32_t V, int64_t R, int32_t* out, void* stream);

/* ---- batched beam search step (fairseq/sequence_generator.py:355-609, fairseq/search.py:103-144) -------------
 * merge: out[n, v] = masked fused log-prob + prev_scores[n]: fp32 log-softmax of x/temperature (x_is_logits) or x as
 *   given, + lm_weight * (LM log-probs) (:385-393), NaN -> -inf, pad -> -inf, unk -= penalty, force_eos (step >=
 *   max_len, :401-403), eos_factor gate (:404-410), ban_eos (step < min_len, :422-424).  x / lm: bf16 or fp32 rows.
 * topk: per sentence, the best K of n_cand = nb*V candidates (row stride sent_stride), ordered by (score desc, flat
 *   index asc); token = idx % V, beam = idx / V.
 * bookkeep: finalise eos candidates, pick the next `beam` hypotheses, re-gather tokens [N, max_len+2] / cumulative
 *   scores [N, max_len+1] into the *_out buffers, emit new_order (source row of every new hypothesis) and keep a
 *   device count of unfinished sentences.  fin_tokens / fin_pos: [bsz, beam, max_len+1]; fin_len / fin_score: [bsz, beam].
 * gather_rows: dst[i, :] = src[idx[i], :] for incremental-state reordering (multihead_attention.py:964-989). */
int esp_beam_merge(const void* x, int32_t x_f32, int64_t ld_x, int32_t x_is_logits, float temperature, const void* lm,
                   int32_t lm_f32, int64_t ld_lm, int32_t lm_is_logits, float lm_weight, int32_t N, int32_t V,
                   const float* prev_scores, int32_t pad, int32_t unk, float unk_penalty, int32_t eos, int32_t force_eos,
                   int32_t use_eos_factor, float eos_factor, int32_t ban_eos, float* out, void* stream);
int esp_beam_topk(const float* cand, int64_t sent_stride, int32_t bsz, int32_t n_cand, int32_t K, int32_t V,
                  float* out_scores, int32_t* out_tokens, int32_t* out_beams, void* stream);
int esp_beam_bookkeep(int32_t step, int32_t max_len, int32_t bsz, int32_t beam, int32_t K, int32_t eos, int32_t pad,
                      int32_t normalize, float len_penalty, const float* cand_scores, const int32_t* cand_tokens,
                      const int32_t* cand_beams, const int32_t* tokens_in, int32_t* tokens_out, const float* scores_in,
                      float* scores_out, uint8_t* ignore, uint8_t* finished, int32_t* nfin, int32_t* fin_tokens,
                      int32_t* fin_len, float* fin_score, float* fin_pos, int32_t* new_order, int32_t* n_unfinished,
                      void* stream);
/* bookkeep_attn: esp_beam_bookkeep plus the encoder attention of every hypothesis it finalises (replaces the per-step
 *   `attn` index_select and the finalisation slice of fairseq/sequence_generator.py:603-605,690,739-748).  att [T_max, N, Tk]
 *   fp32 holds the decoder's attention row of cache row r at step t (esp_decode_cross_attn_weights); anc [T_max, N] is the
 *   ancestry table of this step (esp_decode_update_ancestry).  A hypothesis finalised at `step` from row r into slot k gets
 *   fin_attn[sentence, k, t, :] = att[t][anc[t][r]] for t = 0..step; fin_attn: fp32 [bsz, beam, max_len+1, Tk].  Every
 *   other output is bit-identical to esp_beam_bookkeep. */
int esp_beam_bookkeep_attn(int32_t step, int32_t max_len, int32_t bsz, int32_t beam, int32_t K, int32_t eos, int32_t pad,
                           int32_t normalize, float len_penalty, const float* cand_scores, const int32_t* cand_tokens,
                           const int32_t* cand_beams, const int32_t* tokens_in, int32_t* tokens_out, const float* scores_in,
                           float* scores_out, uint8_t* ignore, uint8_t* finished, int32_t* nfin, int32_t* fin_tokens,
                           int32_t* fin_len, float* fin_score, float* fin_pos, int32_t* new_order, int32_t* n_unfinished,
                           const float* att, const int32_t* anc, int32_t Tk, float* fin_attn, void* stream);
int esp_gather_rows(const void* src, const int32_t* idx, int64_t row_bytes, int64_t n_rows, void* dst, void* stream);

/* ---- search options of the beam search step (csrc/beam_options.cu) ---------------------------------------------------
 * block_ngrams (--no-repeat-ngram-size n; replaces NGramRepeatBlock, fairseq/ngram_repeat_block.py, called at
 *   fairseq/sequence_generator.py:448-449): for each of the N rows of the int32 token buffer (column 0 = the start symbol,
 *   columns 1..step = the hypothesis), every earlier window tokens[i .. i+n-2], i < step-n+2, equal to the row's last n-1
 *   tokens (columns step-n+2 .. step) bans tokens[i+n-1]: lprobs[row, tokens[i+n-1]] = -inf, in place.  Nothing happens
 *   while step < n - 1.  n = 1 bans every token of the row, the start symbol included.
 * prefix (--prefix-size; replaces fairseq/sequence_generator.py:414-424 and _prefix_tokens :623-657): prefix int32
 *   [bsz, >= step+1] (row stride ld_prefix); for each sentence whose prefix[s, step] is not pad, every beam's candidate row
 *   of cand fp32 [bsz*beam, V] keeps only that token (the rest = -inf).  If that token is eos, beam 0's tokens
 *   [bsz*beam, L] row, scores [bsz*beam, L-1] row and candidate row are copied into every other beam of the sentence.
 *   The caller applies it only while step < prefix length and step < max_len, and drops the min-length eos ban there.
 * diverse_groups (--diverse-beam-groups G, --diverse-beam-strength; replaces DiverseBeamSearch.step, fairseq/search.py:
 *   551-618): lprobs fp32 [bsz*beam, V] without cumulative scores; prev_scores fp32 [bsz*beam] (NULL at step 0).  Group g
 *   (beams g, g+G, ...) ranks (lprobs - strength * count[token]) + prev over its beams (step 0: its first beam only), where
 *   count[token] is how often earlier groups picked the token at this step, and keeps its top Kg = min(2*beam/G,
 *   n_cand - 1).  Outputs [bsz, Kg*G], entry r*G + g = group g's r-th candidate, beams in sentence numbering.  beam % G
 *   must be 0.  One launch.
 * sibling_topk (--diversity-rate; replaces DiverseSiblingsSearch.step at step > 0, fairseq/search.py:745-810): cand fp32
 *   [bsz*beam, V] with cumulative scores (esp_beam_merge's output); each row's top k, its r-th entry minus (r+1) * rate,
 *   then the sentence's top k of the beam*k pool -> out [bsz, k] (scores keep the penalty).  work_s / work_t / work_b:
 *   [bsz*beam*k] scratch.  Four launches (row top-k, penalty, pool top-k, token remap).
 * sample (--sampling, --sampling-topk, --sampling-topp; replaces Sampling.step / _sample_topp, fairseq/search.py:621-742):
 *   lprobs fp32 [bsz*beam, V] without cumulative scores; prev_scores fp32 [bsz*beam], NULL at step 0.  Candidate
 *   o = s*beam + j draws one token from p = exp(lprobs) of row o (step 0: of row s*beam, the sentence's first beam, one draw
 *   per j) -> out [bsz, beam]: score = log p[token] (+ prev_scores[o]), token, beam j (0 at step 0).  Tokens are ranked by
 *   (p descending, token ascending) with fixed-point masses W = floor(p * 2^40), whose sums are exact: topp > 0 keeps the
 *   tokens whose preceding mass is < floor(topp * 2^40) (the reference's cumsum < p plus one more token; topp <= 1); else
 *   0 < topk < V keeps the first topk tokens; else all.  The draw: h = esp_hash_u64(esp_hash_u64(*seed, step),
 *   (row << 16) | draw), draw = j at step 0 and 0 after; T = floor(h * sum W / 2^64); the token is the first kept token, in
 *   token order, whose cumulative W exceeds T.  A row without mass gives token 0 at -inf.  *seed is read from device
 *   memory at run time (CUDA graphs replay with the current seed).  V * 4 bytes of shared memory, V <= 51200.  One launch.
 * Limits: prefix tokens outside [0, V) are skipped by esp_beam_prefix (the generator refuses them before the search);
 *   esp_beam_diverse_groups takes Kg <= 64 and V <= 51200, so one group (G = 1) is limited to beam <= 32. */
int esp_beam_block_ngrams(const int32_t* tokens, int64_t ld_tokens, int32_t N, int32_t step, int32_t n, float* lprobs,
                          int64_t ld_lprobs, int32_t V, void* stream);
int esp_beam_prefix(const int32_t* prefix, int64_t ld_prefix, int32_t bsz, int32_t beam, int32_t step, int32_t pad, int32_t eos,
                    float* cand, int32_t V, int32_t* tokens, int32_t L, float* scores, void* stream);
int esp_beam_diverse_groups(const float* lprobs, const float* prev_scores, int32_t bsz, int32_t beam, int32_t V, int32_t groups,
                            int32_t Kg, float strength, float* out_scores, int32_t* out_tokens, int32_t* out_beams, void* stream);
int esp_beam_sibling_topk(const float* cand, int32_t bsz, int32_t beam, int32_t V, int32_t k, float rate, float* work_s,
                          int32_t* work_t, int32_t* work_b, float* out_scores, int32_t* out_tokens, int32_t* out_beams,
                          void* stream);
int esp_beam_sample(const float* lprobs, const float* prev_scores, int32_t bsz, int32_t beam, int32_t V, int32_t topk, float topp,
                    const uint64_t* seed, int32_t step, float* out_scores, int32_t* out_tokens, int32_t* out_beams, void* stream);

/* ---- look-ahead word-LM fusion (espresso/models/tensorized_lookahead_language_model.py:84-262) -------------
 * A word LM scores subword hypotheses through a lexical prefix tree (espresso/tools/tensorized_prefix_tree.py:15-108,
 * here in CSR form: node 0 = "outside the lexicon", node 1 = root, edges sorted by subword id; node_lo/node_hi =
 * (first word id - 1, last word id) of the words below a node, node_word = word id ending at the node or -1).
 * One search step = three calls:
 *   lookahead_words: nodes_out[n] = nodes_in[new_order[n]] (new_order NULL = identity); words[n] = the word the
 *     hypothesis has just completed (word_unk if none) -- the word LM's input (:126-130).
 *   wordlm_cumsum: rows whose previous subword (prev_tokens[n * tok_stride]) is <space>, or all rows when first != 0:
 *     cum_out[n, :] = inclusive cumsum(softmax(logits[n, :Vw])) (fp32) and eos_logprob[n] = log softmax[word_eos];
 *     every other row copies cum_in[new_order[n], :] (the reference's reorder_incremental_state, :264-272).
 *     logits: bf16 or fp32 [N, ld]; cum_in != cum_out.  log_mode != 0: the rows hold log_softmax instead (no scan) --
 *     the per-word log-probabilities the multi-level LM keeps (external_language_model.py:425-436).
 *   lookahead_step: tree transition on prev_tokens (nodes_in -> nodes_out, :150-164) and the subword log-probability row
 *     out[n, :Vs] (fp32, Eqn. 15 cases 1-4 of arXiv:1808.02608 as implemented at :173-263; columns Vs..ld_out-1 = -inf).
 *     open_vocab = 0: probability `zero` outside the lexicon; zero = 1e-10 in the reference. */
int esp_lookahead_words(const int32_t* nodes_in, const int32_t* new_order, const int32_t* node_word, int32_t word_unk,
                        int32_t N, int32_t* nodes_out, int32_t* words, void* stream);
int esp_wordlm_cumsum(const void* logits, int32_t logits_f32, int64_t ld, int32_t N, int32_t Vw, const int32_t* prev_tokens,
                      int64_t tok_stride, int32_t space_idx, int32_t first, const float* cum_in, const int32_t* new_order,
                      float* cum_out, float* eos_logprob, int32_t word_eos, int32_t log_mode, void* stream);
int esp_lookahead_step(const int32_t* prev_tokens, int64_t tok_stride, int32_t N, int32_t first, const int32_t* nodes_in,
                       int32_t* nodes_out, const float* cum, int32_t Vw, const float* eos_logprob, const int32_t* child_off,
                       const int32_t* child_tok, const int32_t* child_node, const int32_t* node_word, const int32_t* node_lo,
                       const int32_t* node_hi, int32_t space_idx, int32_t eos_idx, int32_t pad_idx, int32_t word_unk,
                       float oov_penalty, int32_t open_vocab, float zero, float* out, int64_t ld_out, int32_t Vs,
                       void* stream);

/* multilevel_step (MultiLevelLanguageModel, espresso/models/external_language_model.py:385-555): the subword LM's row
 * (sub: bf16 / fp32 [N, ld_sub], logits or log-probs) is scaled by sub_weight; <space> gets the word LM's log-probability
 * of the completed word minus what the subword LM accumulated inside it (cumlp), or the <unk> score + log_oov_penalty
 * outside the lexicon; </s> adds the word-level </s>.  out_prev / cumlp_in are the previous step's out / cumlp_out
 * (read at row new_order[n]); nodes_in is already reordered (esp_lookahead_words).  logzero = -10 in the reference. */
int esp_multilevel_step(const int32_t* prev_tokens, int64_t tok_stride, int32_t N, int32_t first, const int32_t* nodes_in,
                        int32_t* nodes_out, const int32_t* new_order, const float* wordlm_logprobs, int32_t Vw, const void* sub,
                        int32_t sub_f32, int64_t ld_sub, int32_t sub_is_logits, float sub_weight, const float* out_prev,
                        const float* cumlp_in, float* cumlp_out, const int32_t* child_off, const int32_t* child_tok,
                        const int32_t* child_node, const int32_t* node_word, int32_t space_idx, int32_t eos_idx,
                        int32_t word_unk, int32_t word_eos, float log_oov_penalty, int32_t open_vocab, float logzero, float* out,
                        int64_t ld_out, int32_t Vs, void* stream);

/* ---- incremental decoding (fairseq/modules/multihead_attention.py:639-760,878-897,964-989) --------------
 * One query per hypothesis.  Self-attention: kv_cache [T_max, N, 2d] (k | v) is written in place by the K/V
 * projection GEMM of each step; anc [T_max, N] maps (time, hypothesis) -> cache row, so beam reordering never
 * moves K/V (update_ancestry re-gathers only the int table).  Cross-attention: kv [bsz, Tk, 2d] per SENTENCE
 * (hypothesis n reads sentence n / beam), lens = valid encoder frames or NULL. */
int esp_decode_self_attn(const void* q, const void* kv_cache, const int32_t* anc, int32_t N, int32_t H, int32_t hd, int32_t T,
                         float scale, void* out, void* stream);
int esp_decode_cross_attn(const void* q, const void* kv, const int32_t* lens, int32_t N, int32_t beam, int32_t H, int32_t hd,
                          int32_t Tk, float scale, void* out, void* stream);
/* cross_attn_weights: esp_decode_cross_attn (bit-identical context) that also writes weights[n, 0:Tk] = the fp32 softmax
 *   probabilities of hypothesis n averaged over the H heads (summed in head order, no atomics; padded keys exactly 0) --
 *   the encoder attention the reference returns with need_weights (fairseq/modules/multihead_attention.py:864,913-915;
 *   last decoder layer, fairseq/models/transformer/transformer_decoder.py:283-284).  1 <= H <= 32. */
int esp_decode_cross_attn_weights(const void* q, const void* kv, const int32_t* lens, int32_t N, int32_t beam, int32_t H,
                                  int32_t hd, int32_t Tk, float scale, void* out, float* weights, void* stream);
int esp_decode_update_ancestry(const int32_t* anc_in, int32_t* anc_out, const int32_t* new_order, int32_t N, int32_t step,
                               void* stream);
/* Prefix decoding: hypotheses that grow on different frames, by different amounts (a CTC prefix beam search fused with a
 * Transformer LM).  An addition beyond the reference, whose CTC decoder fuses KenLM only.  The cache is indexed by frame
 * SLOT: kv_cache [S, N, 2d], slot 0 = the eos context, slot f + 1 written at frame f for every row, so a write never
 * lands on a cell another hypothesis still reads.  Hypothesis n's keys are the flat cells (slot * N + row)
 * cells[i * N + n], i < len[n] (cells int32 [S, N], len int32 [N], both double-buffered like anc).
 * update_paths, with p = new_order[n]: cells_out[i][n] = cells_in[i][p] for i < len_in[p]; if grown[n] != 0,
 *   cells_out[len_in[p]][n] = slot * N + n; len_out[n] = len_in[p] + (grown[n] != 0); pos_out[n] = len_in[p] (the
 *   position row of the token row n feeds at this slot; may be NULL).  Requires len_in[*] <= slot.  One launch per frame.
 * self_attn_paths: esp_decode_self_attn over len[n] keys read through cells (len[n] <= slots <= 1280); len[n] = 0 writes
 *   zeros.  Same per-warp softmax and P.V code as esp_decode_self_attn. */
int esp_decode_update_paths(const int32_t* cells_in, const int32_t* len_in, int32_t* cells_out, int32_t* len_out,
                            int32_t* pos_out, const int32_t* new_order, const int32_t* grown, int32_t slot, int32_t N,
                            void* stream);
int esp_decode_self_attn_paths(const void* q, const void* kv_cache, const int32_t* cells, const int32_t* len, int32_t slots,
                               int32_t N, int32_t H, int32_t hd, float scale, void* out, void* stream);

/* ---- transducer (RNN-T) ---------------------------------------------------------------------------------
 * joint: F[b,t,u,:] = relu(enc[b,t,:] + dec[b,u,:]) (espresso/models/transformer/speech_transformer_transducer_base.py:
 *   279-299, after the two projection+LayerNorm stages); backward: denc = sum_u dF*(F>0) (bf16, written),
 *   ddec += sum_t dF*(F>0) (fp32, accumulated).  J % 8 == 0; enc, dec, out, dF, F and denc 16-byte aligned;
 *   backward B <= 65535.
 * rnnt_loss: torchaudio.functional.rnnt_loss(logits [B,T,U1,V] (row stride ld), targets int32 [B,u_max], t_lens, u_lens,
 *   blank, clamp=-1, fused_log_softmax=True) as called by espresso/criterions/transducer_loss.py:130-140: loss fp32 [B]
 *   (negative log-likelihood per utterance) and grad = grad_scale * d(sum loss)/d(logits) (bf16, same layout; every
 *   cell's columns [0, ceil8(V)) are written, cells outside the utterance's lattice and columns [V, ceil8(V)) as zero,
 *   nothing else).  ld % 8 == 0, logits 16-byte aligned.  workspace: esp_rnnt_workspace_bytes(B, T, U1). */
int esp_joint_fwd(const void* enc, const void* dec, int32_t B, int32_t T, int32_t U1, int32_t J, void* out, void* stream);
int esp_joint_bwd(const void* df, const void* f, int32_t B, int32_t T, int32_t U1, int32_t J, void* denc, float* ddec, void* stream);
int64_t esp_rnnt_workspace_bytes(int32_t B, int32_t T, int32_t U1);
int esp_rnnt_loss(const void* logits, int64_t ld, int32_t V, int32_t B, int32_t T, int32_t U1, const int32_t* t_lens,
                  const int32_t* u_lens, const int32_t* targets, int32_t u_max, int32_t blank, float grad_scale, float* loss,
                  void* grad, void* workspace, void* stream);

/* ---- transducer beam search (adaptive expansion), the whole batch at once ---------------------------------------
 * Replaces the search steps of espresso/tools/transducer_beam_search_decoder.py:270-463 (prefix search),
 * :465-601 (expansion rounds, final blank, n-best) and espresso/tools/transducer_utils.py select_k_expansions; the
 * host loop (espresso_b200/tools/transducer_beam_search_decoder.py: BatchedAdaptiveExpansionSearch) runs the
 * prediction network, LM and joint GEMMs in between.  EspRnntBeam holds the search's device tables (all flat,
 * utterance-major; K = beam + beta rows per utterance, A = E * K set-aside entries, P pool nodes, Pm = beam(beam-1)/2
 * merge pairs, S = Pm * alpha path steps; ring_stride = rows of one age of the decoder-output rings).  Ties rank by
 * (key desc, candidate index asc), see csrc/transducer_beam.cu.  Limits: K <= 32, beam <= 16, alpha <= 8,
 * A + K <= 1024; rows of V (+ the LM's vocabulary) fp32 fit one CTA's shared memory.
 * lprobs: logits bf16 [n, ld] (and lm_logits [n, ld_lm], bf16 or fp32, V or V - 1 columns) -> val fp32 [n, k],
 *   tok int32 [n, k] (top k of log_softmax(logits / temperature), LM-fused, eos folded, + scores), lpb fp32 [n] (raw
 *   blank log-prob).  gamma < 0 in select: no pruning by value. */
typedef struct EspRnntBeam {
  int32_t B, K, E, A, P, Pm, S, alpha, ring_stride;
  float* score; int32_t* nemit; int32_t* len; int32_t* node; int32_t* srow; int32_t* fsrc; int32_t* parent; int32_t* prev;
  int32_t* nrow; int32_t* nlive; const int32_t* nframes;
  float* a_score; int32_t* a_nemit; int32_t* a_len; int32_t* a_node; int32_t* a_src; int32_t* na;
  int32_t* p_parent; int32_t* p_tok; int32_t* p_len; unsigned long long* p_hash; int32_t* npool;
  int32_t* m_pair; int32_t* m_ring; int32_t* m_tok; int32_t* m_npair;
} EspRnntBeam;
int esp_rnnt_beam_lprobs(const void* logits, int64_t ld, int32_t V, int32_t n, const float* scores, int32_t k, int32_t blank,
                         float temperature, int32_t eos, int32_t fold_eos, const void* lm_logits, int64_t ld_lm, int32_t lm_f32,
                         float lm_weight, int32_t no_blank_in_lm, float* val, int32_t* tok, float* lpb, void* stream);
int esp_rnnt_beam_prefix_merge(const EspRnntBeam* s, int32_t t, void* stream);
int esp_rnnt_beam_merge_scores(const void* logits, int64_t ld, int32_t V, const EspRnntBeam* s, float temperature, int32_t blank,
                               const void* lm_logits, int64_t ld_lm, int32_t lm_f32, float lm_weight, int32_t no_blank_in_lm,
                               void* stream);
int esp_rnnt_beam_select(const float* val, const int32_t* tok, int32_t k, const float* lpb, const EspRnntBeam* s, int32_t rnd,
                         int32_t beam, int32_t blank, float gamma, int32_t normalize, int32_t final, void* stream);
int esp_rnnt_beam_finalize(const EspRnntBeam* s, int32_t L, int32_t pad, int64_t* tokens, float* scores, int32_t* lens,
                           void* stream);

/* ---- host-side batch packing (no GPU work) -------------------------------------------------------
 * The native packer behind fairseq.data.data_utils.batch_by_size (fairseq/data/data_utils_fast.pyx:20-105,
 * batch_by_size_vec): num_tokens[i] = size of the i-th sample in packing order; writes the split points into
 * ends[0..n) and returns how many there are (use them like numpy.split), -1 on error. */
int64_t esp_batch_by_size(const int64_t* num_tokens, int64_t n, int64_t max_tokens, int64_t max_sentences,
                          int32_t bsz_mult, int32_t* ends);

#ifdef __cplusplus
}
#endif
#endif /* ESPRESSO_B200_H_ */
