// espresso_b200 -- FLAC decoding on the device (RFC 9639): a batch of compressed streams -> the float32 waveform layout
// the front end reads, [B, ld] in int16 range.
//
// Reference path being replaced (CPU, per utterance, in DataLoader workers):
//   fairseq/data/audio/audio_utils.py:69-126 get_waveform -> soundfile.read (libsndfile + libFLAC), then
//   `wav * 2**15` for normalization=False and the channel mean for mono.
//
// A frame's length is only known once the frame has been decoded, so frames are found by search and then chained:
//   flac_scan_kernel     every byte: a sync code (0xFFF8 / 0xFFF9) whose header parses, agrees with the stream's
//                        STREAMINFO and passes CRC-8 becomes a candidate; cand_at[byte] = candidate index or -1.
//   flac_measure_kernel  one warp per candidate: lane 0 parses every subframe with a bounds-checked bit reader (no
//                        sample reconstruction), finds the frame's end and checks its CRC-16.
//   flac_chain_kernel    one CTA per stream: from the stream's first byte, each next frame must begin exactly where the
//                        previous frame's CRC-16 ends and carry the next sample number, until STREAMINFO's total is
//                        covered exactly.  Only then are its frames marked; the row's tail (or the whole row of a
//                        stream that fails) is zeroed and the stream's status written.
//   flac_decode_kernel   one warp per MARKED frame: lane 0 parses again and stores warm-up samples and residuals as
//                        int32 in scratch, lanes 0..channels-1 run their channel's predictor, then all lanes undo the
//                        stereo decorrelation and write s / 2^(bps-1) * 2^15, channels averaged in float32.
// A false sync inside residual or verbatim data can pass CRC-8 and even CRC-16, but it never begins where a frame of
// the chain ends, so it never reaches `out`.
//
// The predictor is a serial recurrence over each subframe's samples (int64 accumulation, since side channels carry
// bps + 1 bits and LPC coefficients up to 15), and the Rice codes before it are serial within the frame: the kernels
// are latency-bound, with one warp per frame as the unit of parallelism.
#include "common.cuh"
#include "espresso_b200.h"

namespace {

constexpr int kMaxCh = 8;
constexpr int kMaxOrder = 32;
constexpr int kWarps = 4;  // warps per CTA of the frame kernels
constexpr int kParams = 5;  // int64 per stream: total samples, sample rate, channels, bps, max block size

struct Cand {
  long long first;  // first sample number
  int pos;          // byte offset of the sync code in the batch buffer
  int end;          // byte offset just past the CRC-16 (measure pass)
  int b;            // stream
  int bs;           // block size
  int hdr;          // header bytes incl. CRC-8
  int assign;       // channel assignment
  int status;       // ESP_FLAC_* of the measure pass
  int keep;         // on its stream's chain
};

struct SubDesc {
  int type;  // 0 constant, 1 verbatim, 2 predicted (FIXED as LPC with shift 0)
  int order, shift, wasted, value;
  int coef[kMaxOrder];
};

__device__ __forceinline__ bool stream_supported(const long long* P, int max_ch) {
  return P[0] > 0 && P[2] >= 1 && P[2] <= max_ch && P[3] >= 4 && P[3] <= 24 && P[4] >= 1 && P[4] <= 65535;
}

__device__ __forceinline__ unsigned crc8_byte(unsigned c, unsigned b) {
  c ^= b;
#pragma unroll
  for (int i = 0; i < 8; ++i) c = ((c << 1) ^ ((c & 0x80) ? 0x07u : 0u)) & 0xFFu;
  return c;
}

// Frame header at p (avail bytes left in the stream) -> true if it is a header of this stream.
__device__ bool parse_header(const uint8_t* p, long long avail, const long long* P, long long& first, int& bs, int& hdr,
                             int& assign) {
  if (avail < 6 || p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return false;
  const int variable = p[1] & 1;
  const int bsc = p[2] >> 4, src = p[2] & 15, a = p[3] >> 4, bpsc = (p[3] >> 1) & 7;
  if (bsc == 0 || src == 15 || a > 10 || bpsc == 3 || (p[3] & 1)) return false;
  int i = 4;
  const unsigned b0 = p[i++];
  long long num = b0;
  if (b0 >= 0x80) {  // UTF-8-like coded number, 2-7 bytes
    const int n = __clz(~(b0 << 24));
    if (n < 2 || n > 7) return false;
    num = b0 & (0x7Fu >> n);
    for (int k = 1; k < n; ++k) {
      if (i >= avail) return false;
      const unsigned c = p[i++];
      if ((c & 0xC0) != 0x80) return false;
      num = (num << 6) | (c & 0x3F);
    }
  }
  if (!variable && num >= (1LL << 31)) return false;
  if (bsc == 6) {
    if (i + 1 > avail) return false;
    bs = p[i] + 1, i += 1;
  } else if (bsc == 7) {
    if (i + 2 > avail) return false;
    bs = ((p[i] << 8) | p[i + 1]) + 1, i += 2;
  } else {
    bs = bsc == 1 ? 192 : bsc <= 5 ? 576 << (bsc - 2) : 256 << (bsc - 8);
  }
  long long rate = P[1];
  if (src >= 12) {
    const int nb = src == 12 ? 1 : 2;
    if (i + nb > avail) return false;
    const int v = nb == 1 ? p[i] : (p[i] << 8) | p[i + 1];
    rate = src == 12 ? v * 1000LL : src == 13 ? v : v * 10LL;
    i += nb;
  } else if (src > 0) {
    const int rates[12] = {0, 88200, 176400, 192000, 8000, 16000, 22050, 24000, 32000, 44100, 48000, 96000};
    rate = rates[src];
  }
  if (i + 1 > avail) return false;
  unsigned crc = 0;
  for (int k = 0; k < i; ++k) crc = crc8_byte(crc, p[k]);
  if (crc != p[i]) return false;
  const int bps_codes[8] = {0, 8, 12, 0, 16, 20, 24, 32};
  const int bps = bpsc ? bps_codes[bpsc] : (int)P[3];
  const int channels = a < 8 ? a + 1 : 2;
  if (bps != P[3] || channels != P[2] || rate != P[1] || bs > P[4]) return false;
  first = variable ? num : num * P[4];
  hdr = i + 1;
  assign = a;
  return true;
}

// MSB-first bit reader over bytes [0, nbytes) of the batch buffer; bits past the end read as 0 and make overrun() true.
struct BitReader {
  const uint8_t* base;
  long long nbytes, next, pos;
  unsigned long long cache;
  int n;

  __device__ void init(const uint8_t* b, long long end_byte, long long start_byte) {
    base = b, nbytes = end_byte, next = start_byte, pos = start_byte * 8, cache = 0, n = 0;
  }
  __device__ __forceinline__ void refill() {
    while (n <= 56) {
      const unsigned long long v = next < nbytes ? __ldg(base + next) : 0;
      cache |= v << (56 - n);
      n += 8, ++next;
    }
  }
  __device__ __forceinline__ bool overrun() const { return pos > nbytes * 8; }
  __device__ __forceinline__ unsigned get(int k) {  // 0 <= k <= 32
    if (k == 0) return 0;
    refill();
    const unsigned v = (unsigned)(cache >> (64 - k));
    cache <<= k;
    n -= k, pos += k;
    return v;
  }
  __device__ __forceinline__ int sget(int k) {
    if (k == 0) return 0;
    const unsigned v = get(k);
    return (int)(v << (32 - k)) >> (32 - k);
  }
  // zero bits before the next 1 (consumed); -1 past the end or beyond max_q
  __device__ __forceinline__ long long unary(long long max_q) {
    long long q = 0;
    for (;;) {
      refill();
      if (cache == 0) {
        q += n, pos += n, n = 0;
        if (overrun() || q > max_q) return -1;
        continue;
      }
      const int z = __clzll(cache);
      q += z, pos += z + 1, n -= z + 1;
      cache = z == 63 ? 0ull : cache << (z + 1);
      return q > max_q ? -1 : q;
    }
  }
  __device__ void seek(long long bit) {
    next = bit >> 3, pos = next * 8, cache = 0, n = 0;
    get((int)(bit & 7));
  }
};

// Residual of one subframe into dst[order, bs) (kStore), or just skipped.
template <bool kStore>
__device__ int read_residual(BitReader& br, int bs, int order, int* dst) {
  const int method = br.get(2);
  if (method > 1) return ESP_FLAC_RESERVED;
  const int pbits = method ? 5 : 4, esc = method ? 31 : 15;
  const int po = br.get(4);
  if ((bs & ((1 << po) - 1)) || (bs >> po) < order) return ESP_FLAC_RESERVED;
  int at = order;
  for (int p = 0; p < (1 << po); ++p) {
    const int n = (bs >> po) - (p == 0 ? order : 0);
    const int k = br.get(pbits);
    if (k == esc) {
      const int nb = br.get(5);
      if (kStore) {
        for (int i = 0; i < n; ++i) dst[at + i] = br.sget(nb);
      } else {
        br.seek(br.pos + (long long)n * nb);
      }
    } else {
      const long long max_q = (1LL << (32 - k)) - 1;  // the folded residual must fit 32 bits
      for (int i = 0; i < n; ++i) {
        const long long q = br.unary(max_q);
        if (q < 0) return br.overrun() ? ESP_FLAC_TRUNCATED : ESP_FLAC_RESERVED;
        const unsigned u = ((unsigned)q << k) | br.get(k);
        if (kStore) dst[at + i] = (int)(u >> 1) ^ -(int)(u & 1);
      }
    }
    at += n;
    if (br.overrun()) return ESP_FLAC_TRUNCATED;
  }
  return ESP_FLAC_OK;
}

template <bool kStore>
__device__ int read_subframe(BitReader& br, int bs, int sbps, SubDesc& d, int* dst) {
  if (br.get(1)) return ESP_FLAC_RESERVED;
  const int t = br.get(6);
  int wasted = 0;
  if (br.get(1)) {
    const long long q = br.unary(sbps);
    if (q < 0) return br.overrun() ? ESP_FLAC_TRUNCATED : ESP_FLAC_RESERVED;
    wasted = (int)q + 1;
    if (wasted >= sbps) return ESP_FLAC_RESERVED;
  }
  const int b = sbps - wasted;
  d.wasted = wasted, d.order = 0, d.shift = 0;
  if (t == 0) {
    d.type = 0;
    d.value = br.sget(b);
  } else if (t == 1) {
    d.type = 1;
    if (kStore) {
      for (int i = 0; i < bs; ++i) dst[i] = br.sget(b);
    } else {
      br.seek(br.pos + (long long)bs * b);
    }
  } else if ((t >= 8 && t <= 12) || t >= 32) {
    const int order = t >= 32 ? t - 31 : t - 8;
    if (order > bs) return ESP_FLAC_RESERVED;
    d.type = 2, d.order = order;
    for (int i = 0; i < order; ++i) {
      const int v = br.sget(b);
      if (kStore) dst[i] = v;
    }
    if (t >= 32) {
      const int prec = br.get(4) + 1;
      if (prec == 16) return ESP_FLAC_RESERVED;
      d.shift = br.sget(5);
      if (d.shift < 0) return ESP_FLAC_LPC_SHIFT;
      for (int j = 0; j < order; ++j) d.coef[j] = br.sget(prec);
    } else {
      const int fixed[5][4] = {{0, 0, 0, 0}, {1, 0, 0, 0}, {2, -1, 0, 0}, {3, -3, 1, 0}, {4, -6, 4, -1}};
      for (int j = 0; j < order; ++j) d.coef[j] = fixed[order][j];
    }
    const int st = read_residual<kStore>(br, bs, order, dst);
    if (st) return st;
  } else {
    return ESP_FLAC_RESERVED;
  }
  return br.overrun() ? ESP_FLAC_TRUNCATED : ESP_FLAC_OK;
}

__device__ __forceinline__ bool is_side(int assign, int c) {
  return (assign == 8 && c == 1) || (assign == 9 && c == 0) || (assign == 10 && c == 1);
}

// Every subframe of candidate k; sets *end to the byte just past its CRC-16.  kStore: descriptors into sd[], samples of
// channel c into pcm + c * ld.
template <bool kStore>
__device__ int read_frame(const uint8_t* bytes, long long stream_end, const Cand& k, int bps, SubDesc* sd, int* pcm,
                          long long ld, int* end) {
  BitReader br;
  br.init(bytes, stream_end, k.pos + k.hdr);
  const int channels = k.assign < 8 ? k.assign + 1 : 2;
  SubDesc scratch;
  for (int c = 0; c < channels; ++c) {
    const int st = read_subframe<kStore>(br, k.bs, bps + is_side(k.assign, c), kStore ? sd[c] : scratch,
                                         kStore ? pcm + c * ld : nullptr);
    if (st) return st;
  }
  const int r = (int)(br.pos & 7);
  if (r && br.get(8 - r)) return ESP_FLAC_RESERVED;  // padding must be zero
  const long long e = br.pos / 8 + 2;
  if (e > stream_end) return ESP_FLAC_TRUNCATED;
  *end = (int)e;
  return ESP_FLAC_OK;
}

// x[order, bs) += (sum_j coef[j] x[i-1-j]) >> shift, in place; MAXO >= order keeps the history in registers.
template <int MAXO>
__device__ void restore(int* x, int bs, const SubDesc& d) {
  int c[MAXO], h[MAXO];
#pragma unroll
  for (int j = 0; j < MAXO; ++j) {
    c[j] = j < d.order ? d.coef[j] : 0;
    h[j] = j < d.order ? x[d.order - 1 - j] : 0;
  }
  const int shift = d.shift;
  for (int i = d.order; i < bs; ++i) {
    long long acc = 0;
#pragma unroll
    for (int j = 0; j < MAXO; ++j) acc += (long long)c[j] * h[j];
    const int s = (int)((unsigned)x[i] + (unsigned)(acc >> shift));
    x[i] = s;
#pragma unroll
    for (int j = MAXO - 1; j > 0; --j) h[j] = h[j - 1];
    h[0] = s;
  }
}

__device__ void reconstruct(int* x, int bs, const SubDesc& d) {
  if (d.type == 0) {
    for (int i = 0; i < bs; ++i) x[i] = (int)((unsigned)d.value << d.wasted);
    return;
  }
  if (d.type == 2) {
    if (d.order <= 4) restore<4>(x, bs, d);
    else if (d.order <= 8) restore<8>(x, bs, d);
    else if (d.order <= 16) restore<16>(x, bs, d);
    else restore<32>(x, bs, d);
  }
  if (d.wasted)
    for (int i = 0; i < bs; ++i) x[i] = (int)((unsigned)x[i] << d.wasted);
}

__global__ void __launch_bounds__(256)
flac_scan_kernel(const uint8_t* __restrict__ bytes, long long n_bytes, const long long* __restrict__ offsets,
                 const long long* __restrict__ prm, int B, int max_ch, int* __restrict__ cand_at, Cand* __restrict__ cands,
                 int* __restrict__ count, int cap) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n_bytes; p += (long long)gridDim.x * blockDim.x) {
    int idx = -1;
    if (bytes[p] == 0xFF && p >= offsets[0] && p < offsets[B]) {
      int lo = 0, hi = B - 1;  // the last stream starting at or before p
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (offsets[mid] <= p) lo = mid;
        else hi = mid - 1;
      }
      const long long* P = prm + (long long)lo * kParams;
      long long first;
      int bs, hdr, assign;
      if (stream_supported(P, max_ch) && parse_header(bytes + p, offsets[lo + 1] - p, P, first, bs, hdr, assign)) {
        const int i = atomicAdd(count, 1);
        if (i < cap) {
          Cand c;
          c.first = first, c.pos = (int)p, c.end = -1, c.b = lo, c.bs = bs, c.hdr = hdr, c.assign = assign;
          c.status = ESP_FLAC_NO_FRAME, c.keep = 0;
          cands[i] = c;
          idx = i;
        }
      }
    }
    cand_at[p] = idx;
  }
}

__global__ void __launch_bounds__(kWarps * 32)
flac_measure_kernel(const uint8_t* __restrict__ bytes, const long long* __restrict__ offsets, const long long* __restrict__ prm,
                    Cand* __restrict__ cands, const int* __restrict__ count, int cap) {
  __shared__ unsigned short s_crc[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    unsigned c = (unsigned)i << 8;
    for (int k = 0; k < 8; ++k) c = (c << 1) ^ ((c & 0x8000) ? 0x8005u : 0u);
    s_crc[i] = (unsigned short)c;
  }
  __syncthreads();
  const int n = min(*count, cap);
  const int nw = gridDim.x * kWarps;
  for (int ci = blockIdx.x * kWarps + (threadIdx.x >> 5); ci < n; ci += nw) {
    if ((threadIdx.x & 31) != 0) continue;
    Cand& k = cands[ci];
    const long long stream_end = offsets[k.b + 1];
    int end = -1;
    int st = read_frame<false>(bytes, stream_end, k, (int)prm[(long long)k.b * kParams + 3], nullptr, nullptr, 0, &end);
    if (st == ESP_FLAC_OK) {
      unsigned crc = 0;
      for (int i = k.pos; i < end - 2; ++i) crc = ((crc << 8) & 0xFFFFu) ^ s_crc[(crc >> 8) ^ __ldg(bytes + i)];
      if (crc != ((unsigned)bytes[end - 2] << 8 | bytes[end - 1])) st = ESP_FLAC_CRC16;
    }
    k.end = end;
    k.status = st;
  }
}

__global__ void __launch_bounds__(256)
flac_chain_kernel(const long long* __restrict__ offsets, const long long* __restrict__ prm, int max_ch,
                  const int* __restrict__ cand_at, Cand* __restrict__ cands, float* __restrict__ out, long long ld,
                  int* __restrict__ status) {
  __shared__ int s_st;
  const int b = blockIdx.x;
  const long long* P = prm + (long long)b * kParams;
  const long long total = P[0];
  if (threadIdx.x == 0) {
    int st = stream_supported(P, max_ch) && total <= ld ? ESP_FLAC_OK : ESP_FLAC_BAD_PARAMS;
    const long long begin = offsets[b], end = offsets[b + 1];
    for (int pass = 0; pass < 2 && st == ESP_FLAC_OK; ++pass) {  // pass 0 checks the chain, pass 1 marks it
      long long p = begin, s = 0;
      while (st == ESP_FLAC_OK && s < total) {
        const int c = p < end ? cand_at[p] : -1;
        if (c < 0) {
          st = ESP_FLAC_NO_FRAME;
          break;
        }
        Cand& k = cands[c];
        if (k.status != ESP_FLAC_OK) st = k.status;
        else if (k.first != s || s + k.bs > total) st = ESP_FLAC_BAD_SEQUENCE;
        if (st != ESP_FLAC_OK) break;
        if (pass == 1) k.keep = 1;
        s += k.bs;
        p = k.end;
      }
    }
    status[b] = st;
    s_st = st;
  }
  __syncthreads();
  float* row = out + (long long)b * ld;
  for (long long i = (s_st == ESP_FLAC_OK ? total : 0) + threadIdx.x; i < ld; i += blockDim.x) row[i] = 0.f;
}

__global__ void __launch_bounds__(kWarps * 32)
flac_decode_kernel(const uint8_t* __restrict__ bytes, const long long* __restrict__ offsets, const long long* __restrict__ prm,
                   int max_ch, const Cand* __restrict__ cands, const int* __restrict__ count, int cap, int* __restrict__ pcm,
                   float* __restrict__ out, long long ld) {
  __shared__ SubDesc s_sd[kWarps][kMaxCh];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = min(*count, cap);
  const int nw = gridDim.x * kWarps;
  for (int ci = blockIdx.x * kWarps + w; ci < n; ci += nw) {
    const Cand k = cands[ci];
    if (!k.keep) continue;  // warp-uniform
    const long long* P = prm + (long long)k.b * kParams;
    const int C = (int)P[2], bps = (int)P[3];
    int* x = pcm + (long long)k.b * max_ch * ld + k.first;
    if (lane == 0) {
      int end;
      read_frame<true>(bytes, offsets[k.b + 1], k, bps, s_sd[w], x, ld, &end);  // passed in the measure kernel
    }
    __syncwarp();
    if (lane < C) reconstruct(x + lane * ld, k.bs, s_sd[w][lane]);
    __syncwarp();
    const float scale = __int_as_float((128 - bps) << 23);  // 2^(1 - bps), exact
    float* o = out + (long long)k.b * ld + k.first;
    for (int i = lane; i < k.bs; i += 32) {
      int v0 = x[i], v1 = C > 1 ? x[ld + i] : 0;
      if (k.assign == 8) {
        v1 = v0 - v1;
      } else if (k.assign == 9) {
        v0 = v0 + v1;
      } else if (k.assign == 10) {
        const int mid = (int)((unsigned)v0 << 1) | (v1 & 1);
        v0 = (mid + v1) >> 1;
        v1 = (mid - v1) >> 1;
      }
      float acc = __fmul_rn(__int2float_rn(v0), scale);
      if (C > 1) {
        acc = __fadd_rn(acc, __fmul_rn(__int2float_rn(v1), scale));
        for (int c = 2; c < C; ++c) acc = __fadd_rn(acc, __fmul_rn(__int2float_rn(x[c * ld + i]), scale));
        acc = __fdiv_rn(acc, (float)C);
      }
      o[i] = __fmul_rn(acc, 32768.f);
    }
    __syncwarp();
  }
}

long long cand_capacity(int B, long long n_bytes) {
  // two sync candidates whose headers both parse are at least 4 bytes apart (bytes 2 and 3 of a header are never 0xFF)
  return n_bytes / 4 + B + 1;
}

}  // namespace

extern "C" int64_t esp_flac_decode_workspace_bytes(int32_t B, int64_t n_bytes, int32_t max_channels, int64_t ld) {
  if (B <= 0 || n_bytes < 0 || max_channels < 1 || ld < 0) return 0;
  return align256(sizeof(int)) + align256(cand_capacity(B, n_bytes) * (long)sizeof(Cand)) + align256(n_bytes * 4) +
         align256((long)B * max_channels * ld * 4);
}

extern "C" int esp_flac_decode(const void* bytes, int64_t n_bytes, const int64_t* offsets, const int64_t* params, int32_t B,
                               int32_t max_channels, float* out, int64_t ld, int32_t* status, void* workspace, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(B >= 0 && n_bytes >= 0 && ld >= 0, "bad FLAC batch shape B=%d n_bytes=%lld ld=%lld", B, (long long)n_bytes,
            (long long)ld);
  ESP_CHECK(max_channels >= 1 && max_channels <= kMaxCh, "max_channels must be in [1, %d]", kMaxCh);
  ESP_CHECK(n_bytes < (1LL << 31), "a FLAC batch holds less than 2 GiB of frames");
  if (B == 0) return 0;
  ESP_CHECK(offsets && params && out && status && workspace && (bytes || n_bytes == 0),
            "null pointer passed to esp_flac_decode");
  const long long cap = cand_capacity(B, n_bytes);
  char* ws = (char*)workspace;
  int* count = (int*)ws;
  ws += align256(sizeof(int));
  Cand* cands = (Cand*)ws;
  ws += align256(cap * (long)sizeof(Cand));
  int* cand_at = (int*)ws;
  ws += align256(n_bytes * 4);
  int* pcm = (int*)ws;
  const uint8_t* in = (const uint8_t*)bytes;
  const long long* off = (const long long*)offsets;
  const long long* prm = (const long long*)params;
  ESP_CUDA(cudaMemsetAsync(count, 0, sizeof(int), st));
  if (n_bytes > 0)
    ESP_CUDA(esp_launch_plain(flac_scan_kernel, grid_for(n_bytes, 256), 256, 0, st, in, (long long)n_bytes, off, prm, B,
                              (int)max_channels, cand_at, cands, count, (int)cap));
  const int frame_grid = esp_num_sms() * 8;
  ESP_CUDA(esp_launch_plain(flac_measure_kernel, frame_grid, kWarps * 32, 0, st, in, off, prm, cands, (const int*)count,
                            (int)cap));
  ESP_CUDA(esp_launch_plain(flac_chain_kernel, B, 256, 0, st, off, prm, (int)max_channels, (const int*)cand_at, cands, out,
                            (long long)ld, status));
  ESP_CUDA(esp_launch_plain(flac_decode_kernel, frame_grid, kWarps * 32, 0, st, in, off, prm, (int)max_channels,
                            (const Cand*)cands, (const int*)count, (int)cap, pcm, out, (long long)ld));
  return 0;
}
