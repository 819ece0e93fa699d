// espresso_b200 -- C-ABI plumbing: error strings, launch counter, cached device attributes.
#include "common.cuh"
#include "espresso_b200.h"
#include <atomic>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

namespace {
thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};
}  // namespace

void esp_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void esp_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int esp_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;  // H100 SXM
  }
  return sms;
}

bool esp_pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("ESP_PDL");
    on = (e && e[0] == '0') ? 0 : 1;
  }
  return on == 1;
}

extern "C" const char* esp_last_error(void) { return g_err; }
extern "C" int esp_version(void) { return 103; }
extern "C" int64_t esp_launch_count(void) { return (int64_t)g_launches.load(); }
extern "C" void esp_note_graph_replay(int64_t launches) { g_launches.fetch_add(launches, std::memory_order_relaxed); }

// ---- host-side batch packing -----------------------------------------------------------------------
// Greedy length-bucketed packing of consecutive (already ordered) samples under max_tokens (= longest sample x batch
// size), max_sentences and a batch-size multiple: the native code behind fairseq.data.data_utils.batch_by_size
// (fairseq/data/data_utils_fast.pyx:20-105, `batch_by_size_vec`).  A running batch [start, end) and a tail [end, pos]
// are tracked; the tail joins the batch whenever the union is valid and its size is below / a multiple of bsz_mult; on
// overflow the batch is closed and the tail starts the next one (a tail that overflows by itself is closed as well).
// num_tokens[i] is the size of the i-th sample IN PACKING ORDER.  Writes the split points (exclusive batch ends, the
// final end n omitted like numpy.split wants) to `ends` (capacity n) and returns their count, or -1 on error.
extern "C" int64_t esp_batch_by_size(const int64_t* num_tokens, int64_t n, int64_t max_tokens, int64_t max_sentences,
                                     int32_t bsz_mult, int32_t* ends) {
  if (n < 0 || (n > 0 && (!num_tokens || !ends)) || bsz_mult < 1) {
    esp_set_error("esp_batch_by_size: bad arguments");
    return -1;
  }
  if (n == 0) return 0;
  for (int64_t i = 0; i < n; ++i) {
    ends[i] = 0;
    if (max_tokens > 0 && num_tokens[i] > max_tokens) {
      esp_set_error("Sentences lengths should not exceed max_tokens=%lld (sample %lld has %lld)", (long long)max_tokens,
                    (long long)i, (long long)num_tokens[i]);
      return -1;
    }
  }
  int64_t count = 0, start = 0, tail_max = 0, batch_max = 0;
  for (int64_t pos = 0; pos < n; ++pos) {
    if (num_tokens[pos] > tail_max) tail_max = num_tokens[pos];
    const int64_t new_end = pos + 1;
    int64_t new_max = batch_max > tail_max ? batch_max : tail_max;
    const int64_t sentences = new_end - start;
    const bool overflow = (max_sentences > 0 && sentences > max_sentences) || (max_tokens > 0 && sentences * new_max > max_tokens);
    const bool size_ok = sentences < bsz_mult || sentences % bsz_mult == 0;
    if (overflow) {
      const bool tail_overflow = max_tokens > 0 && tail_max * (new_end - ends[count]) > max_tokens;
      if (tail_overflow) {  // the tail without the current sample becomes a batch of its own
        ++count;
        ends[count] = (int32_t)pos;
        tail_max = num_tokens[pos];
      }
      start = ends[count];
      ++count;
      new_max = tail_max;
    }
    if (overflow || size_ok) {
      ends[count] = (int32_t)new_end;
      batch_max = new_max;
      tail_max = 0;
    }
  }
  if (ends[count] != n) ++count;
  return count;
}
