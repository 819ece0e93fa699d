// espresso_b200 -- ARPA n-gram tables: the host parser behind esp_ngram_build (no GPU work).
//
// The text is read in place, section by section; each order is resolved against the orders below it, which are
// complete by then (ARPA lists the orders in increasing order): an n-gram's context is walked down from its first
// word's 1-gram through the child ranges, and its suffix link is the longest of its proper suffixes that the same walk
// finds.  Entries of one order are sorted by (context entry, word id), so each entry's children form one contiguous
// range of the next order.  Layout and scoring: include/espresso_b200.h (EspNgram).
#include "common.cuh"
#include "espresso_b200.h"
#include <algorithm>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

namespace {

constexpr int kMaxOrder = 6;

struct Reader {
  const char* p;
  const char* end;
  long line = 0;
  // next line without its newline and trailing whitespace; false at the end of the text
  bool next(std::string_view& s) {
    if (p >= end) return false;
    const char* e = (const char*)memchr(p, '\n', end - p);
    if (!e) e = end;
    const char* q = e;
    while (q > p && (q[-1] == '\r' || q[-1] == ' ' || q[-1] == '\t')) --q;
    s = std::string_view(p, q - p);
    p = e < end ? e + 1 : end;
    ++line;
    return true;
  }
};

inline bool is_ws(char c) { return c == ' ' || c == '\t'; }

int split(std::string_view s, std::string_view* f, int cap) {
  int n = 0;
  size_t i = 0;
  while (i < s.size()) {
    while (i < s.size() && is_ws(s[i])) ++i;
    if (i >= s.size()) break;
    size_t j = i;
    while (j < s.size() && !is_ws(s[j])) ++j;
    if (n == cap) return cap + 1;
    f[n++] = s.substr(i, j - i);
    i = j;
  }
  return n;
}

bool blank(std::string_view s) {
  for (char c : s)
    if (!is_ws(c)) return false;
  return true;
}

bool parse_float(std::string_view s, float& v) {
  char buf[64];
  if (s.empty() || s.size() >= sizeof(buf)) return false;
  memcpy(buf, s.data(), s.size());
  buf[s.size()] = 0;
  char* e = nullptr;
  v = strtof(buf, &e);
  return e == buf + s.size() && !isnan(v);
}

bool parse_long(std::string_view s, long& v) {
  char buf[32];
  if (s.empty() || s.size() >= sizeof(buf)) return false;
  memcpy(buf, s.data(), s.size());
  buf[s.size()] = 0;
  char* e = nullptr;
  v = strtol(buf, &e, 10);
  return e == buf + s.size();
}

struct Tmp {
  int ctx, w, suffix;
  float prob, bo;
};

// child of global entry e labelled w, or -1
inline int find_child(const EspArpaTables* t, int e, int w) {
  const int lo = t->child_lo[e], hi = t->child_hi[e];
  const int* b = t->word + lo;
  const int* it = std::lower_bound(b, (const int*)t->word + hi, w);
  return (it != t->word + hi && *it == w) ? (int)(it - t->word) : -1;
}

// entry of the n-gram ws[0..n) (every order < n complete), or -1
inline int find_ngram(const EspArpaTables* t, const int* ws, int n) {
  int e = ws[0];
  for (int i = 1; i < n && e >= 0; ++i) e = find_child(t, e, ws[i]);
  return e;
}

}  // namespace

extern "C" int esp_ngram_build(const char* text, int64_t len, EspArpaTables* t) {
  ESP_CHECK(t && (text || len == 0) && len >= 0, "esp_ngram_build: bad arguments");
  const bool fill = t->word != nullptr;
  ESP_CHECK(!(len >= 8 && memcmp(text, "mmap lm ", 8) == 0),
            "this is a KenLM binary file; only ARPA text (.arpa or .arpa.gz) is read -- load the ARPA it was built from");
  ESP_CHECK(memchr(text, 0, (size_t)std::min<int64_t>(len, 4096)) == nullptr,
            "binary data where ARPA text was expected (KenLM binary files are not read; pass the .arpa or .arpa.gz)");
  Reader r{text, text + len};
  std::string_view s;
  // header
  bool found = false;
  while (r.next(s)) {
    if (s == "\\data\\") { found = true; break; }
  }
  ESP_CHECK(found, "not an ARPA file: no \\data\\ line");
  long count[kMaxOrder] = {0};
  int order = 0;
  while (true) {
    const char* before = r.p;  // the first line after the counts may start the 1-grams: it is read again below
    const long line_before = r.line;
    if (!r.next(s)) break;
    if (blank(s)) {
      if (order > 0) break;
      continue;
    }
    std::string_view f[3];
    if (split(s, f, 2) != 2 || f[0] != "ngram") {
      r.p = before;
      r.line = line_before;
      break;
    }
    const size_t eq = f[1].find('=');
    long k = 0, c = 0;
    ESP_CHECK(eq != std::string_view::npos && parse_long(f[1].substr(0, eq), k) && parse_long(f[1].substr(eq + 1), c),
              "malformed ARPA header at line %ld", r.line);
    ESP_CHECK(k == order + 1, "ARPA header at line %ld: expected ngram %d=, got ngram %ld=", r.line, order + 1, k);
    ESP_CHECK(k <= kMaxOrder, "ARPA order %ld is above the supported maximum %d", k, kMaxOrder);
    ESP_CHECK(c >= 0 && c < (1L << 31), "ARPA header at line %ld: bad count %ld", r.line, c);
    count[order++] = c;
  }
  ESP_CHECK(order >= 1, "ARPA header lists no n-gram counts");
  ESP_CHECK(count[0] >= 1, "ARPA file without 1-grams");
  long total = 0;
  for (int k = 0; k < order; ++k) total += count[k];
  ESP_CHECK(total + 1 < (1L << 31), "ARPA file too large (%ld n-grams)", total);

  std::unordered_map<std::string_view, int> vocab;
  vocab.reserve((size_t)count[0] * 2);
  std::vector<Tmp> tmp;
  int64_t off[kMaxOrder + 1] = {0};
  for (int k = 1; k <= order; ++k) {
    // section header
    char want[16];
    snprintf(want, sizeof(want), "\\%d-grams:", k);
    found = false;
    while (r.next(s)) {
      if (blank(s)) continue;
      ESP_CHECK(s == want, "line %ld: expected %s, got '%.*s'", r.line, want, (int)std::min<size_t>(s.size(), 40), s.data());
      found = true;
      break;
    }
    ESP_CHECK(found, "ARPA file ends before its %s section", want);
    tmp.clear();
    if (k > 1) tmp.reserve((size_t)count[k - 1]);
    long n = 0;
    while (true) {
      const char* before = r.p;
      const long line_before = r.line;
      if (!r.next(s)) break;
      if (blank(s)) continue;
      if (s[0] == '\\') { r.p = before; r.line = line_before; break; }
      ++n;
      if (!fill && k == 1) {  // sizing pass: the 1-gram words only
        std::string_view f[kMaxOrder + 3];
        const int nf = split(s, f, kMaxOrder + 2);
        ESP_CHECK(nf == 2 || nf == 3, "malformed 1-gram at line %ld", r.line);
        ESP_CHECK(vocab.emplace(f[1], (int)vocab.size()).second, "duplicated 1-gram '%.*s' at line %ld",
                  (int)f[1].size(), f[1].data(), r.line);
        continue;
      }
      if (!fill) continue;
      std::string_view f[kMaxOrder + 3];
      const int nf = split(s, f, kMaxOrder + 2);
      ESP_CHECK(nf == k + 1 || (nf == k + 2 && k < order), "malformed %d-gram at line %ld (%d fields)", k, r.line, nf);
      float p = 0.f, bo = 0.f;
      ESP_CHECK(parse_float(f[0], p), "malformed log-probability at line %ld", r.line);
      ESP_CHECK(p <= 0.f, "positive log-probability %g at line %ld", p, r.line);
      if (nf == k + 2) ESP_CHECK(parse_float(f[k + 1], bo) && isfinite(bo), "malformed backoff at line %ld", r.line);
      int ws[kMaxOrder];
      if (k == 1) {
        ESP_CHECK(vocab.emplace(f[1], (int)vocab.size()).second, "duplicated 1-gram '%.*s' at line %ld",
                  (int)f[1].size(), f[1].data(), r.line);
        const int w = (int)vocab.size() - 1;
        t->word[w] = w; t->prob[w] = p; t->backoff[w] = bo; t->suffix[w] = -1;
        t->child_lo[w] = t->child_hi[w] = 0;
        continue;
      }
      for (int i = 0; i < k; ++i) {
        auto it = vocab.find(f[1 + i]);
        ESP_CHECK(it != vocab.end(), "line %ld: word '%.*s' is not among the 1-grams", r.line, (int)f[1 + i].size(),
                  f[1 + i].data());
        ws[i] = it->second;
      }
      const int ctx = find_ngram(t, ws, k - 1);
      ESP_CHECK(ctx >= 0, "line %ld: the context of this %d-gram is not listed among the %d-grams", r.line, k, k - 1);
      int suf = -1;
      for (int i = 1; i < k && suf < 0; ++i) suf = find_ngram(t, ws + i, k - i);
      tmp.push_back(Tmp{ctx, ws[k - 1], suf, p, bo});
    }
    ESP_CHECK(n == count[k - 1], "the %d-gram section has %ld entries, the header says %ld", k, n, count[k - 1]);
    if (k == 1) {
      // an ARPA without <unk> gets one as its last 1-gram, log10 p = -100 (as KenLM does)
      t->unk_added = vocab.find(std::string_view("<unk>")) == vocab.end();
      if (t->unk_added) {
        const int w = (int)vocab.size();
        vocab.emplace(std::string_view("<unk>"), w);
        if (fill) {
          t->word[w] = w; t->prob[w] = -100.f; t->backoff[w] = 0.f; t->suffix[w] = -1;
          t->child_lo[w] = t->child_hi[w] = 0;
        }
      }
      off[1] = (int64_t)vocab.size();
      if (!fill) break;
      continue;
    }
    const int64_t base = off[k - 1];
    off[k] = base + n;
    std::sort(tmp.begin(), tmp.end(), [](const Tmp& a, const Tmp& b) { return a.ctx != b.ctx ? a.ctx < b.ctx : a.w < b.w; });
    for (size_t i = 0; i < tmp.size(); ++i) {
      ESP_CHECK(i == 0 || tmp[i].ctx != tmp[i - 1].ctx || tmp[i].w != tmp[i - 1].w,
                "duplicated %d-gram in the ARPA file", k);
      const int64_t e = base + (int64_t)i;
      t->word[e] = tmp[i].w; t->prob[e] = tmp[i].prob; t->backoff[e] = tmp[i].bo; t->suffix[e] = tmp[i].suffix;
      t->child_lo[e] = t->child_hi[e] = 0;
      if (i == 0 || tmp[i].ctx != tmp[i - 1].ctx) t->child_lo[tmp[i].ctx] = (int)e;
      t->child_hi[tmp[i].ctx] = (int)(e + 1);
    }
  }
  if (!fill) {
    t->order = order;
    for (int k = 0; k < kMaxOrder; ++k) t->count[k] = k == 0 ? off[1] : (k < order ? count[k] : 0);
    int64_t vb = 0;
    for (const auto& kv : vocab) vb += (int64_t)kv.first.size() + 1;
    t->vocab_bytes = vb;
    return 0;
  }
  ESP_CHECK(t->order == order, "esp_ngram_build: the sizing call saw a different text");
  ESP_CHECK(vocab.count(std::string_view("<s>")), "the ARPA file has no <s> 1-gram");
  ESP_CHECK(vocab.count(std::string_view("</s>")), "the ARPA file has no </s> 1-gram");
  std::vector<std::string_view> words(vocab.size());
  for (const auto& kv : vocab) words[kv.second] = kv.first;
  char* vp = t->vocab;
  for (const auto& w : words) {
    memcpy(vp, w.data(), w.size());
    vp += w.size();
    *vp++ = 0;
  }
  t->unk = vocab.find(std::string_view("<unk>"))->second;
  t->eos = vocab.find(std::string_view("</s>"))->second;
  t->start = order > 1 ? vocab.find(std::string_view("<s>"))->second : -1;
  return 0;
}
