// SoftLexicon host builder (SURVEY 8(f) rank 3): the step just before the gather-and-pool kernel.
//
// Replaces, for whole datasets at a time, the reference's per-sentence Python
//   build_soft_lexicon      data/word_enhance.py:302-337   every substring of <= 10 characters found in the word
//                                                          vocabulary joins the B/M/E/S sets of the characters it covers
//   align_with_token        data/word_enhance.py:89-119    characters one word piece swallowed share one row (set union)
//   postproc_soft_lexicon   data/word_enhance.py:163-205   pad to / keep the 10 most frequent per set, weights =
//                                                          frequency / sum over the token's four sets
//   SoftLexiconProc.format_soft_seq  data/base_preprocess.py:397-412  [CLS]/[SEP]/[PAD] rows are all-zero, flatten
// (the reference tests `word in dict` for up to 10 freshly sliced substrings per character; the author's own attempt
// at a faster path, data/trie.py, is unfinished).
//
// Here the vocabulary is a trie over Unicode code points stored in one open-addressing hash table
// (key = parent node << 21 | code point): the scan from a start character walks at most 10 edges and stops at the first
// missing edge, so a sentence costs O(L * depth reached), no substring is materialised, and sentences are processed by a
// pool of host threads writing straight into the caller's [n_sent, max_seq_len, 40] id / weight arrays — the layout the
// kernel ner_softlexicon_pool_fwd consumes.  Host-only code: no CUDA call is made in this file.
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "ner_b200.h"

namespace {
constexpr int kMaxWordLen = 10;   // MaxWordLen    data/word_enhance.py:32
constexpr int kSlots = 10;        // MaxLexiconLen data/word_enhance.py:33
constexpr int kGroups = 4;        // B, M, E, S in the order build_soft_lexicon creates the dict
enum { G_B = 0, G_M = 1, G_E = 2, G_S = 3 };

inline uint64_t mix(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
  return x;
}
}  // namespace

struct ner_lexicon {
  std::vector<uint64_t> keys;     // 0 = empty slot; key = ((node + 1) << 21) | code point
  std::vector<int32_t> child;
  uint64_t mask = 0;
  std::vector<int32_t> node_word;  // word id ending at this node, -1 if none
  std::vector<double> freq;        // [n_words + 2]: words, <None>, <PAD>
  int32_t n_words = 0;

  int32_t find(int32_t node, uint32_t cp) const {
    const uint64_t key = ((uint64_t)(node + 1) << 21) | cp;
    for (uint64_t h = mix(key) & mask;; h = (h + 1) & mask) {
      if (keys[h] == key) return child[h];
      if (keys[h] == 0) return -1;
    }
  }
  int32_t find_or_add(int32_t node, uint32_t cp) {
    const uint64_t key = ((uint64_t)(node + 1) << 21) | cp;
    for (uint64_t h = mix(key) & mask;; h = (h + 1) & mask) {
      if (keys[h] == key) return child[h];
      if (keys[h] == 0) {
        keys[h] = key;
        child[h] = (int32_t)node_word.size();
        node_word.push_back(-1);
        return child[h];
      }
    }
  }
};

extern "C" ner_lexicon* ner_lexicon_create(const uint32_t* word_codepoints_host, const int64_t* word_offsets_host,
                                           const double* freq_host, int n_words) {
  if (n_words < 0 || (n_words > 0 && (!word_codepoints_host || !word_offsets_host)) || !freq_host) return nullptr;
  try {
    ner_lexicon* lx = new ner_lexicon();
    lx->n_words = n_words;
    lx->freq.assign(freq_host, freq_host + n_words + 2);
    const int64_t total = n_words ? word_offsets_host[n_words] : 0;
    uint64_t cap = 64;
    while (cap < (uint64_t)total * 2 + 16) cap <<= 1;
    lx->keys.assign(cap, 0);
    lx->child.assign(cap, -1);
    lx->mask = cap - 1;
    lx->node_word.reserve((size_t)total + 1);
    lx->node_word.push_back(-1);   // root
    for (int w = 0; w < n_words; ++w) {
      const int64_t a = word_offsets_host[w], b = word_offsets_host[w + 1];
      if (b <= a) continue;          // the empty string matches no substring
      int32_t node = 0;
      for (int64_t i = a; i < b; ++i) {
        if (word_codepoints_host[i] >= (1u << 21)) { delete lx; return nullptr; }
        node = lx->find_or_add(node, word_codepoints_host[i]);
      }
      if (lx->node_word[node] < 0) lx->node_word[node] = w;   // a repeated word keeps its first id (dict semantics differ only
    }                                                          // for duplicates, which a vocabulary does not hold)
    return lx;
  } catch (...) {
    return nullptr;
  }
}

extern "C" void ner_lexicon_destroy(ner_lexicon* lx) { delete lx; }

extern "C" int64_t ner_lexicon_num_nodes(const ner_lexicon* lx) { return lx ? (int64_t)lx->node_word.size() : -1; }

namespace {
inline void add_unique(std::vector<int32_t>& v, int32_t id) {
  for (int32_t x : v)
    if (x == id) return;
  v.push_back(id);
}

void build_one(const ner_lexicon& lx, const uint32_t* cp, int n, const int32_t* tok_len, int n_tok, int L, int bert_mode,
               int32_t* ids, float* wts, std::vector<std::vector<int32_t>>& g, std::vector<std::vector<int32_t>>& merged) {
  const int row_w = kGroups * kSlots;
  std::memset(ids, 0, sizeof(int32_t) * (size_t)L * row_w);
  std::memset(wts, 0, sizeof(float) * (size_t)L * row_w);
  const int32_t none_id = lx.n_words, pad_id = lx.n_words + 1;
  if ((int)g.size() < n * kGroups) g.resize((size_t)n * kGroups);
  for (int i = 0; i < n * kGroups; ++i) g[i].clear();
  for (int i = 0; i < n; ++i) {
    int32_t node = 0;
    const int jend = std::min(i + kMaxWordLen, n);
    for (int j = i; j < jend; ++j) {
      node = lx.find(node, cp[j]);
      if (node < 0) break;
      const int32_t w = lx.node_word[node];
      if (w < 0) continue;
      if (j == i) {
        add_unique(g[i * kGroups + G_S], w);
      } else {
        add_unique(g[i * kGroups + G_B], w);
        add_unique(g[j * kGroups + G_E], w);
        for (int k = i + 1; k < j; ++k) add_unique(g[k * kGroups + G_M], w);
      }
    }
  }
  for (int i = 0; i < n * kGroups; ++i)
    if (g[i].empty()) g[i].push_back(none_id);   // "no matching E soft lexicon, fill in with None Token"

  // rows: one per character, or one per token when word pieces cover several characters (union, first-seen order)
  const std::vector<int32_t>* rows = g.data();
  int n_rows = n;
  if (tok_len && n_tok != n) {
    if ((int)merged.size() < n_tok * kGroups) merged.resize((size_t)n_tok * kGroups);
    int pos = 0;
    for (int t = 0; t < n_tok; ++t) {
      const int tl = std::max(tok_len[t], 1);
      for (int k = 0; k < kGroups; ++k) {
        auto& m = merged[t * kGroups + k];
        m.clear();
        for (int c = pos; c < std::min(pos + tl, n); ++c)
          for (int32_t id : g[c * kGroups + k]) add_unique(m, id);
        if (m.empty()) m.push_back(none_id);    // a token past the end of the text (the reference would raise)
      }
      pos += tl;
    }
    rows = merged.data();
    n_rows = n_tok;
  }

  const int keep = std::min(n_rows, bert_mode ? std::max(L - 2, 0) : L);
  const int shift = bert_mode ? 1 : 0;
  std::pair<int32_t, double> tmp[64];
  std::vector<std::pair<int32_t, double>> big;
  for (int r = 0; r < keep; ++r) {
    int32_t* rid = ids + (size_t)(r + shift) * row_w;
    float* rw = wts + (size_t)(r + shift) * row_w;
    double fr[kGroups * kSlots];
    double total = 0.0;
    for (int k = 0; k < kGroups; ++k) {
      const auto& v = rows[r * kGroups + k];
      const int cnt = (int)v.size();
      if (cnt <= kSlots) {
        for (int s = 0; s < kSlots; ++s) {
          const int32_t id = s < cnt ? v[s] : pad_id;
          rid[k * kSlots + s] = id;
          fr[k * kSlots + s] = lx.freq[id];
        }
      } else {   // keep the 10 most frequent; stable, as Python's sorted(..., reverse=True) is
        std::pair<int32_t, double>* p = tmp;
        if (cnt > 64) { big.resize(cnt); p = big.data(); }
        for (int s = 0; s < cnt; ++s) p[s] = {v[s], lx.freq[v[s]]};
        std::stable_sort(p, p + cnt, [](const std::pair<int32_t, double>& a, const std::pair<int32_t, double>& b) { return a.second > b.second; });
        for (int s = 0; s < kSlots; ++s) { rid[k * kSlots + s] = p[s].first; fr[k * kSlots + s] = p[s].second; }
      }
      for (int s = 0; s < kSlots; ++s) total += fr[k * kSlots + s];
    }
    for (int s = 0; s < row_w; ++s) rw[s] = (float)(fr[s] / total);
  }
}
}  // namespace

extern "C" int ner_lexicon_build(const ner_lexicon* lx, const uint32_t* codepoints_host, const int64_t* sent_offsets_host,
                                 int n_sent, const int32_t* tok_len_host, const int64_t* tok_offsets_host, int max_seq_len,
                                 int bert_mode, int32_t* ids_out_host, float* weights_out_host, int n_threads) {
  if (!lx || !sent_offsets_host || !ids_out_host || !weights_out_host || n_sent < 0 || max_seq_len < 1) return NER_ERR_INVALID_ARG;
  if ((tok_len_host == nullptr) != (tok_offsets_host == nullptr)) return NER_ERR_INVALID_ARG;
  if (n_sent == 0) return NER_OK;
  if (!codepoints_host && sent_offsets_host[n_sent] > 0) return NER_ERR_INVALID_ARG;
  const size_t row = (size_t)max_seq_len * kGroups * kSlots;
  int nt = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
  nt = std::max(1, std::min(nt, std::min(n_sent, 256)));
  std::atomic<int> next(0), failed(0);
  auto work = [&]() {
    try {
      std::vector<std::vector<int32_t>> g, merged;
      for (;;) {
        const int s0 = next.fetch_add(64);
        if (s0 >= n_sent) break;
        for (int s = s0; s < std::min(s0 + 64, n_sent); ++s) {
          const int64_t a = sent_offsets_host[s], b = sent_offsets_host[s + 1];
          const int32_t* tl = tok_len_host ? tok_len_host + tok_offsets_host[s] : nullptr;
          const int n_tok = tok_len_host ? (int)(tok_offsets_host[s + 1] - tok_offsets_host[s]) : 0;
          build_one(*lx, codepoints_host + a, (int)(b - a), tl, n_tok, max_seq_len, bert_mode, ids_out_host + s * row,
                    weights_out_host + s * row, g, merged);
        }
      }
    } catch (...) {
      failed.store(1);
    }
  };
  if (nt == 1) {
    work();
  } else {
    std::vector<std::thread> pool;
    try {
      for (int t = 0; t < nt; ++t) pool.emplace_back(work);
    } catch (...) {   // could not start every thread: the started ones (or this thread, below) finish the job
    }
    for (auto& th : pool) th.join();
    if (pool.empty()) work();
  }
  return failed.load() ? NER_ERR_UNSUPPORTED : NER_OK;
}

namespace {
// Lattice lists of one sentence: per start b, the 2..10-character vocabulary words at [b, b + n), trie order (increasing
// length), cut to the Kw most frequent (stable).  -> number of matches the cut dropped.
int64_t build_lattice_one(const ner_lexicon& lx, const uint32_t* cp, int n, int L, int Kw, int32_t* ids, int32_t* lens) {
  const int32_t pad_id = lx.n_words + 1;
  for (int s = 0; s < L * Kw; ++s) { ids[s] = pad_id; lens[s] = 0; }
  const int n_keep = std::min(n, L);
  int64_t dropped = 0;
  std::pair<int32_t, int32_t> found[kMaxWordLen];   // (word id, length)
  for (int b = 0; b < n_keep; ++b) {
    int cnt = 0;
    int32_t node = 0;
    const int jend = std::min(b + kMaxWordLen, n_keep);
    for (int j = b; j < jend; ++j) {
      node = lx.find(node, cp[j]);
      if (node < 0) break;
      const int32_t w = lx.node_word[node];
      if (w >= 0 && j > b) found[cnt++] = {w, j - b + 1};
    }
    if (cnt > Kw) {
      std::stable_sort(found, found + cnt, [&](const std::pair<int32_t, int32_t>& a, const std::pair<int32_t, int32_t>& c) {
        return lx.freq[a.first] > lx.freq[c.first];
      });
      dropped += cnt - Kw;
      cnt = Kw;
    }
    for (int k = 0; k < cnt; ++k) { ids[b * Kw + k] = found[k].first; lens[b * Kw + k] = found[k].second; }
  }
  return dropped;
}
}  // namespace

extern "C" int ner_lexicon_build_lattice(const ner_lexicon* lx, const uint32_t* codepoints_host,
                                         const int64_t* sent_offsets_host, int n_sent, int max_seq_len, int Kw,
                                         int32_t* ids_out_host, int32_t* lens_out_host, int64_t* dropped_out_host,
                                         int n_threads) {
  if (!lx || !sent_offsets_host || !ids_out_host || !lens_out_host || n_sent < 0 || max_seq_len < 1) return NER_ERR_INVALID_ARG;
  if (Kw < 1 || Kw > 8) return NER_ERR_INVALID_ARG;
  if (dropped_out_host) *dropped_out_host = 0;
  if (n_sent == 0) return NER_OK;
  if (!codepoints_host && sent_offsets_host[n_sent] > 0) return NER_ERR_INVALID_ARG;
  const size_t row = (size_t)max_seq_len * Kw;
  int nt = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
  nt = std::max(1, std::min(nt, std::min(n_sent, 256)));
  std::atomic<int> next(0);
  std::atomic<int64_t> dropped(0);
  auto work = [&]() {
    int64_t mine = 0;
    for (;;) {
      const int s0 = next.fetch_add(64);
      if (s0 >= n_sent) break;
      for (int s = s0; s < std::min(s0 + 64, n_sent); ++s) {
        const int64_t a = sent_offsets_host[s], b = sent_offsets_host[s + 1];
        mine += build_lattice_one(*lx, codepoints_host + a, (int)(b - a), max_seq_len, Kw, ids_out_host + s * row,
                                  lens_out_host + s * row);
      }
    }
    dropped.fetch_add(mine);
  };
  if (nt == 1) {
    work();
  } else {
    std::vector<std::thread> pool;
    try {
      for (int t = 0; t < nt; ++t) pool.emplace_back(work);
    } catch (...) {   // could not start every thread: the started ones (or this thread, below) finish the job
    }
    for (auto& th : pool) th.join();
    if (pool.empty()) work();
  }
  if (dropped_out_host) *dropped_out_host = dropped.load();
  return NER_OK;
}
