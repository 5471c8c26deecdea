// Raw text -> BasicProc.build_seq_feature features on the device (the serving head of InferHelper.infer_batch).
//
// ner_featurize_wordpiece restates FullTokenizer.tokenize (BasicTokenizer + WordPiece, data/tokenizer.py) followed by
// BasicProc.format_sequence; ner_featurize_chars restates TokenizerAdapter.tokenize + format_sequence.  Every Unicode
// property the host tokenizer asks unicodedata / str for comes from tables the caller builds from the running Python
// (data/device_featurize.py), so the two agree by construction; this file holds only the control flow.
//
// One thread per text.  A thread streams its text once, left to right, and stops as soon as its row holds L - 2 (L)
// tokens.  WordPiece needs random access to the current punctuation-split token only, which is at most 200 code points
// long (a longer one is [UNK] whatever it holds), so shared memory is 201 words per thread whatever the text's length.
//
// Exactness of the streamed BasicTokenizer (do_lower_case):
//   - lower() is per code point except for U+03A3, whose Final_Sigma context is read off the raw text: the last
//     non-case-ignorable character of the word before it (a running flag) and the first one after it (a forward scan
//     that stops at the word's end);
//   - NFD(lower(word)) = canonical reordering of the concatenated per-code-point expansions NFD(lower(c)); the Mn strip
//     commutes with the (stable) reordering, so a surviving mark with a nonzero combining class is insertion-sorted into
//     the current run of the token buffer, a run being cut by every class-0 code point, kept or stripped;
//   - no punctuation code point has a nonzero combining class (checked when the tables are built), so a punctuation
//     code point closes the buffered token before any later mark could move across it.
#include "common.cuh"

namespace {
constexpr int kThreads = 32;          // texts per CTA of the WordPiece kernel
constexpr int kMaxWord = 200;         // WordpieceTokenizer.max_input_chars_per_word
constexpr int kCharThreads = 128;

// per-code-point record: bits 0-7 flags, 8-15 canonical combining class, 16-31 index into the expansion table (0: the
// code point maps to itself)
enum : uint32_t {
  F_CONTROL = 1,      // _is_control
  F_WHITESPACE = 2,   // _is_whitespace
  F_SPACE = 4,        // str.isspace (what split() / strip() use)
  F_PUNCT = 8,        // _is_punctuation
  F_CJK = 16,         // _is_chinese_char
  F_MN = 32,          // category Mn
  F_CASED = 64,       // cased and not case-ignorable
  F_IGNORABLE = 128,  // case-ignorable
};

struct Uni {
  const uint16_t* stage1;
  const uint32_t* stage2;
  __device__ __forceinline__ uint32_t operator()(uint32_t cp) const {
    return __ldg(stage2 + ((uint32_t)__ldg(stage1 + (cp >> 8)) << 8) + (cp & 0xFFu));
  }
};

struct Vocab {
  const int32_t* slots;     // [n_slots] entry index or -1, n_slots a power of two
  const int32_t* entries;   // [n_keys, 3]: blob offset, byte length, id
  const uint8_t* blob;
  uint32_t slot_mask;
};

// Python's encode('utf-8', 'surrogatepass') reversed; a malformed sequence reads as U+FFFD and never runs past `end`.
__device__ __forceinline__ uint32_t next_cp(const uint8_t* __restrict__ s, int64_t& i, int64_t end) {
  uint32_t c = s[i++];
  if (c < 0x80u) return c;
  int n;
  if ((c & 0xE0u) == 0xC0u) { n = 1; c &= 0x1Fu; }
  else if ((c & 0xF0u) == 0xE0u) { n = 2; c &= 0x0Fu; }
  else if ((c & 0xF8u) == 0xF0u) { n = 3; c &= 0x07u; }
  else return 0xFFFDu;
  for (int k = 0; k < n; ++k) {
    if (i >= end || (s[i] & 0xC0u) != 0x80u) return 0xFFFDu;
    c = (c << 6) | (s[i++] & 0x3Fu);
  }
  return c > 0x10FFFFu ? 0xFFFDu : c;
}

__device__ __forceinline__ int utf8_bytes(uint32_t cp, uint8_t* out) {
  if (cp < 0x80u) { out[0] = (uint8_t)cp; return 1; }
  if (cp < 0x800u) { out[0] = (uint8_t)(0xC0u | (cp >> 6)); out[1] = (uint8_t)(0x80u | (cp & 0x3Fu)); return 2; }
  if (cp < 0x10000u) {
    out[0] = (uint8_t)(0xE0u | (cp >> 12)); out[1] = (uint8_t)(0x80u | ((cp >> 6) & 0x3Fu));
    out[2] = (uint8_t)(0x80u | (cp & 0x3Fu));
    return 3;
  }
  out[0] = (uint8_t)(0xF0u | (cp >> 18)); out[1] = (uint8_t)(0x80u | ((cp >> 12) & 0x3Fu));
  out[2] = (uint8_t)(0x80u | ((cp >> 6) & 0x3Fu)); out[3] = (uint8_t)(0x80u | (cp & 0x3Fu));
  return 4;
}

// Vocabulary id of ("##" if cont) + the code points cps[0..n) (low 21 bits of each word), or -1.  FNV-1a over the
// UTF-8 bytes, linear probing, every hit verified against the key's bytes.
__device__ int lookup(const Vocab& v, const uint32_t* cps, int n, bool cont) {
  uint32_t h = 2166136261u;
  int nbytes = 0;
  uint8_t u[4];
  if (cont) {
    h = (h ^ '#') * 16777619u;
    h = (h ^ '#') * 16777619u;
    nbytes = 2;
  }
  for (int k = 0; k < n; ++k) {
    const int m = utf8_bytes(cps[k] & 0x1FFFFFu, u);
    for (int j = 0; j < m; ++j) h = (h ^ u[j]) * 16777619u;
    nbytes += m;
  }
  for (uint32_t slot = h & v.slot_mask;; slot = (slot + 1) & v.slot_mask) {
    const int e = __ldg(v.slots + slot);
    if (e < 0) return -1;
    if (__ldg(v.entries + 3 * e + 1) != nbytes) continue;
    const uint8_t* key = v.blob + __ldg(v.entries + 3 * e);
    int at = 0;
    bool same = true;
    if (cont) { same = key[0] == '#' && key[1] == '#'; at = 2; }
    for (int k = 0; k < n && same; ++k) {
      const int m = utf8_bytes(cps[k] & 0x1FFFFFu, u);
      for (int j = 0; j < m; ++j) same = same && key[at + j] == u[j];
      at += m;
    }
    if (same) return __ldg(v.entries + 3 * e + 2);
  }
}

struct Row {
  int32_t* ids;
  int32_t* cursor;
  int n = 0;          // tokens written after [CLS]
  int cap;            // L - 2
  int fix_cursor = 0; // fix_tokens' cursor: characters of the tokens so far, [UNK] counting one
  int unk_id;

  __device__ void piece(int id, int len) {
    if (n >= cap) return;
    ids[1 + n] = id;
    cursor[1 + n] = -1;
    ++n;
    fix_cursor += len;
  }
  __device__ void unk() {
    if (n >= cap) return;
    ids[1 + n] = unk_id;
    cursor[1 + n] = fix_cursor;
    ++n;
    fix_cursor += 1;
  }
};

// WordpieceTokenizer.tokenize of one token held in buf[0..len) (len > kMaxWord: [UNK]).  Greedy longest match first;
// the pieces overwrite the consumed front of buf (piece k ends past index k) and are written to the row only once the
// whole token has matched, since one unmatched position makes the whole token a single [UNK].
__device__ void wordpiece(uint32_t* buf, int len, const Vocab& v, int max_piece, Row& row) {
  if (len > kMaxWord) { row.unk(); return; }
  int start = 0, k = 0;
  while (start < len) {
    int end = min(len, start + max_piece), id = -1;
    for (; end > start; --end) {
      id = lookup(v, buf + start, end - start, start > 0);
      if (id >= 0) break;
    }
    if (id < 0) { row.unk(); return; }
    buf[k++] = (uint32_t)id | ((uint32_t)(end - start) << 24);
    start = end;
  }
  for (int j = 0; j < k; ++j) row.piece((int)(buf[j] & 0xFFFFFFu), (int)(buf[j] >> 24));
}

// The punctuation-split token being built: code points in the low 21 bits, combining class in the top 8.
struct Token {
  uint32_t* buf;
  int len = 0, run = 0;   // run: first index a mark with a nonzero class may move to

  __device__ void push(uint32_t cp, uint32_t ccc) {
    if (len >= kMaxWord) { len = kMaxWord + 1; return; }   // [UNK] whatever else it holds
    int j = len++;
    if (ccc) {
      for (; j > run && (buf[j - 1] >> 24) > ccc; --j) buf[j] = buf[j - 1];
    } else {
      run = len;
    }
    buf[j] = cp | (ccc << 24);
  }
};

__global__ void __launch_bounds__(kThreads) featurize_wordpiece_kernel(
    const uint8_t* __restrict__ text, const int64_t* __restrict__ offsets, int B, int L, Uni uni,
    const uint32_t* __restrict__ expand, Vocab vocab, int max_piece, int lower, int cls_id, int sep_id, int pad_id,
    int unk_id, int32_t* __restrict__ token_ids, int32_t* __restrict__ mask, int32_t* __restrict__ segment_ids,
    int32_t* __restrict__ seq_len, int32_t* __restrict__ unk_cursor) {
  __shared__ uint32_t smem[kThreads * (kMaxWord + 1)];
  const int b = blockIdx.x * kThreads + threadIdx.x;
  if (b >= B) return;
  const size_t r0 = (size_t)b * L;
  Row row;
  row.ids = token_ids + r0;
  row.cursor = unk_cursor + r0;
  row.cap = L - 2;
  row.unk_id = unk_id;
  Token tok;
  tok.buf = smem + threadIdx.x * (kMaxWord + 1);

  auto flush = [&]() {
    if (tok.len) wordpiece(tok.buf, tok.len, vocab, max_piece, row);
    tok.len = tok.run = 0;
  };
  // one code point of the lowered / decomposed word (or of the raw word without lower-casing)
  auto emit = [&](uint32_t cp, uint32_t rec) {
    if (lower && (rec & F_MN)) {
      if (((rec >> 8) & 0xFFu) == 0) tok.run = tok.len;
      return;
    }
    if (rec & F_PUNCT) {
      flush();
      tok.push(cp, 0);
      flush();
      return;
    }
    tok.push(cp, lower ? (rec >> 8) & 0xFFu : 0u);
  };

  int64_t i = offsets[b];
  const int64_t end = offsets[b + 1];
  bool prev_cased = false;   // Final_Sigma look-behind: the word's last non-case-ignorable character was cased
  while (i < end && row.n < row.cap) {
    const uint32_t cp = next_cp(text, i, end);
    if (cp == 0 || cp == 0xFFFDu) continue;
    const uint32_t rec = uni(cp);
    if (rec & F_CONTROL) continue;
    if (rec & (F_WHITESPACE | F_SPACE | F_CJK)) {   // _clean_text / _tokenize_chinese_chars spaces, then split()
      flush();
      prev_cased = false;
      if (!(rec & F_CJK)) continue;
    }
    if (!lower) {
      emit(cp, rec);
    } else if (cp == 0x3A3u) {
      bool final_sigma = prev_cased;
      for (int64_t j = i; final_sigma && j < end;) {   // look-ahead to the end of the word
        const uint32_t c = next_cp(text, j, end);
        if (c == 0 || c == 0xFFFDu) continue;
        const uint32_t r = uni(c);
        if (r & F_CONTROL) continue;
        if (r & (F_WHITESPACE | F_SPACE | F_CJK)) break;
        if (r & F_IGNORABLE) continue;
        final_sigma = !(r & F_CASED);
        break;
      }
      const uint32_t s = final_sigma ? 0x3C2u : 0x3C3u;
      emit(s, uni(s));
    } else if (const uint32_t x = rec >> 16) {
      for (int k = 0; k < 4; ++k) {
        const uint32_t c = __ldg(expand + 4 * x + k);
        if (!c) break;
        emit(c, uni(c));
      }
    } else {
      emit(cp, rec);
    }
    if (!(rec & F_IGNORABLE)) prev_cased = (rec & F_CASED) != 0;
    if (rec & F_CJK) {
      flush();
      prev_cased = false;
    }
  }
  flush();

  const int n = row.n + 2;
  token_ids[r0] = cls_id;
  unk_cursor[r0] = -1;
  token_ids[r0 + n - 1] = sep_id;
  unk_cursor[r0 + n - 1] = -1;
  for (int p = 0; p < L; ++p) {
    if (p >= n) {
      token_ids[r0 + p] = pad_id;
      unk_cursor[r0 + p] = -1;
    }
    mask[r0 + p] = p < n;
    segment_ids[r0 + p] = 0;
  }
  seq_len[b] = n;
}

__global__ void __launch_bounds__(kCharThreads) featurize_chars_kernel(
    const uint8_t* __restrict__ text, const int64_t* __restrict__ offsets, int B, int L, Uni uni, Vocab vocab,
    int pad_id, int unk_id, int32_t* __restrict__ token_ids, int32_t* __restrict__ mask,
    int32_t* __restrict__ segment_ids, int32_t* __restrict__ seq_len, int32_t* __restrict__ unk_cursor) {
  const int b = blockIdx.x * kCharThreads + threadIdx.x;
  if (b >= B) return;
  const size_t r0 = (size_t)b * L;
  int64_t i = offsets[b];
  const int64_t end = offsets[b + 1];
  int n = 0, at = 0;
  for (; i < end && n < L; ++at) {
    uint32_t cp = next_cp(text, i, end);
    if (uni(cp) & F_SPACE) continue;                     // str.strip() empties it
    if (cp == 0x3000u) cp = 0x20u;                       // TokenizerAdapter.full2half
    else if (cp >= 0xFF01u && cp <= 0xFF5Eu) cp -= 0xFEE0u;
    const int id = lookup(vocab, &cp, 1, false);
    token_ids[r0 + n] = id >= 0 ? id : unk_id;
    unk_cursor[r0 + n] = id >= 0 ? -1 : at;
    ++n;
  }
  for (int p = 0; p < L; ++p) {
    if (p >= n) {
      token_ids[r0 + p] = pad_id;
      unk_cursor[r0 + p] = -1;
    }
    mask[r0 + p] = p < n;
    segment_ids[r0 + p] = 0;
  }
  seq_len[b] = n;
}

// Shared argument checks; every one runs before any CUDA call.
int check_common(const uint8_t* text, const int64_t* offsets, const int64_t* offsets_host, int B, int L,
                 const uint16_t* stage1, const uint32_t* stage2, const int32_t* slots, int n_slots,
                 const int32_t* entries, const uint8_t* blob, int pad_id, int unk_id, const int32_t* token_ids,
                 const int32_t* mask, const int32_t* segment_ids, const int32_t* seq_len, const int32_t* unk_cursor) {
  if (B < 0 || L < 1) return NER_ERR_INVALID_ARG;
  if (B == 0) return NER_OK;
  if (!text || !offsets || !offsets_host || !stage1 || !stage2 || !slots || !entries || !blob || !token_ids || !mask ||
      !segment_ids || !seq_len || !unk_cursor)
    return NER_ERR_INVALID_ARG;
  if (n_slots < 1 || (n_slots & (n_slots - 1)) || pad_id < 0 || unk_id < 0) return NER_ERR_INVALID_ARG;
  if (offsets_host[0] != 0) return NER_ERR_INVALID_ARG;
  for (int b = 0; b < B; ++b)
    if (offsets_host[b + 1] < offsets_host[b]) return NER_ERR_INVALID_ARG;
  if ((int64_t)B * L >= ((int64_t)1 << 31)) return NER_ERR_UNSUPPORTED;
  return 1;
}
}  // namespace

extern "C" int ner_featurize_wordpiece(const uint8_t* text, const int64_t* offsets, const int64_t* offsets_host, int B,
                                       int L, const uint16_t* uni_stage1, const uint32_t* uni_stage2,
                                       const uint32_t* uni_expand, const int32_t* slots, int n_slots,
                                       const int32_t* entries, const uint8_t* blob, int max_piece, int do_lower_case,
                                       int cls_id, int sep_id, int pad_id, int unk_id, int32_t* token_ids,
                                       int32_t* mask, int32_t* segment_ids, int32_t* seq_len, int32_t* unk_cursor,
                                       ner_stream_t stream) {
  if (L < 2) return NER_ERR_INVALID_ARG;                 // [CLS] and [SEP] always fit
  const int st = check_common(text, offsets, offsets_host, B, L, uni_stage1, uni_stage2, slots, n_slots, entries,
                              blob, pad_id, unk_id, token_ids, mask, segment_ids, seq_len, unk_cursor);
  if (st != 1) return st;
  if (!uni_expand || max_piece < 1 || cls_id < 0 || sep_id < 0) return NER_ERR_INVALID_ARG;
  if (max_piece > kMaxWord) max_piece = kMaxWord;
  const Uni uni{uni_stage1, uni_stage2};
  const Vocab vocab{slots, entries, blob, (uint32_t)(n_slots - 1)};
  featurize_wordpiece_kernel<<<(B + kThreads - 1) / kThreads, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      text, offsets, B, L, uni, uni_expand, vocab, max_piece, do_lower_case != 0, cls_id, sep_id, pad_id, unk_id,
      token_ids, mask, segment_ids, seq_len, unk_cursor);
  return ner_launch_status();
}

extern "C" int ner_featurize_chars(const uint8_t* text, const int64_t* offsets, const int64_t* offsets_host, int B,
                                   int L, const uint16_t* uni_stage1, const uint32_t* uni_stage2, const int32_t* slots,
                                   int n_slots, const int32_t* entries, const uint8_t* blob, int pad_id, int unk_id,
                                   int32_t* token_ids, int32_t* mask, int32_t* segment_ids, int32_t* seq_len,
                                   int32_t* unk_cursor, ner_stream_t stream) {
  const int st = check_common(text, offsets, offsets_host, B, L, uni_stage1, uni_stage2, slots, n_slots, entries,
                              blob, pad_id, unk_id, token_ids, mask, segment_ids, seq_len, unk_cursor);
  if (st != 1) return st;
  const Uni uni{uni_stage1, uni_stage2};
  const Vocab vocab{slots, entries, blob, (uint32_t)(n_slots - 1)};
  featurize_chars_kernel<<<(B + kCharThreads - 1) / kCharThreads, kCharThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      text, offsets, B, L, uni, vocab, pad_id, unk_id, token_ids, mask, segment_ids, seq_len, unk_cursor);
  return ner_launch_status();
}
