// The text front end on the device (DESIGN.md section 23): UTF-8 upload and checks, Trim / LowerCase, Tokenizer, term frequencies
// over tokens or n-grams, CommonSparseFeatures / AllSparseFeatures, SparseFeatureVectorizer and (NGrams)HashingTF.
//
// Work runs over bytes, tokens or terms, never one thread per document over its contents: a 100 KB document sits next to 1 KB ones.
// Boundaries and output positions come from flags and CUB scans; every grouping is a stable CUB radix sort (least significant key
// first) followed by adjacent compares, so no output is ordered by atomics and a rerun repeats bit for bit.  Terms are identified by
// their bytes: a token's 64-bit content hash orders the vocabulary sort, equal hashes are compared byte by byte, and n-gram keys are
// the packed vocabulary ids of their tokens.
#include "engine.h"
#include "lower_table.h"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <thrust/execution_policy.h>
#include <thrust/iterator/transform_iterator.h>
#include <thrust/sort.h>

#include <algorithm>
#include <cmath>
#include <limits>
#include <vector>

namespace ks {

enum TextKind { TX_TEXT = 0, TX_TOKENS = 1, TX_TF = 2, TX_SPACE = 3 };

struct TextObj {
  int kind = TX_TEXT;
  std::shared_ptr<TextObj> src;  // tokens: the text their bytes lie in; tf / space: the tokens their terms are made of
  // text: the UTF-8 bytes.  doc_off: byte offsets (text), token offsets (tokens), term offsets (tf); n_docs + 1 entries
  DevBuf bytes;
  int64_t n_bytes = 0;
  DevBuf doc_off;
  int64_t n_docs = 0;
  // tokens: byte ranges into src->bytes, String.hashCode, content hash; vocabulary ids (built on first use) and their count
  DevBuf tb, te, jh, ch, ids;
  int64_t n_tok = 0, vocab = -1;
  // tf / space: term t is tokens [first[t], first[t] + max(order[t], 1)) of src, a String at order 0; tf: count and value per term
  DevBuf first, order, count, value;
  int64_t n_terms = 0, max_count = 0;
  DevBuf sh, sf;  // space: the features' content hashes, ascending, and the feature of each
};

namespace {

constexpr int kT = 256;

unsigned grid_of(int64_t n) {
  return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((n + kT - 1) / kT, 132 * 32)));
}
#define TX_LOOP(i, n) for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < (n); i += static_cast<int64_t>(gridDim.x) * blockDim.x)

int bits_for(uint64_t max_value) {  // bits to hold every value in [0, max_value]
  int b = 0;
  while (b < 64 && (max_value >> b) != 0) ++b;
  return b;
}

template <class T>
T read1(const DevBuf& b, int64_t i, cudaStream_t st) {
  T v{};
  KS_CUDA(cudaMemcpyAsync(&v, b.as<T>() + i, sizeof(T), cudaMemcpyDeviceToHost, st));
  KS_CUDA(cudaStreamSynchronize(st));
  return v;
}

// ------------------------------------------------------------------------------------ device helpers
__device__ __forceinline__ bool is_cont(uint8_t b) { return (b & 0xC0) == 0x80; }
__device__ __forceinline__ int u8_len(uint8_t b) {
  return b < 0x80 ? 1 : (b >> 5) == 6 ? 2 : (b >> 4) == 14 ? 3 : (b >> 3) == 30 ? 4 : 0;
}
__device__ __forceinline__ uint32_t u8_decode(const uint8_t* p, int len) {
  if (len == 1) return p[0];
  if (len == 2) return ((p[0] & 0x1Fu) << 6) | (p[1] & 0x3Fu);
  if (len == 3) return ((p[0] & 0x0Fu) << 12) | ((p[1] & 0x3Fu) << 6) | (p[2] & 0x3Fu);
  return ((p[0] & 0x07u) << 18) | ((p[1] & 0x3Fu) << 12) | ((p[2] & 0x3Fu) << 6) | (p[3] & 0x3Fu);
}
__device__ __forceinline__ int u8_enc_len(uint32_t c) { return c < 0x80 ? 1 : c < 0x800 ? 2 : c < 0x10000 ? 3 : 4; }
__device__ __forceinline__ void u8_encode(uint32_t c, uint8_t* o) {
  if (c < 0x80) {
    o[0] = static_cast<uint8_t>(c);
  } else if (c < 0x800) {
    o[0] = static_cast<uint8_t>(0xC0 | (c >> 6));
    o[1] = static_cast<uint8_t>(0x80 | (c & 0x3F));
  } else if (c < 0x10000) {
    o[0] = static_cast<uint8_t>(0xE0 | (c >> 12));
    o[1] = static_cast<uint8_t>(0x80 | ((c >> 6) & 0x3F));
    o[2] = static_cast<uint8_t>(0x80 | (c & 0x3F));
  } else {
    o[0] = static_cast<uint8_t>(0xF0 | (c >> 18));
    o[1] = static_cast<uint8_t>(0x80 | ((c >> 12) & 0x3F));
    o[2] = static_cast<uint8_t>(0x80 | ((c >> 6) & 0x3F));
    o[3] = static_cast<uint8_t>(0x80 | (c & 0x3F));
  }
}
__device__ __forceinline__ uint32_t lower_cp(uint32_t c) {
  if (c < 0x80) return (c >= 'A' && c <= 'Z') ? c + 32 : c;
  int lo = 0, hi = kLowerCount;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (kLowerFrom[mid] < c) lo = mid + 1;
    else hi = mid;
  }
  return (lo < kLowerCount && kLowerFrom[lo] == c) ? kLowerTo[lo] : c;
}
// \p{Punct} (the 32 ASCII punctuation characters) and \s ([ \t\n\x0B\f\r]) of java.util.regex
__device__ __forceinline__ bool is_sep(uint8_t b) {
  return (b >= 0x21 && b <= 0x2F) || (b >= 0x3A && b <= 0x40) || (b >= 0x5B && b <= 0x60) || (b >= 0x7B && b <= 0x7E) || b == ' ' ||
         (b >= 0x09 && b <= 0x0D);
}
__device__ __forceinline__ uint64_t mix64(uint64_t z) {  // splitmix64's finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t hash_mask(int bits) { return bits >= 64 ? ~0ull : ((1ull << bits) - 1); }
// the last d in [0, n) with off[d] <= i (the document of byte / token / term i; empty documents before it are skipped)
__device__ __forceinline__ int64_t owner_of(const int64_t* __restrict__ off, int64_t n, int64_t i) {
  int64_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (off[mid] <= i) lo = mid;
    else hi = mid;
  }
  return lo;
}
// Scala's MurmurHash3 steps, as NGramsHashingTF.scala restates them
__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
__device__ __forceinline__ uint32_t mm_mix(uint32_t h, uint32_t data) {
  uint32_t k = data * 0xcc9e2d51u;
  k = rotl32(k, 15) * 0x1b873593u;
  h ^= k;
  return rotl32(h, 13) * 5u + 0xe6546b64u;
}
__device__ __forceinline__ uint32_t mm_finalize(uint32_t h, uint32_t len) {
  h ^= len;
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return h;
}
constexpr uint32_t kSeqSeed = 83007u;  // "Seq".hashCode
__device__ __forceinline__ int32_t non_negative_mod(int32_t x, int32_t m) {
  const int32_t r = x % m;  // C++ and Java % both truncate toward zero
  return r + (r < 0 ? m : 0);
}
// content hash of term (first, order) over the tokens' content hashes
__device__ __forceinline__ uint64_t term_hash(const uint64_t* __restrict__ ch, int64_t first, int order, uint64_t mask) {
  uint64_t h = mix64(0x9E3779B97F4A7C15ull + static_cast<uint64_t>(order));
  const int n = order > 0 ? order : 1;
  for (int j = 0; j < n; ++j) h = mix64(h ^ ch[first + j]);
  return h & mask;
}
__device__ __forceinline__ bool same_bytes(const uint8_t* a, int64_t ab, int64_t ae, const uint8_t* b, int64_t bb, int64_t be) {
  if (ae - ab != be - bb) return false;
  for (int64_t k = 0; k < ae - ab; ++k)
    if (a[ab + k] != b[bb + k]) return false;
  return true;
}

// ------------------------------------------------------------------------------------ kernels
__global__ void tx_doc_start_kernel(const int64_t* __restrict__ off, int64_t n_docs, int64_t n, uint8_t* __restrict__ start) {
  TX_LOOP(d, n_docs) if (off[d] < n) start[off[d]] = 1;  // documents that share a start write the same value
}
// flag |= 1 for a byte that is not part of a valid UTF-8 sequence within its document
__global__ void tx_validate_kernel(const uint8_t* __restrict__ s, int64_t n, const uint8_t* __restrict__ start, unsigned* flag) {
  TX_LOOP(i, n) {
    const uint8_t b = s[i];
    bool bad = false;
    if (is_cont(b)) {
      int k = 1;
      while (k <= 3 && i - k >= 0 && is_cont(s[i - k])) ++k;
      bad = start[i] || k > 3 || i - k < 0 || u8_len(s[i - k]) <= k;
      for (int q = 1; q < k && !bad; ++q) bad = start[i - q + 1] != 0;  // no document starts between the lead byte and this one
    } else {
      const int L = u8_len(b);
      bad = L == 0;
      for (int k = 1; k < L && !bad; ++k) bad = i + k >= n || start[i + k] || !is_cont(s[i + k]);
      if (!bad && L > 1) {
        const uint32_t c = u8_decode(s + i, L);
        bad = (L == 2 && c < 0x80) || (L == 3 && c < 0x800) || (L == 4 && c < 0x10000) || (c >= 0xD800 && c < 0xE000) || c > 0x10FFFF;
      }
    }
    if (bad) atomicOr(flag, 1u);
  }
}
// Trim: the leading and trailing bytes <= 0x20 of each document are dropped (such code points are single bytes)
__global__ void tx_trim_kernel(const uint8_t* __restrict__ s, const int64_t* __restrict__ off, int64_t n_docs, uint8_t* __restrict__ drop) {
  TX_LOOP(d, n_docs) {
    const int64_t b = off[d], e = off[d + 1];
    int64_t a = b;
    while (a < e && s[a] <= 0x20) drop[a++] = 1;
    for (int64_t z = e - 1; z >= a && s[z] <= 0x20; --z) drop[z] = 1;
  }
}
// output bytes of the code point that starts at byte i (0 for continuation and dropped bytes)
__global__ void tx_out_len_kernel(const uint8_t* __restrict__ s, int64_t n, const uint8_t* __restrict__ drop, int lower, uint8_t* __restrict__ len) {
  TX_LOOP(i, n) {
    const uint8_t b = s[i];
    int l = 0;
    if (!is_cont(b) && !(drop && drop[i])) {
      l = u8_len(b);
      if (lower) {
        const uint32_t c = u8_decode(s + i, l);
        l = c == 0x130 ? 3 : u8_enc_len(lower_cp(c));
      }
    }
    len[i] = static_cast<uint8_t>(l);
  }
}
__global__ void tx_write_kernel(const uint8_t* __restrict__ s, int64_t n, const uint8_t* __restrict__ len, const int64_t* __restrict__ pos,
                                int lower, uint8_t* __restrict__ out) {
  TX_LOOP(i, n) {
    if (!len[i]) continue;
    const int l = u8_len(s[i]);
    uint8_t* o = out + pos[i];
    if (!lower) {
      for (int k = 0; k < l; ++k) o[k] = s[i + k];
      continue;
    }
    const uint32_t c = u8_decode(s + i, l);
    if (c == 0x130) {  // U+0069 U+0307, as Java lowers it
      o[0] = 0x69;
      o[1] = 0xCC;
      o[2] = 0x87;
    } else {
      u8_encode(lower_cp(c), o);
    }
  }
}
__global__ void tx_gather_offsets_kernel(const int64_t* __restrict__ off, int64_t n, const int64_t* __restrict__ pos, int64_t* __restrict__ out) {
  TX_LOOP(d, n + 1) out[d] = pos[off[d]];
}
__global__ void tx_run_start_kernel(const uint8_t* __restrict__ s, int64_t n, const uint8_t* __restrict__ start, uint8_t* __restrict__ rs) {
  TX_LOOP(i, n) rs[i] = !is_sep(s[i]) && (start[i] || (i > 0 && is_sep(s[i - 1])));
}
// tokens of document d: its runs of non-separators, plus one empty token for an empty document or a leading separator (when a run follows)
__global__ void tx_doc_tokens_kernel(const uint8_t* __restrict__ s, const int64_t* __restrict__ off, int64_t n_docs,
                                     const int64_t* __restrict__ runs, int64_t* __restrict__ cnt) {
  TX_LOOP(d, n_docs) {
    const int64_t b = off[d], e = off[d + 1], r = runs[e] - runs[b];
    cnt[d] = r + ((b == e || (is_sep(s[b]) && r > 0)) ? 1 : 0);
  }
}
__global__ void tx_empty_tokens_kernel(const uint8_t* __restrict__ s, const int64_t* __restrict__ off, int64_t n_docs,
                                       const int64_t* __restrict__ runs, const int64_t* __restrict__ toff, int64_t* __restrict__ tb,
                                       int64_t* __restrict__ te) {
  TX_LOOP(d, n_docs) {
    const int64_t b = off[d], e = off[d + 1];
    if (b == e || (is_sep(s[b]) && runs[e] > runs[b])) tb[toff[d]] = te[toff[d]] = b;
  }
}
__global__ void tx_token_bounds_kernel(const uint8_t* __restrict__ s, int64_t n, const uint8_t* __restrict__ start, const int64_t* __restrict__ off,
                                       int64_t n_docs, const int64_t* __restrict__ runs, const int64_t* __restrict__ toff, int64_t* __restrict__ tb,
                                       int64_t* __restrict__ te) {
  TX_LOOP(i, n) {
    if (is_sep(s[i])) continue;
    const bool first = start[i] || (i > 0 && is_sep(s[i - 1]));
    const bool last = i + 1 == n || start[i + 1] || is_sep(s[i + 1]);
    if (!first && !last) continue;
    const int64_t d = owner_of(off, n_docs, i), b = off[d];
    const int64_t base = toff[d] + (is_sep(s[b]) ? 1 : 0) - runs[b];
    if (first) tb[base + runs[i]] = i;
    if (last) te[base + runs[i + 1] - 1] = i + 1;
  }
}
// one thread per token: String.hashCode over UTF-16 code units and the content hash (FNV-1a 64 of the bytes, mixed, then truncated)
__global__ void tx_token_hash_kernel(const uint8_t* __restrict__ s, const int64_t* __restrict__ tb, const int64_t* __restrict__ te, int64_t n_tok,
                                     uint64_t mask, int32_t* __restrict__ jh, uint64_t* __restrict__ ch) {
  TX_LOOP(t, n_tok) {
    uint32_t h = 0;
    uint64_t f = 0xcbf29ce484222325ull;
    for (int64_t i = tb[t]; i < te[t];) {
      const int l = u8_len(s[i]);
      const uint32_t c = u8_decode(s + i, l);
      if (c >= 0x10000) {
        h = 31u * h + (0xD800u + ((c - 0x10000u) >> 10));
        h = 31u * h + (0xDC00u + ((c - 0x10000u) & 0x3FFu));
      } else {
        h = 31u * h + c;
      }
      for (int k = 0; k < l; ++k) f = (f ^ s[i + k]) * 0x100000001b3ull;
      i += l;
    }
    jh[t] = static_cast<int32_t>(h);
    ch[t] = mix64(f ^ static_cast<uint64_t>(te[t] - tb[t])) & mask;
  }
}
__global__ void tx_iota_kernel(int64_t* __restrict__ p, int64_t n) {
  TX_LOOP(i, n) p[i] = i;
}
template <class T>
__global__ void tx_gather_key_kernel(const T* __restrict__ key, const int64_t* __restrict__ perm, int64_t n, uint64_t* __restrict__ out) {
  TX_LOOP(p, n) out[p] = static_cast<uint64_t>(key[perm[p]]);
}
// vocabulary: position p of the hash-sorted tokens starts a new id unless it equals position p - 1 (same hash and same bytes);
// flag |= 1 where the hashes agree and the bytes do not (a collision that the adjacent compare cannot resolve)
__global__ void tx_vocab_heads_kernel(const uint64_t* __restrict__ sh, const int64_t* __restrict__ si, int64_t n, const uint8_t* __restrict__ s,
                                      const int64_t* __restrict__ tb, const int64_t* __restrict__ te, uint8_t* __restrict__ head, unsigned* flag) {
  TX_LOOP(p, n) {
    bool h = true;
    if (p > 0 && sh[p] == sh[p - 1]) {
      const int64_t a = si[p], b = si[p - 1];
      h = !same_bytes(s, tb[a], te[a], s, tb[b], te[b]);
      if (h && flag) atomicOr(flag, 1u);
    }
    head[p] = h;
  }
}
__global__ void tx_vocab_ids_kernel(const int64_t* __restrict__ si, int64_t n, const int64_t* __restrict__ heads, int32_t* __restrict__ ids) {
  TX_LOOP(p, n) ids[si[p]] = static_cast<int32_t>(heads[p + 1] - 1);
}
// (hash, length, bytes) ordering of the tokens, for the rare batches whose hashes collide
struct TokenLess {
  const uint64_t* ch;
  const uint8_t* s;
  const int64_t *tb, *te;
  __device__ bool operator()(int64_t a, int64_t b) const {
    if (ch[a] != ch[b]) return ch[a] < ch[b];
    const int64_t la = te[a] - tb[a], lb = te[b] - tb[b];
    if (la != lb) return la < lb;
    for (int64_t k = 0; k < la; ++k)
      if (s[tb[a] + k] != s[tb[b] + k]) return s[tb[a] + k] < s[tb[b] + k];
    return false;
  }
};
__global__ void tx_gather_u64_kernel(const uint64_t* __restrict__ v, const int64_t* __restrict__ perm, int64_t n, uint64_t* __restrict__ out) {
  TX_LOOP(p, n) out[p] = v[perm[p]];
}
// emissions: token t of a document with T tokens starts min(T - i - mn + 1, mx - mn + 1)^+ n-grams (i: its position), or one term (mn = 0)
__global__ void tx_emit_count_kernel(const int64_t* __restrict__ toff, int64_t n_docs, int64_t n_tok, int mn, int mx, int64_t* __restrict__ cnt) {
  TX_LOOP(t, n_tok) {
    if (mn == 0) {
      cnt[t] = 1;
      continue;
    }
    const int64_t d = owner_of(toff, n_docs, t);
    const int64_t rem = toff[d + 1] - t - mn + 1;
    const int64_t k = rem < mx - mn + 1 ? rem : mx - mn + 1;
    cnt[t] = k > 0 ? k : 0;
  }
}
// TF emissions: (first token, order, document) of every term
__global__ void tx_emit_terms_kernel(const int64_t* __restrict__ toff, int64_t n_docs, int64_t n_tok, int mn, const int64_t* __restrict__ eoff,
                                     int64_t* __restrict__ efirst, int32_t* __restrict__ eorder, int32_t* __restrict__ edoc) {
  TX_LOOP(t, n_tok) {
    const int64_t d = owner_of(toff, n_docs, t);
    for (int64_t e = eoff[t]; e < eoff[t + 1]; ++e) {
      efirst[e] = t;
      eorder[e] = mn == 0 ? 0 : static_cast<int32_t>(mn + (e - eoff[t]));
      edoc[e] = static_cast<int32_t>(d);
    }
  }
}
// HashingTF emissions: the column and document of every term; a Seq hashes as NGramsHashingTF's rolling MurmurHash3
__global__ void tx_emit_hash_kernel(const int64_t* __restrict__ toff, int64_t n_docs, int64_t n_tok, int mn, const int64_t* __restrict__ eoff,
                                    const int32_t* __restrict__ jh, int32_t nf, int32_t* __restrict__ ecol, int32_t* __restrict__ edoc) {
  TX_LOOP(t, n_tok) {
    const int64_t e0 = eoff[t], e1 = eoff[t + 1];
    if (e0 == e1) continue;
    const int32_t d = static_cast<int32_t>(owner_of(toff, n_docs, t));
    if (mn == 0) {
      ecol[e0] = non_negative_mod(jh[t], nf);
      edoc[e0] = d;
      continue;
    }
    uint32_t h = kSeqSeed;
    for (int j = 0; j < mn; ++j) h = mm_mix(h, static_cast<uint32_t>(jh[t + j]));
    for (int64_t e = e0; e < e1; ++e) {
      const int order = static_cast<int>(mn + (e - e0));
      if (order > mn) h = mm_mix(h, static_cast<uint32_t>(jh[t + order - 1]));
      ecol[e] = non_negative_mod(static_cast<int32_t>(mm_finalize(h, static_cast<uint32_t>(order))), nf);
      edoc[e] = d;
    }
  }
}
// the exact key of term (first, order): order in 3 bits, then the vocabulary ids of its tokens in b bits each, as 128 bits (lo, hi)
__global__ void tx_term_key_kernel(const int64_t* __restrict__ first, const int32_t* __restrict__ order, int64_t n, const int32_t* __restrict__ ids,
                                   int b, uint64_t* __restrict__ lo, uint64_t* __restrict__ hi) {
  TX_LOOP(e, n) {
    const int o = order[e];
    unsigned __int128 k = static_cast<unsigned __int128>(o);
    const int m = o > 0 ? o : 1;
    for (int j = 0; j < m; ++j) k |= static_cast<unsigned __int128>(static_cast<uint32_t>(ids[first[e] + j])) << (3 + j * b);
    lo[e] = static_cast<uint64_t>(k);
    hi[e] = static_cast<uint64_t>(k >> 64);
  }
}
// groups of equal keys in sorted order: head[p] = 1 where position p differs from p - 1 in any of the keys (each may be null)
__global__ void tx_heads_kernel(const int64_t* __restrict__ perm, int64_t n, const uint64_t* __restrict__ k0, const uint64_t* __restrict__ k1,
                                const int32_t* __restrict__ k2, const int32_t* __restrict__ k3, uint8_t* __restrict__ head) {
  TX_LOOP(p, n) {
    bool h = p == 0;
    if (!h) {
      const int64_t a = perm[p], b = perm[p - 1];
      h = (k0 && k0[a] != k0[b]) || (k1 && k1[a] != k1[b]) || (k2 && k2[a] != k2[b]) || (k3 && k3[a] != k3[b]);
    }
    head[p] = h;
  }
}
// gstart[g] = the sorted position where group g starts (heads: inclusive-scanned head flags, shifted by one); gstart[G] = n
__global__ void tx_group_start_kernel(const uint8_t* __restrict__ head, const int64_t* __restrict__ heads, int64_t n, int64_t* __restrict__ gstart) {
  TX_LOOP(p, n) if (head[p]) gstart[heads[p + 1] - 1] = p;
  if (blockIdx.x == 0 && threadIdx.x == 0) gstart[heads[n]] = n;
}
// TF: the first emission of each group is flagged with the group's size
__global__ void tx_tf_mark_kernel(const int64_t* __restrict__ gstart, int64_t G, const int64_t* __restrict__ perm, uint8_t* __restrict__ flag,
                                  int32_t* __restrict__ cnt_at) {
  TX_LOOP(g, G) {
    const int64_t e = perm[gstart[g]];
    flag[e] = 1;
    cnt_at[e] = static_cast<int32_t>(gstart[g + 1] - gstart[g]);
  }
}
__global__ void tx_tf_write_kernel(const uint8_t* __restrict__ flag, const int64_t* __restrict__ pos, int64_t E, const int64_t* __restrict__ efirst,
                                   const int32_t* __restrict__ eorder, const int32_t* __restrict__ cnt_at, int64_t* __restrict__ first,
                                   int32_t* __restrict__ order, int32_t* __restrict__ count, double* __restrict__ value) {
  TX_LOOP(e, E) {
    if (!flag[e]) continue;
    const int64_t q = pos[e];
    first[q] = efirst[e];
    order[q] = eorder[e];
    count[q] = cnt_at[e];
    value[q] = static_cast<double>(cnt_at[e]);
  }
}
__global__ void tx_weights_kernel(const int32_t* __restrict__ count, int64_t n, const double* __restrict__ table, double* __restrict__ value) {
  TX_LOOP(e, n) value[e] = table[count[e] - 1];
}
__global__ void tx_term_doc_kernel(const int64_t* __restrict__ off, int64_t n_docs, int64_t n, int32_t* __restrict__ doc) {
  TX_LOOP(e, n) doc[e] = static_cast<int32_t>(owner_of(off, n_docs, e));
}
// feature selection: per group its document frequency (as maxdf - df, so that ascending is by count descending) and first entry
__global__ void tx_group_stats_kernel(const int64_t* __restrict__ gstart, int64_t G, const int64_t* __restrict__ perm, int64_t maxdf,
                                      uint64_t* __restrict__ neg_df, int64_t* __restrict__ gfirst) {
  TX_LOOP(g, G) {
    neg_df[g] = static_cast<uint64_t>(maxdf - (gstart[g + 1] - gstart[g]));
    gfirst[g] = perm[gstart[g]];
  }
}
// space copy: feature f's tokens; src_tok[new token] = the token it copies
__global__ void tx_feature_tokens_kernel(const int64_t* __restrict__ sel, int64_t K, const int64_t* __restrict__ first, const int32_t* __restrict__ order,
                                         const int64_t* __restrict__ ntoff, int64_t* __restrict__ src_tok, int32_t* __restrict__ forder) {
  TX_LOOP(f, K) {
    const int64_t e = sel[f];
    forder[f] = order[e];
    for (int64_t j = ntoff[f]; j < ntoff[f + 1]; ++j) src_tok[j] = first[e] + (j - ntoff[f]);
  }
}
__global__ void tx_feature_count_kernel(const int64_t* __restrict__ sel, int64_t K, const int32_t* __restrict__ order, int64_t* __restrict__ cnt) {
  TX_LOOP(f, K) cnt[f] = order[sel[f]] > 0 ? order[sel[f]] : 1;
}
__global__ void tx_token_len_kernel(const int64_t* __restrict__ src_tok, int64_t n, const int64_t* __restrict__ tb, const int64_t* __restrict__ te,
                                    int64_t* __restrict__ len) {
  TX_LOOP(j, n) len[j] = te[src_tok[j]] - tb[src_tok[j]];
}
__global__ void tx_copy_tokens_kernel(const int64_t* __restrict__ src_tok, int64_t n, const uint8_t* __restrict__ s, const int64_t* __restrict__ tb,
                                      const int64_t* __restrict__ boff, uint8_t* __restrict__ out, int64_t* __restrict__ ntb, int64_t* __restrict__ nte) {
  TX_LOOP(j, n) {
    const int64_t a = tb[src_tok[j]], l = boff[j + 1] - boff[j];
    for (int64_t k = 0; k < l; ++k) out[boff[j] + k] = s[a + k];
    ntb[j] = boff[j];
    nte[j] = boff[j + 1];
  }
}
__global__ void tx_term_hash_kernel(const int64_t* __restrict__ first, const int32_t* __restrict__ order, int64_t n, const uint64_t* __restrict__ ch,
                                    uint64_t mask, uint64_t* __restrict__ out) {
  TX_LOOP(e, n) out[e] = term_hash(ch, first[e], order[e], mask);
}
// vectorizer: the column of every term found in the space (-1 if none), compared byte by byte among the features of equal hash
struct TermsView {
  const uint8_t* s;
  const int64_t *tb, *te;
  const uint64_t* ch;
  const int64_t* first;
  const int32_t* order;
};
__global__ void tx_lookup_kernel(TermsView q, int64_t n, TermsView sp, const uint64_t* __restrict__ sh, const int64_t* __restrict__ sf, int64_t n_feat,
                                 uint64_t mask, int32_t* __restrict__ col) {
  TX_LOOP(e, n) {
    const int o = q.order[e];
    const uint64_t h = term_hash(q.ch, q.first[e], o, mask);
    int64_t lo = 0, hi = n_feat;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (sh[mid] < h) lo = mid + 1;
      else hi = mid;
    }
    int32_t found = -1;
    for (int64_t p = lo; p < n_feat && sh[p] == h && found < 0; ++p) {
      const int64_t f = sf[p];
      if (sp.order[f] != o) continue;
      bool eq = true;
      for (int j = 0; j < (o > 0 ? o : 1) && eq; ++j) {
        const int64_t a = q.first[e] + j, b = sp.first[f] + j;
        eq = same_bytes(q.s, q.tb[a], q.te[a], sp.s, sp.tb[b], sp.te[b]);
      }
      if (eq) found = static_cast<int32_t>(f);
    }
    col[e] = found;
  }
}
__global__ void tx_found_kernel(const int32_t* __restrict__ col, int64_t n, uint8_t* __restrict__ flag) {
  TX_LOOP(e, n) flag[e] = col[e] >= 0;
}
__global__ void tx_compact_kernel(const uint8_t* __restrict__ flag, const int64_t* __restrict__ pos, int64_t n, const int32_t* __restrict__ col,
                                  const double* __restrict__ val, const int32_t* __restrict__ doc, int32_t* __restrict__ ccol, double* __restrict__ cval,
                                  int32_t* __restrict__ cdoc) {
  TX_LOOP(e, n) {
    if (!flag[e]) continue;
    const int64_t q = pos[e];
    ccol[q] = col[e];
    cval[q] = val[e];
    cdoc[q] = doc[e];
  }
}
// one CSR entry per group of equal (document, column) in sorted order: the values of the group added in entry order
__global__ void tx_csr_groups_kernel(const int64_t* __restrict__ gstart, int64_t G, const int64_t* __restrict__ perm, const int32_t* __restrict__ col,
                                     const double* __restrict__ val, const int32_t* __restrict__ doc, int32_t* __restrict__ idx,
                                     double* __restrict__ out, int32_t* __restrict__ gdoc) {
  TX_LOOP(g, G) {
    const int64_t e = perm[gstart[g]];
    double a = 0.0;
    for (int64_t p = gstart[g]; p < gstart[g + 1]; ++p) a += val[perm[p]];
    idx[g] = col[e];
    gdoc[g] = doc[e];
    out[g] = a;
  }
}
// HashingTF: one CSR entry per group of equal (document, column), its size as the value
__global__ void tx_hash_groups_kernel(const int64_t* __restrict__ gstart, int64_t G, const int64_t* __restrict__ perm, const int32_t* __restrict__ ecol,
                                      const int32_t* __restrict__ edoc, int32_t* __restrict__ idx, double* __restrict__ val, int32_t* __restrict__ gdoc) {
  TX_LOOP(g, G) {
    const int64_t e = perm[gstart[g]];
    idx[g] = ecol[e];
    gdoc[g] = edoc[e];
    val[g] = static_cast<double>(gstart[g + 1] - gstart[g]);
  }
}
// indptr[r] = the first entry whose document is >= r, r in [0, rows]
__global__ void tx_indptr_kernel(const int32_t* __restrict__ doc_sorted, int64_t n, int64_t rows, int64_t* __restrict__ indptr) {
  TX_LOOP(r, rows + 1) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (doc_sorted[mid] < r) lo = mid + 1;
      else hi = mid;
    }
    indptr[r] = lo;
  }
}
struct ToI64 {
  template <class T>
  __host__ __device__ int64_t operator()(T v) const { return static_cast<int64_t>(v); }
};

// ------------------------------------------------------------------------------------ host helpers
// out[0] = 0, out[i + 1] = in[0] + ... + in[i] for i < n, as int64; returns out[n]
template <class T>
int64_t excl_scan(Ctx& c, const T* in, int64_t n, DevBuf& out) {
  cudaStream_t st = c.st;
  out.alloc(sizeof(int64_t) * (n + 1));
  KS_CUDA(cudaMemsetAsync(out.p, 0, sizeof(int64_t), st));
  if (n > 0) {
    auto it = thrust::make_transform_iterator(in, ToI64());
    size_t tb = 0;
    KS_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb, it, out.as<int64_t>() + 1, n, st));
    DevBuf temp;
    temp.alloc(tb);
    KS_CUDA(cub::DeviceScan::InclusiveSum(temp.p, tb, it, out.as<int64_t>() + 1, n, st));
  }
  return read1<int64_t>(out, n, st);
}

// A stable LSD radix sort of positions [0, n): perm ends as the order of the keys, the last pass most significant.  Each pass reads
// key[i] of the original element i (as uint64) and sorts its low `bits` bits; a pass of 0 bits is skipped.
struct SortPass {
  const void* key;
  int type;  // 0: uint64, 1: int32, 2: int64
  int bits;
};
void sort_perm(Ctx& c, DevBuf& perm, int64_t n, const std::vector<SortPass>& passes) {
  cudaStream_t st = c.st;
  perm.alloc(sizeof(int64_t) * n);
  tx_iota_kernel<<<grid_of(n), kT, 0, st>>>(perm.as<int64_t>(), n);
  c.launches += 1;
  if (n <= 1) return;
  DevBuf kin, kout, pout, temp;
  kin.alloc(sizeof(uint64_t) * n);
  kout.alloc(sizeof(uint64_t) * n);
  pout.alloc(sizeof(int64_t) * n);
  for (const SortPass& ps : passes) {
    if (ps.bits <= 0) continue;
    if (ps.type == 0) tx_gather_key_kernel<<<grid_of(n), kT, 0, st>>>(static_cast<const uint64_t*>(ps.key), perm.as<int64_t>(), n, kin.as<uint64_t>());
    else if (ps.type == 1) tx_gather_key_kernel<<<grid_of(n), kT, 0, st>>>(static_cast<const int32_t*>(ps.key), perm.as<int64_t>(), n, kin.as<uint64_t>());
    else tx_gather_key_kernel<<<grid_of(n), kT, 0, st>>>(static_cast<const int64_t*>(ps.key), perm.as<int64_t>(), n, kin.as<uint64_t>());
    size_t tb = 0;
    KS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, kin.as<uint64_t>(), kout.as<uint64_t>(), perm.as<int64_t>(), pout.as<int64_t>(), n, 0,
                                            std::min(ps.bits, 64), st));
    if (temp.bytes < tb) temp.alloc(tb);
    KS_CUDA(cub::DeviceRadixSort::SortPairs(temp.p, tb, kin.as<uint64_t>(), kout.as<uint64_t>(), perm.as<int64_t>(), pout.as<int64_t>(), n, 0,
                                            std::min(ps.bits, 64), st));
    std::swap(perm.p, pout.p);
    std::swap(perm.bytes, pout.bytes);
    c.launches += 2;
  }
}

// groups of equal keys along perm: returns G and gstart[0 .. G] (gstart[G] = n)
int64_t group_starts(Ctx& c, const DevBuf& perm, int64_t n, const uint64_t* k0, const uint64_t* k1, const int32_t* k2, const int32_t* k3,
                     DevBuf& gstart) {
  cudaStream_t st = c.st;
  DevBuf head, heads;
  head.alloc(n);
  tx_heads_kernel<<<grid_of(n), kT, 0, st>>>(perm.as<int64_t>(), n, k0, k1, k2, k3, head.as<uint8_t>());
  const int64_t G = excl_scan(c, head.as<uint8_t>(), n, heads);
  gstart.alloc(sizeof(int64_t) * (G + 1));
  tx_group_start_kernel<<<grid_of(n), kT, 0, st>>>(head.as<uint8_t>(), heads.as<int64_t>(), n, gstart.as<int64_t>());
  c.launches += 2;
  return G;
}

void check_offsets(const int64_t* off, int64_t n, int64_t total, const char* what) {
  if (n < 0) throw KsError{KS_ERR_INVALID, std::string(what) + ": a negative count"};
  if (n > 0 && !off) throw KsError{KS_ERR_INVALID, std::string(what) + ": null offsets"};
  if (n == 0 && total != 0) throw KsError{KS_ERR_INVALID, std::string(what) + ": no documents but a non-empty payload"};
  if (n == 0) return;
  if (off[0] != 0 || off[n] != total) throw KsError{KS_ERR_INVALID, std::string(what) + ": offsets must run from 0 to the total"};
  for (int64_t d = 0; d < n; ++d)
    if (off[d + 1] < off[d]) throw KsError{KS_ERR_INVALID, std::string(what) + ": offsets decrease at " + std::to_string(d)};
}

std::shared_ptr<TextObj> upload_text(Ctx& c, const uint8_t* bytes, int64_t n_bytes, const int64_t* off, int64_t n_docs) {
  if (n_bytes < 0 || (n_bytes > 0 && !bytes)) throw KsError{KS_ERR_INVALID, "bytes: null or a negative size"};
  check_offsets(off, n_docs, n_bytes, "document offsets");
  if (n_docs > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "more than 2^31 - 1 documents"};
  cudaStream_t st = c.st;
  auto t = std::make_shared<TextObj>();
  t->kind = TX_TEXT;
  t->n_bytes = n_bytes;
  t->n_docs = n_docs;
  t->bytes.alloc(n_bytes);
  t->doc_off.alloc(sizeof(int64_t) * (n_docs + 1));
  if (n_bytes) KS_CUDA(cudaMemcpyAsync(t->bytes.p, bytes, n_bytes, cudaMemcpyHostToDevice, st));
  if (n_docs) KS_CUDA(cudaMemcpyAsync(t->doc_off.p, off, sizeof(int64_t) * (n_docs + 1), cudaMemcpyHostToDevice, st));
  else KS_CUDA(cudaMemsetAsync(t->doc_off.p, 0, sizeof(int64_t), st));
  DevBuf start, flag;
  start.alloc(n_bytes + 1);
  flag.alloc(sizeof(unsigned));
  KS_CUDA(cudaMemsetAsync(start.p, 0, n_bytes + 1, st));
  KS_CUDA(cudaMemsetAsync(flag.p, 0, sizeof(unsigned), st));
  tx_doc_start_kernel<<<grid_of(n_docs), kT, 0, st>>>(t->doc_off.as<int64_t>(), n_docs, n_bytes, start.as<uint8_t>());
  tx_validate_kernel<<<grid_of(n_bytes), kT, 0, st>>>(t->bytes.as<uint8_t>(), n_bytes, start.as<uint8_t>(), flag.as<unsigned>());
  c.launches += 2;
  if (read1<unsigned>(flag, 0, st)) throw KsError{KS_ERR_INVALID, "the text is not valid UTF-8 (or a sequence crosses a document boundary)"};
  c.check_async("text upload");
  return t;
}

void hash_tokens(Ctx& c, TextObj& tk) {
  const TextObj& tx = *tk.src;
  tk.jh.alloc(sizeof(int32_t) * tk.n_tok);
  tk.ch.alloc(sizeof(uint64_t) * tk.n_tok);
  tx_token_hash_kernel<<<grid_of(tk.n_tok), kT, 0, c.st>>>(tx.bytes.as<uint8_t>(), tk.tb.as<int64_t>(), tk.te.as<int64_t>(), tk.n_tok,
                                                           hash_mask(c.text_hash_bits), tk.jh.as<int32_t>(), tk.ch.as<uint64_t>());
  c.launches += 1;
}

// vocabulary ids of the tokens (equal bytes, equal id), built once per token batch
void build_vocab(Ctx& c, TextObj& tk) {
  if (tk.vocab >= 0) return;
  cudaStream_t st = c.st;
  const int64_t n = tk.n_tok;
  const uint8_t* s = tk.src->bytes.as<uint8_t>();
  DevBuf perm, sh, head, heads, flag;
  sort_perm(c, perm, n, {{tk.ch.p, 0, c.text_hash_bits}});
  sh.alloc(sizeof(uint64_t) * n);
  head.alloc(n);
  flag.alloc(sizeof(unsigned));
  KS_CUDA(cudaMemsetAsync(flag.p, 0, sizeof(unsigned), st));
  tx_gather_u64_kernel<<<grid_of(n), kT, 0, st>>>(tk.ch.as<uint64_t>(), perm.as<int64_t>(), n, sh.as<uint64_t>());
  tx_vocab_heads_kernel<<<grid_of(n), kT, 0, st>>>(sh.as<uint64_t>(), perm.as<int64_t>(), n, s, tk.tb.as<int64_t>(), tk.te.as<int64_t>(),
                                                   head.as<uint8_t>(), flag.as<unsigned>());
  c.launches += 2;
  if (read1<unsigned>(flag, 0, st)) {
    // different tokens share a hash: order by (hash, length, bytes) so that equal tokens are adjacent, then compare again
    thrust::stable_sort(thrust::cuda::par.on(st), perm.as<int64_t>(), perm.as<int64_t>() + n,
                        TokenLess{tk.ch.as<uint64_t>(), s, tk.tb.as<int64_t>(), tk.te.as<int64_t>()});
    tx_gather_u64_kernel<<<grid_of(n), kT, 0, st>>>(tk.ch.as<uint64_t>(), perm.as<int64_t>(), n, sh.as<uint64_t>());
    tx_vocab_heads_kernel<<<grid_of(n), kT, 0, st>>>(sh.as<uint64_t>(), perm.as<int64_t>(), n, s, tk.tb.as<int64_t>(), tk.te.as<int64_t>(),
                                                     head.as<uint8_t>(), nullptr);
    c.launches += 3;
  }
  const int64_t V = excl_scan(c, head.as<uint8_t>(), n, heads);
  if (V > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "more than 2^31 - 1 distinct tokens"};
  tk.ids.alloc(sizeof(int32_t) * n);
  tx_vocab_ids_kernel<<<grid_of(n), kT, 0, st>>>(perm.as<int64_t>(), n, heads.as<int64_t>(), tk.ids.as<int32_t>());
  c.launches += 1;
  tk.vocab = V;
}

void check_orders(int mn, int mx, int max_allowed) {
  if (mn == 0 && mx == 0) return;
  if (mn < 1 || mx < mn) throw KsError{KS_ERR_INVALID, "orders must be consecutive integers >= 1 (min " + std::to_string(mn) + ", max " + std::to_string(mx) + ")"};
  if (max_allowed > 0 && mx > max_allowed)
    throw KsError{KS_ERR_INVALID, "n-gram orders above " + std::to_string(max_allowed) + " are not supported here (max " + std::to_string(mx) + ")"};
}

// emission offsets of the terms of a token batch: eoff[t] .. eoff[t + 1] are the terms that start at token t; returns their number
int64_t emission_offsets(Ctx& c, const TextObj& tk, int mn, int mx, DevBuf& eoff) {
  DevBuf cnt;
  cnt.alloc(sizeof(int64_t) * tk.n_tok);
  tx_emit_count_kernel<<<grid_of(tk.n_tok), kT, 0, c.st>>>(tk.doc_off.as<int64_t>(), tk.n_docs, tk.n_tok, mn, mx, cnt.as<int64_t>());
  c.launches += 1;
  return excl_scan(c, cnt.as<int64_t>(), tk.n_tok, eoff);
}

// the exact 128-bit keys of terms over the tokens tk; returns the number of key bits used
int term_keys(Ctx& c, TextObj& tk, const int64_t* first, const int32_t* order, int64_t n, int max_order, DevBuf& lo, DevBuf& hi) {
  build_vocab(c, tk);
  const int b = std::max(1, bits_for(static_cast<uint64_t>(std::max<int64_t>(tk.vocab - 1, 0))));
  const int total = 3 + std::max(max_order, 1) * b;
  if (total > 128) throw KsError{KS_ERR_INVALID, "term keys need more than 128 bits"};
  lo.alloc(sizeof(uint64_t) * n);
  hi.alloc(sizeof(uint64_t) * n);
  tx_term_key_kernel<<<grid_of(n), kT, 0, c.st>>>(first, order, n, tk.ids.as<int32_t>(), b, lo.as<uint64_t>(), hi.as<uint64_t>());
  c.launches += 1;
  return total;
}

TextObj& get(Ctx& c, int64_t h, int kind, const char* what) {
  auto it = c.texts.find(h);
  if (it == c.texts.end()) throw KsError{KS_ERR_HANDLE, std::string("unknown text handle ") + std::to_string(h)};
  if (kind >= 0 && it->second->kind != kind) throw KsError{KS_ERR_HANDLE, std::string("handle ") + std::to_string(h) + " is not " + what};
  return *it->second;
}
std::shared_ptr<TextObj> get_ptr(Ctx& c, int64_t h) { return c.texts.at(h); }
int64_t add(Ctx& c, std::shared_ptr<TextObj> o) {
  const int64_t id = c.next_id++;
  c.texts[id] = std::move(o);
  return id;
}

// CSR rows x cols from entries in sorted (document, column) order on the device, then the library's sparse matrix of it
int64_t csr_to_sparse(Ctx& c, int64_t rows, int64_t cols, int64_t nnz, DevBuf& idx, DevBuf& val, const int32_t* doc_sorted) {
  if (cols < 1 || cols > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "a sparse result needs 1 to 2^31 - 1 columns"};
  auto s = std::make_unique<SparseMat>();
  s->rows = rows;
  s->cols = cols;
  s->nnz = nnz;
  s->indptr.alloc(sizeof(int64_t) * (rows + 1));
  tx_indptr_kernel<<<grid_of(rows + 1), kT, 0, c.st>>>(doc_sorted, nnz, rows, s->indptr.as<int64_t>());
  c.launches += 1;
  std::swap(s->indices.p, idx.p);
  std::swap(s->indices.bytes, idx.bytes);
  std::swap(s->values.p, val.p);
  std::swap(s->values.bytes, val.bytes);
  if (!s->indices.p) s->indices.alloc(16);
  if (!s->values.p) s->values.alloc(16);
  auto sm = sparse_from_device_csr(c, std::move(s), nullptr);
  const int64_t id = c.next_id++;
  c.sparses[id] = std::move(sm);
  return id;
}

// ------------------------------------------------------------------------------------ the operations
int64_t text_transform(Ctx& c, int64_t h, int flags) {
  if (flags < 0 || flags > (KS_TEXT_TRIM | KS_TEXT_LOWER)) throw KsError{KS_ERR_INVALID, "unknown transform flags"};
  TextObj& in = get(c, h, TX_TEXT, "a text batch");
  cudaStream_t st = c.st;
  const int64_t n = in.n_bytes;
  DevBuf drop, len, pos;
  if (flags & KS_TEXT_TRIM) {
    drop.alloc(n);
    KS_CUDA(cudaMemsetAsync(drop.p, 0, drop.bytes, st));
    tx_trim_kernel<<<grid_of(in.n_docs), kT, 0, st>>>(in.bytes.as<uint8_t>(), in.doc_off.as<int64_t>(), in.n_docs, drop.as<uint8_t>());
    c.launches += 1;
  }
  len.alloc(n);
  const int lower = (flags & KS_TEXT_LOWER) ? 1 : 0;
  tx_out_len_kernel<<<grid_of(n), kT, 0, st>>>(in.bytes.as<uint8_t>(), n, drop.p ? drop.as<uint8_t>() : nullptr, lower, len.as<uint8_t>());
  c.launches += 1;
  const int64_t total = excl_scan(c, len.as<uint8_t>(), n, pos);
  auto out = std::make_shared<TextObj>();
  out->kind = TX_TEXT;
  out->n_bytes = total;
  out->n_docs = in.n_docs;
  out->bytes.alloc(total);
  out->doc_off.alloc(sizeof(int64_t) * (in.n_docs + 1));
  tx_write_kernel<<<grid_of(n), kT, 0, st>>>(in.bytes.as<uint8_t>(), n, len.as<uint8_t>(), pos.as<int64_t>(), lower, out->bytes.as<uint8_t>());
  tx_gather_offsets_kernel<<<grid_of(in.n_docs + 1), kT, 0, st>>>(in.doc_off.as<int64_t>(), in.n_docs, pos.as<int64_t>(), out->doc_off.as<int64_t>());
  c.launches += 2;
  c.check_async("text transform");
  return add(c, out);
}

int64_t text_tokenize(Ctx& c, int64_t h) {
  TextObj& in = get(c, h, TX_TEXT, "a text batch");
  cudaStream_t st = c.st;
  const int64_t n = in.n_bytes, nd = in.n_docs;
  const uint8_t* s = in.bytes.as<uint8_t>();
  const int64_t* off = in.doc_off.as<int64_t>();
  DevBuf start, rs, runs, cnt;
  start.alloc(n + 1);
  KS_CUDA(cudaMemsetAsync(start.p, 0, n + 1, st));
  tx_doc_start_kernel<<<grid_of(nd), kT, 0, st>>>(off, nd, n, start.as<uint8_t>());
  rs.alloc(n);
  tx_run_start_kernel<<<grid_of(n), kT, 0, st>>>(s, n, start.as<uint8_t>(), rs.as<uint8_t>());
  c.launches += 2;
  excl_scan(c, rs.as<uint8_t>(), n, runs);
  cnt.alloc(sizeof(int64_t) * nd);
  tx_doc_tokens_kernel<<<grid_of(nd), kT, 0, st>>>(s, off, nd, runs.as<int64_t>(), cnt.as<int64_t>());
  c.launches += 1;
  auto tk = std::make_shared<TextObj>();
  tk->kind = TX_TOKENS;
  tk->src = get_ptr(c, h);
  tk->n_docs = nd;
  tk->n_tok = excl_scan(c, cnt.as<int64_t>(), nd, tk->doc_off);
  tk->tb.alloc(sizeof(int64_t) * tk->n_tok);
  tk->te.alloc(sizeof(int64_t) * tk->n_tok);
  tx_empty_tokens_kernel<<<grid_of(nd), kT, 0, st>>>(s, off, nd, runs.as<int64_t>(), tk->doc_off.as<int64_t>(), tk->tb.as<int64_t>(), tk->te.as<int64_t>());
  tx_token_bounds_kernel<<<grid_of(n), kT, 0, st>>>(s, n, start.as<uint8_t>(), off, nd, runs.as<int64_t>(), tk->doc_off.as<int64_t>(),
                                                    tk->tb.as<int64_t>(), tk->te.as<int64_t>());
  c.launches += 2;
  hash_tokens(c, *tk);
  c.check_async("Tokenizer");
  return add(c, tk);
}

int64_t tokens_from_host(Ctx& c, const uint8_t* bytes, int64_t n_bytes, const int64_t* tok_off, int64_t n_tok, const int64_t* doc_off, int64_t n_docs) {
  check_offsets(tok_off, n_tok, n_bytes, "token offsets");
  check_offsets(doc_off, n_docs, n_tok, "document offsets");
  if (n_docs > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "more than 2^31 - 1 documents"};
  // the tokens are uploaded as a text batch with one document per token (so UTF-8 is checked per token)
  auto tx = upload_text(c, bytes, n_bytes, tok_off, n_tok);
  cudaStream_t st = c.st;
  auto tk = std::make_shared<TextObj>();
  tk->kind = TX_TOKENS;
  tk->src = tx;
  tk->n_tok = n_tok;
  tk->n_docs = n_docs;
  tk->tb.alloc(sizeof(int64_t) * n_tok);
  tk->te.alloc(sizeof(int64_t) * n_tok);
  tk->doc_off.alloc(sizeof(int64_t) * (n_docs + 1));
  if (n_tok) {
    KS_CUDA(cudaMemcpyAsync(tk->tb.p, tok_off, sizeof(int64_t) * n_tok, cudaMemcpyHostToDevice, st));
    KS_CUDA(cudaMemcpyAsync(tk->te.p, tok_off + 1, sizeof(int64_t) * n_tok, cudaMemcpyHostToDevice, st));
  }
  if (n_docs) KS_CUDA(cudaMemcpyAsync(tk->doc_off.p, doc_off, sizeof(int64_t) * (n_docs + 1), cudaMemcpyHostToDevice, st));
  else KS_CUDA(cudaMemsetAsync(tk->doc_off.p, 0, sizeof(int64_t), st));
  hash_tokens(c, *tk);
  c.check_async("token upload");
  return add(c, tk);
}

int64_t term_frequency(Ctx& c, int64_t h, int mn, int mx, int64_t* max_count) {
  check_orders(mn, mx, 4);
  TextObj& tk = get(c, h, TX_TOKENS, "a token batch");
  cudaStream_t st = c.st;
  DevBuf eoff;
  const int64_t E = emission_offsets(c, tk, mn, mx, eoff);
  DevBuf efirst, eorder, edoc;
  efirst.alloc(sizeof(int64_t) * E);
  eorder.alloc(sizeof(int32_t) * E);
  edoc.alloc(sizeof(int32_t) * E);
  tx_emit_terms_kernel<<<grid_of(tk.n_tok), kT, 0, st>>>(tk.doc_off.as<int64_t>(), tk.n_docs, tk.n_tok, mn, eoff.as<int64_t>(), efirst.as<int64_t>(),
                                                         eorder.as<int32_t>(), edoc.as<int32_t>());
  c.launches += 1;
  DevBuf lo, hi, perm, gstart;
  const int bits = term_keys(c, tk, efirst.as<int64_t>(), eorder.as<int32_t>(), E, mx, lo, hi);
  sort_perm(c, perm, E, {{lo.p, 0, std::min(bits, 64)}, {hi.p, 0, bits - 64}, {edoc.p, 1, bits_for(static_cast<uint64_t>(tk.n_docs))}});
  const int64_t G = group_starts(c, perm, E, lo.as<uint64_t>(), hi.as<uint64_t>(), edoc.as<int32_t>(), nullptr, gstart);
  DevBuf flag, cnt_at, pos;
  flag.alloc(E);
  cnt_at.alloc(sizeof(int32_t) * E);
  KS_CUDA(cudaMemsetAsync(flag.p, 0, flag.bytes, st));
  tx_tf_mark_kernel<<<grid_of(G), kT, 0, st>>>(gstart.as<int64_t>(), G, perm.as<int64_t>(), flag.as<uint8_t>(), cnt_at.as<int32_t>());
  c.launches += 1;
  excl_scan(c, flag.as<uint8_t>(), E, pos);
  auto tf = std::make_shared<TextObj>();
  tf->kind = TX_TF;
  tf->src = get_ptr(c, h);
  tf->n_terms = G;
  tf->n_docs = tk.n_docs;
  tf->first.alloc(sizeof(int64_t) * G);
  tf->order.alloc(sizeof(int32_t) * G);
  tf->count.alloc(sizeof(int32_t) * G);
  tf->value.alloc(sizeof(double) * G);
  tf->doc_off.alloc(sizeof(int64_t) * (tk.n_docs + 1));
  tx_tf_write_kernel<<<grid_of(E), kT, 0, st>>>(flag.as<uint8_t>(), pos.as<int64_t>(), E, efirst.as<int64_t>(), eorder.as<int32_t>(), cnt_at.as<int32_t>(),
                                                tf->first.as<int64_t>(), tf->order.as<int32_t>(), tf->count.as<int32_t>(), tf->value.as<double>());
  // the terms of document d start at the flagged emissions before its first emission
  DevBuf edoc_off;
  edoc_off.alloc(sizeof(int64_t) * (tk.n_docs + 1));
  tx_gather_offsets_kernel<<<grid_of(tk.n_docs + 1), kT, 0, st>>>(tk.doc_off.as<int64_t>(), tk.n_docs, eoff.as<int64_t>(), edoc_off.as<int64_t>());
  tx_gather_offsets_kernel<<<grid_of(tk.n_docs + 1), kT, 0, st>>>(edoc_off.as<int64_t>(), tk.n_docs, pos.as<int64_t>(), tf->doc_off.as<int64_t>());
  c.launches += 3;
  int64_t mc = 0;
  if (G > 0) {
    DevBuf mx_out, temp;
    mx_out.alloc(sizeof(int32_t));
    size_t tb = 0;
    KS_CUDA(cub::DeviceReduce::Max(nullptr, tb, tf->count.as<int32_t>(), mx_out.as<int32_t>(), G, st));
    temp.alloc(tb);
    KS_CUDA(cub::DeviceReduce::Max(temp.p, tb, tf->count.as<int32_t>(), mx_out.as<int32_t>(), G, st));
    mc = read1<int32_t>(mx_out, 0, st);
  }
  tf->max_count = mc;
  if (max_count) *max_count = mc;
  c.check_async("TermFrequency");
  return add(c, tf);
}

void check_terms(const TextObj& tk, const int64_t* first, const int32_t* order, int64_t n) {
  if (n > 0 && (!first || !order)) throw KsError{KS_ERR_INVALID, "null term arrays"};
  for (int64_t e = 0; e < n; ++e) {
    if (order[e] < 0 || order[e] > 4) throw KsError{KS_ERR_INVALID, "term orders must lie in [0, 4]"};
    if (first[e] < 0 || first[e] + std::max(order[e], 1) > tk.n_tok) throw KsError{KS_ERR_INVALID, "a term's tokens lie outside the token batch"};
  }
}

int64_t tf_from_host(Ctx& c, int64_t h, const int64_t* first, const int32_t* order, const double* values, int64_t n, const int64_t* doc_off,
                     int64_t n_docs) {
  TextObj& tk = get(c, h, TX_TOKENS, "a token batch");
  check_terms(tk, first, order, n);
  check_offsets(doc_off, n_docs, n, "document offsets");
  if (n_docs > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "more than 2^31 - 1 documents"};
  for (int64_t e = 0; e < n; ++e)
    if (!std::isfinite(values[e])) throw KsError{KS_ERR_INVALID, "a term-frequency value is not finite"};
  cudaStream_t st = c.st;
  auto tf = std::make_shared<TextObj>();
  tf->kind = TX_TF;
  tf->src = get_ptr(c, h);
  tf->n_terms = n;
  tf->n_docs = n_docs;
  tf->first.alloc(sizeof(int64_t) * n);
  tf->order.alloc(sizeof(int32_t) * n);
  tf->value.alloc(sizeof(double) * n);
  tf->doc_off.alloc(sizeof(int64_t) * (n_docs + 1));
  if (n) {
    KS_CUDA(cudaMemcpyAsync(tf->first.p, first, sizeof(int64_t) * n, cudaMemcpyHostToDevice, st));
    KS_CUDA(cudaMemcpyAsync(tf->order.p, order, sizeof(int32_t) * n, cudaMemcpyHostToDevice, st));
    KS_CUDA(cudaMemcpyAsync(tf->value.p, values, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  }
  if (n_docs) KS_CUDA(cudaMemcpyAsync(tf->doc_off.p, doc_off, sizeof(int64_t) * (n_docs + 1), cudaMemcpyHostToDevice, st));
  else KS_CUDA(cudaMemsetAsync(tf->doc_off.p, 0, sizeof(int64_t), st));
  c.check_async("term-frequency upload");
  return add(c, tf);
}

void tf_set_weights(Ctx& c, int64_t h, const double* table, int64_t n) {
  TextObj& tf = get(c, h, TX_TF, "a term-frequency batch");
  if (!tf.count.p) throw KsError{KS_ERR_INVALID, "this term-frequency batch carries no counts (it was uploaded with its values)"};
  if (n < tf.max_count || (n > 0 && !table)) throw KsError{KS_ERR_INVALID, "the weight table must cover every count up to the largest"};
  for (int64_t i = 0; i < n; ++i)
    if (!std::isfinite(table[i])) throw KsError{KS_ERR_INVALID, "the weight of count " + std::to_string(i + 1) + " is not finite"};
  if (tf.n_terms == 0) return;
  DevBuf t;
  t.alloc(sizeof(double) * n);
  KS_CUDA(cudaMemcpyAsync(t.p, table, sizeof(double) * n, cudaMemcpyHostToDevice, c.st));
  tx_weights_kernel<<<grid_of(tf.n_terms), kT, 0, c.st>>>(tf.count.as<int32_t>(), tf.n_terms, t.as<double>(), tf.value.as<double>());
  c.launches += 1;
  c.check_async("TermFrequency weights");
}

// a feature space: the features' own token batch, their (first, order) and their content hashes in ascending order
void finish_space(Ctx& c, TextObj& sp) {
  const TextObj& tk = *sp.src;
  const int64_t K = sp.n_terms;
  DevBuf gh, perm;
  gh.alloc(sizeof(uint64_t) * K);
  tx_term_hash_kernel<<<grid_of(K), kT, 0, c.st>>>(sp.first.as<int64_t>(), sp.order.as<int32_t>(), K, tk.ch.as<uint64_t>(), hash_mask(c.text_hash_bits),
                                                  gh.as<uint64_t>());
  c.launches += 1;
  sort_perm(c, perm, K, {{gh.p, 0, c.text_hash_bits}});
  sp.sh.alloc(sizeof(uint64_t) * K);
  tx_gather_u64_kernel<<<grid_of(K), kT, 0, c.st>>>(gh.as<uint64_t>(), perm.as<int64_t>(), K, sp.sh.as<uint64_t>());
  c.launches += 1;
  std::swap(sp.sf.p, perm.p);
  std::swap(sp.sf.bytes, perm.bytes);
}

int64_t features_fit(Ctx& c, int64_t h, int64_t num_features) {
  if (c.world > 1)
    throw KsError{KS_ERR_INVALID, "CommonSparseFeatures / AllSparseFeatures fit on one rank only (an exact top-K over ranks is not implemented)"};
  if (num_features < -1 || num_features == 0) throw KsError{KS_ERR_INVALID, "num_features must be >= 1 (or -1: all features)"};
  TextObj& tf = get(c, h, TX_TF, "a term-frequency batch");
  TextObj& tk = *tf.src;
  cudaStream_t st = c.st;
  const int64_t n = tf.n_terms;
  int max_order = 0;
  if (n > 0) {
    DevBuf mo, temp;
    mo.alloc(sizeof(int32_t));
    size_t tb = 0;
    KS_CUDA(cub::DeviceReduce::Max(nullptr, tb, tf.order.as<int32_t>(), mo.as<int32_t>(), n, st));
    temp.alloc(tb);
    KS_CUDA(cub::DeviceReduce::Max(temp.p, tb, tf.order.as<int32_t>(), mo.as<int32_t>(), n, st));
    max_order = read1<int32_t>(mo, 0, st);
  }
  DevBuf lo, hi, perm, gstart;
  const int bits = term_keys(c, tk, tf.first.as<int64_t>(), tf.order.as<int32_t>(), n, max_order, lo, hi);
  sort_perm(c, perm, n, {{lo.p, 0, std::min(bits, 64)}, {hi.p, 0, bits - 64}});
  const int64_t G = group_starts(c, perm, n, lo.as<uint64_t>(), hi.as<uint64_t>(), nullptr, nullptr, gstart);
  DevBuf neg_df, gfirst, order2;
  neg_df.alloc(sizeof(uint64_t) * G);
  gfirst.alloc(sizeof(int64_t) * G);
  tx_group_stats_kernel<<<grid_of(G), kT, 0, st>>>(gstart.as<int64_t>(), G, perm.as<int64_t>(), n, neg_df.as<uint64_t>(), gfirst.as<int64_t>());
  c.launches += 1;
  // by first entry, then (stably) by count descending
  sort_perm(c, order2, G, {{gfirst.p, 2, bits_for(static_cast<uint64_t>(n))}, {neg_df.p, 0, bits_for(static_cast<uint64_t>(n))}});
  const int64_t K = num_features < 0 ? G : std::min(G, num_features);
  if (K == 0) throw KsError{KS_ERR_INVALID, "the batch holds no terms: a feature space needs at least one feature"};
  if (K > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "more than 2^31 - 1 features"};
  DevBuf sel;
  sel.alloc(sizeof(int64_t) * K);
  tx_gather_key_kernel<<<grid_of(K), kT, 0, st>>>(gfirst.as<int64_t>(), order2.as<int64_t>(), K, sel.as<uint64_t>());
  // copy the selected terms' tokens into the space's own token batch
  DevBuf fcnt, ntoff;
  fcnt.alloc(sizeof(int64_t) * K);
  tx_feature_count_kernel<<<grid_of(K), kT, 0, st>>>(sel.as<int64_t>(), K, tf.order.as<int32_t>(), fcnt.as<int64_t>());
  c.launches += 2;
  const int64_t NT = excl_scan(c, fcnt.as<int64_t>(), K, ntoff);
  auto sp = std::make_shared<TextObj>();
  sp->kind = TX_SPACE;
  sp->n_terms = K;
  sp->first.alloc(sizeof(int64_t) * K);
  sp->order.alloc(sizeof(int32_t) * K);
  DevBuf src_tok, tlen, boff;
  src_tok.alloc(sizeof(int64_t) * NT);
  tx_feature_tokens_kernel<<<grid_of(K), kT, 0, st>>>(sel.as<int64_t>(), K, tf.first.as<int64_t>(), tf.order.as<int32_t>(), ntoff.as<int64_t>(),
                                                      src_tok.as<int64_t>(), sp->order.as<int32_t>());
  KS_CUDA(cudaMemcpyAsync(sp->first.p, ntoff.p, sizeof(int64_t) * K, cudaMemcpyDeviceToDevice, st));
  tlen.alloc(sizeof(int64_t) * NT);
  tx_token_len_kernel<<<grid_of(NT), kT, 0, st>>>(src_tok.as<int64_t>(), NT, tk.tb.as<int64_t>(), tk.te.as<int64_t>(), tlen.as<int64_t>());
  c.launches += 2;
  const int64_t NB = excl_scan(c, tlen.as<int64_t>(), NT, boff);
  auto ntx = std::make_shared<TextObj>();
  ntx->kind = TX_TEXT;
  ntx->n_bytes = NB;
  ntx->bytes.alloc(NB);
  ntx->doc_off.alloc(sizeof(int64_t));
  KS_CUDA(cudaMemsetAsync(ntx->doc_off.p, 0, sizeof(int64_t), st));
  auto ntk = std::make_shared<TextObj>();
  ntk->kind = TX_TOKENS;
  ntk->src = ntx;
  ntk->n_tok = NT;
  ntk->tb.alloc(sizeof(int64_t) * NT);
  ntk->te.alloc(sizeof(int64_t) * NT);
  ntk->doc_off.alloc(sizeof(int64_t));
  KS_CUDA(cudaMemsetAsync(ntk->doc_off.p, 0, sizeof(int64_t), st));
  tx_copy_tokens_kernel<<<grid_of(NT), kT, 0, st>>>(src_tok.as<int64_t>(), NT, tk.src->bytes.as<uint8_t>(), tk.tb.as<int64_t>(), boff.as<int64_t>(),
                                                    ntx->bytes.as<uint8_t>(), ntk->tb.as<int64_t>(), ntk->te.as<int64_t>());
  c.launches += 1;
  hash_tokens(c, *ntk);
  sp->src = ntk;
  finish_space(c, *sp);
  c.check_async("CommonSparseFeatures.fit");
  return add(c, sp);
}

int64_t features_from_host(Ctx& c, int64_t h, const int64_t* first, const int32_t* order, int64_t n) {
  TextObj& tk = get(c, h, TX_TOKENS, "a token batch");
  check_terms(tk, first, order, n);
  if (n < 1 || n > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "a feature space needs 1 to 2^31 - 1 features"};
  auto sp = std::make_shared<TextObj>();
  sp->kind = TX_SPACE;
  sp->src = get_ptr(c, h);
  sp->n_terms = n;
  sp->first.alloc(sizeof(int64_t) * n);
  sp->order.alloc(sizeof(int32_t) * n);
  if (n) {
    KS_CUDA(cudaMemcpyAsync(sp->first.p, first, sizeof(int64_t) * n, cudaMemcpyHostToDevice, c.st));
    KS_CUDA(cudaMemcpyAsync(sp->order.p, order, sizeof(int32_t) * n, cudaMemcpyHostToDevice, c.st));
  }
  finish_space(c, *sp);
  c.check_async("feature space upload");
  return add(c, sp);
}

int64_t features_apply(Ctx& c, int64_t hs, int64_t htf) {
  TextObj& sp = get(c, hs, TX_SPACE, "a feature space");
  TextObj& tf = get(c, htf, TX_TF, "a term-frequency batch");
  const TextObj& qt = *tf.src;
  const TextObj& st_tok = *sp.src;
  cudaStream_t st = c.st;
  const int64_t n = tf.n_terms;
  DevBuf col, doc, flag, pos;
  col.alloc(sizeof(int32_t) * n);
  doc.alloc(sizeof(int32_t) * n);
  flag.alloc(n);
  TermsView q{qt.src->bytes.as<uint8_t>(), qt.tb.as<int64_t>(), qt.te.as<int64_t>(), qt.ch.as<uint64_t>(), tf.first.as<int64_t>(), tf.order.as<int32_t>()};
  TermsView s{st_tok.src->bytes.as<uint8_t>(), st_tok.tb.as<int64_t>(), st_tok.te.as<int64_t>(), st_tok.ch.as<uint64_t>(), sp.first.as<int64_t>(),
              sp.order.as<int32_t>()};
  tx_lookup_kernel<<<grid_of(n), kT, 0, st>>>(q, n, s, sp.sh.as<uint64_t>(), sp.sf.as<int64_t>(), sp.n_terms, hash_mask(c.text_hash_bits), col.as<int32_t>());
  tx_term_doc_kernel<<<grid_of(n), kT, 0, st>>>(tf.doc_off.as<int64_t>(), tf.n_docs, n, doc.as<int32_t>());
  tx_found_kernel<<<grid_of(n), kT, 0, st>>>(col.as<int32_t>(), n, flag.as<uint8_t>());
  c.launches += 3;
  const int64_t nnz = excl_scan(c, flag.as<uint8_t>(), n, pos);
  DevBuf ccol, cval, cdoc, perm, idx, val, sdoc;
  ccol.alloc(sizeof(int32_t) * nnz);
  cval.alloc(sizeof(double) * nnz);
  cdoc.alloc(sizeof(int32_t) * nnz);
  tx_compact_kernel<<<grid_of(n), kT, 0, st>>>(flag.as<uint8_t>(), pos.as<int64_t>(), n, col.as<int32_t>(), tf.value.as<double>(), doc.as<int32_t>(),
                                               ccol.as<int32_t>(), cval.as<double>(), cdoc.as<int32_t>());
  c.launches += 1;
  sort_perm(c, perm, nnz, {{ccol.p, 1, bits_for(static_cast<uint64_t>(sp.n_terms))}, {cdoc.p, 1, bits_for(static_cast<uint64_t>(tf.n_docs))}});
  // a term repeated within a document of an uploaded batch gives one entry, the sum of its values (the device TF never repeats one)
  DevBuf gstart;
  const int64_t G = group_starts(c, perm, nnz, nullptr, nullptr, ccol.as<int32_t>(), cdoc.as<int32_t>(), gstart);
  idx.alloc(sizeof(int32_t) * G);
  val.alloc(sizeof(double) * G);
  sdoc.alloc(sizeof(int32_t) * G);
  tx_csr_groups_kernel<<<grid_of(G), kT, 0, st>>>(gstart.as<int64_t>(), G, perm.as<int64_t>(), ccol.as<int32_t>(), cval.as<double>(), cdoc.as<int32_t>(),
                                                  idx.as<int32_t>(), val.as<double>(), sdoc.as<int32_t>());
  c.launches += 1;
  const int64_t id = csr_to_sparse(c, tf.n_docs, sp.n_terms, G, idx, val, sdoc.as<int32_t>());
  c.check_async("SparseFeatureVectorizer.apply");
  return id;
}

int64_t hashing_tf(Ctx& c, int64_t h, int mn, int mx, int64_t nf) {
  check_orders(mn, mx, 0);
  if (nf < 1 || nf > std::numeric_limits<int32_t>::max()) throw KsError{KS_ERR_INVALID, "num_features must lie in [1, 2^31 - 1]"};
  TextObj& tk = get(c, h, TX_TOKENS, "a token batch");
  cudaStream_t st = c.st;
  DevBuf eoff;
  const int64_t E = emission_offsets(c, tk, mn, mx, eoff);
  DevBuf ecol, edoc, perm, gstart;
  ecol.alloc(sizeof(int32_t) * E);
  edoc.alloc(sizeof(int32_t) * E);
  tx_emit_hash_kernel<<<grid_of(tk.n_tok), kT, 0, st>>>(tk.doc_off.as<int64_t>(), tk.n_docs, tk.n_tok, mn, eoff.as<int64_t>(), tk.jh.as<int32_t>(),
                                                        static_cast<int32_t>(nf), ecol.as<int32_t>(), edoc.as<int32_t>());
  c.launches += 1;
  sort_perm(c, perm, E, {{ecol.p, 1, bits_for(static_cast<uint64_t>(nf - 1))}, {edoc.p, 1, bits_for(static_cast<uint64_t>(tk.n_docs))}});
  DevBuf idx, val, gdoc;
  const int64_t G = group_starts(c, perm, E, nullptr, nullptr, ecol.as<int32_t>(), edoc.as<int32_t>(), gstart);
  idx.alloc(sizeof(int32_t) * G);
  val.alloc(sizeof(double) * G);
  gdoc.alloc(sizeof(int32_t) * G);
  tx_hash_groups_kernel<<<grid_of(G), kT, 0, st>>>(gstart.as<int64_t>(), G, perm.as<int64_t>(), ecol.as<int32_t>(), edoc.as<int32_t>(), idx.as<int32_t>(),
                                                   val.as<double>(), gdoc.as<int32_t>());
  c.launches += 1;
  const int64_t id = csr_to_sparse(c, tk.n_docs, nf, G, idx, val, gdoc.as<int32_t>());
  c.check_async("HashingTF");
  return id;
}

}  // namespace
}  // namespace ks

// ------------------------------------------------------------------------------------ C ABI
using namespace ks;

extern "C" {

KS_API int32_t ks_text_from_host(int64_t ctx, const uint8_t* bytes, int64_t n_bytes, const int64_t* doc_offsets, int64_t n_docs, int64_t* out_text) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_text) throw KsError{KS_ERR_INVALID, "null out_text"};
    *out_text = add(c, upload_text(c, bytes, n_bytes, doc_offsets, n_docs));
  });
}
KS_API int32_t ks_text_transform(int64_t ctx, int64_t text, int32_t flags, int64_t* out_text) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_text) throw KsError{KS_ERR_INVALID, "null out_text"};
    *out_text = text_transform(c, text, flags);
  });
}
KS_API int32_t ks_text_tokenize(int64_t ctx, int64_t text, int64_t* out_tokens) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_tokens) throw KsError{KS_ERR_INVALID, "null out_tokens"};
    *out_tokens = text_tokenize(c, text);
  });
}
KS_API int32_t ks_tokens_from_host(int64_t ctx, const uint8_t* bytes, int64_t n_bytes, const int64_t* token_offsets, int64_t n_tokens,
                                   const int64_t* doc_offsets, int64_t n_docs, int64_t* out_tokens) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_tokens) throw KsError{KS_ERR_INVALID, "null out_tokens"};
    *out_tokens = tokens_from_host(c, bytes, n_bytes, token_offsets, n_tokens, doc_offsets, n_docs);
  });
}
KS_API int32_t ks_term_frequency(int64_t ctx, int64_t tokens, int32_t min_order, int32_t max_order, int64_t* out_tf, int64_t* out_max_count) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_tf) throw KsError{KS_ERR_INVALID, "null out_tf"};
    *out_tf = term_frequency(c, tokens, min_order, max_order, out_max_count);
  });
}
KS_API int32_t ks_tf_set_weights(int64_t ctx, int64_t tf, const double* table, int64_t n) {
  return guarded(ctx, [&](Ctx& c) { tf_set_weights(c, tf, table, n); });
}
KS_API int32_t ks_tf_from_host(int64_t ctx, int64_t tokens, const int64_t* term_first, const int32_t* term_order, const double* values,
                               int64_t n_terms, const int64_t* doc_offsets, int64_t n_docs, int64_t* out_tf) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_tf) throw KsError{KS_ERR_INVALID, "null out_tf"};
    if (n_terms > 0 && !values) throw KsError{KS_ERR_INVALID, "null values"};
    *out_tf = tf_from_host(c, tokens, term_first, term_order, values, n_terms, doc_offsets, n_docs);
  });
}
KS_API int32_t ks_sparse_features_fit(int64_t ctx, int64_t tf, int64_t num_features, int64_t* out_space) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_space) throw KsError{KS_ERR_INVALID, "null out_space"};
    *out_space = features_fit(c, tf, num_features);
  });
}
KS_API int32_t ks_sparse_features_from_host(int64_t ctx, int64_t tokens, const int64_t* term_first, const int32_t* term_order, int64_t n_features,
                                            int64_t* out_space) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_space) throw KsError{KS_ERR_INVALID, "null out_space"};
    *out_space = features_from_host(c, tokens, term_first, term_order, n_features);
  });
}
KS_API int32_t ks_sparse_features_apply(int64_t ctx, int64_t space, int64_t tf, int64_t* out_sparse) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_sparse) throw KsError{KS_ERR_INVALID, "null out_sparse"};
    *out_sparse = features_apply(c, space, tf);
  });
}
KS_API int32_t ks_hashing_tf(int64_t ctx, int64_t tokens, int32_t min_order, int32_t max_order, int64_t num_features, int64_t* out_sparse) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_sparse) throw KsError{KS_ERR_INVALID, "null out_sparse"};
    *out_sparse = hashing_tf(c, tokens, min_order, max_order, num_features);
  });
}

// (device buffer, element size, element count) of array `which` of a text object
static void text_array(Ctx& c, int64_t h, int which, const DevBuf** buf, size_t* elem, int64_t* n) {
  TextObj& o = get(c, h, -1, "");
  const TextObj* tok = o.kind == TX_TOKENS ? &o : (o.kind == TX_TF || o.kind == TX_SPACE) ? o.src.get() : nullptr;
  const bool terms = o.kind == TX_TF || o.kind == TX_SPACE;
  *buf = nullptr;
  switch (which) {
    case KS_TEXT_BYTES: {
      const TextObj* t = o.kind == TX_TEXT ? &o : tok->src.get();
      *buf = &t->bytes, *elem = 1, *n = t->n_bytes;
      break;
    }
    case KS_TEXT_DOC_OFFSETS:
      if (o.kind != TX_SPACE) *buf = &o.doc_off, *elem = 8, *n = o.n_docs + 1;
      break;
    case KS_TEXT_TOKEN_BEGIN: if (tok) *buf = &tok->tb, *elem = 8, *n = tok->n_tok; break;
    case KS_TEXT_TOKEN_END: if (tok) *buf = &tok->te, *elem = 8, *n = tok->n_tok; break;
    case KS_TEXT_TOKEN_JAVA_HASH: if (tok) *buf = &tok->jh, *elem = 4, *n = tok->n_tok; break;
    case KS_TEXT_TERM_FIRST: if (terms) *buf = &o.first, *elem = 8, *n = o.n_terms; break;
    case KS_TEXT_TERM_ORDER: if (terms) *buf = &o.order, *elem = 4, *n = o.n_terms; break;
    case KS_TEXT_TERM_COUNT: if (o.kind == TX_TF && o.count.p) *buf = &o.count, *elem = 4, *n = o.n_terms; break;
    case KS_TEXT_TERM_VALUE: if (o.kind == TX_TF) *buf = &o.value, *elem = 8, *n = o.n_terms; break;
    default: break;
  }
  if (!*buf) throw KsError{KS_ERR_INVALID, "this text object has no array " + std::to_string(which)};
}
KS_API int32_t ks_text_array_size(int64_t ctx, int64_t obj, int32_t which, int64_t* out_n) {
  return guarded(ctx, [&](Ctx& c) {
    if (!out_n) throw KsError{KS_ERR_INVALID, "null out_n"};
    const DevBuf* b;
    size_t e;
    text_array(c, obj, which, &b, &e, out_n);
  });
}
KS_API int32_t ks_text_array(int64_t ctx, int64_t obj, int32_t which, void* out, int64_t n) {
  return guarded(ctx, [&](Ctx& c) {
    const DevBuf* b;
    size_t e;
    int64_t have;
    text_array(c, obj, which, &b, &e, &have);
    if (n < 0 || n > have) throw KsError{KS_ERR_INVALID, "asked for more elements than the array holds"};
    if (n > 0 && !out) throw KsError{KS_ERR_INVALID, "null out"};
    if (n > 0) KS_CUDA(cudaMemcpyAsync(out, b->p, e * n, cudaMemcpyDeviceToHost, c.st));
    KS_CUDA(cudaStreamSynchronize(c.st));
  });
}
KS_API int32_t ks_text_destroy(int64_t ctx, int64_t obj) {
  return guarded(ctx, [&](Ctx& c) {
    if (!c.texts.erase(obj)) throw KsError{KS_ERR_HANDLE, "unknown text handle"};
  });
}

}  // extern "C"
