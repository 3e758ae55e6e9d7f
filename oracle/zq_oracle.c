/* oracle/zq_oracle.c -- TEST INFRASTRUCTURE ONLY.  Never linked, imported or executed by the
 * product path (zpaqfranz_b200/); only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline
 * leg may use it, and only as the checker.
 *
 * A plain-C, single-threaded restatement of the reference's block-compression hot path
 * (zpaqfranz.cpp of fcorbelli/zpaqfranz, "Z:" below), written from the reference's behaviour, not copied:
 *
 *   zqo_sha1              libzpaq::SHA1                       Z:12637-12819
 *   zqo_suffix_array      divsufsort's *result* (the SA is unique)  Z:19121
 *   zqo_lz_stream         LZBuffer ctor/fill/write_*          Z:19333-19612   (LZ77 hash + SA, BWT)
 *   zqo_e8e9              e8e9                                Z:19162
 *   zqo_block_unmodeled   Compressor framing + unmodeled Encoder  Z:15554,15590-15600,15970-16187
 *   zqo_fragment          dedup fragmenter                    Z:95604-95633, Z:121626-121631
 *
 * Pinned (tests/test_oracle_pinned.py) against oracle/_ref (the reference compiled here) and the
 * reference's own known-answer vectors (Z:77129-77160), so parity is NOT "unpinned".
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint8_t u8;
typedef uint32_t u32;
typedef uint64_t u64;

/* ------------------------------------------------------------------ SHA-1 (FIPS 180-4) */
static u32 rol(u32 x, int k) { return (x << k) | (x >> (32 - k)); }

static void sha1_block(u32 st[5], const u8* p) {
  u32 w[80];
  for (int t = 0; t < 16; ++t) w[t] = (u32)p[4 * t] << 24 | (u32)p[4 * t + 1] << 16 | (u32)p[4 * t + 2] << 8 | p[4 * t + 3];
  for (int t = 16; t < 80; ++t) w[t] = rol(w[t - 3] ^ w[t - 8] ^ w[t - 14] ^ w[t - 16], 1);
  u32 a = st[0], b = st[1], c = st[2], d = st[3], e = st[4];
  for (int t = 0; t < 80; ++t) {
    u32 f, k;
    if (t < 20) f = (b & c) | (~b & d), k = 0x5A827999u;
    else if (t < 40) f = b ^ c ^ d, k = 0x6ED9EBA1u;
    else if (t < 60) f = (b & c) | (b & d) | (c & d), k = 0x8F1BBCDCu;
    else f = b ^ c ^ d, k = 0xCA62C1D6u;
    u32 tmp = rol(a, 5) + f + e + k + w[t];
    e = d; d = c; c = rol(b, 30); b = a; a = tmp;
  }
  st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e;
}

void zqo_sha1(const u8* in, u64 n, u8 out[20]) {
  u32 st[5] = {0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u};
  u64 i = 0;
  for (; i + 64 <= n; i += 64) sha1_block(st, in + i);
  u8 tail[128];
  u64 r = n - i;
  memset(tail, 0, sizeof tail);
  if (r) memcpy(tail, in + i, r);
  tail[r] = 0x80;
  u64 tl = r < 56 ? 64 : 128, bits = n * 8;
  for (int k = 0; k < 8; ++k) tail[tl - 1 - k] = (u8)(bits >> (8 * k));
  for (u64 k = 0; k < tl; k += 64) sha1_block(st, tail + k);
  for (int k = 0; k < 5; ++k) { out[4 * k] = st[k] >> 24; out[4 * k + 1] = st[k] >> 16; out[4 * k + 2] = st[k] >> 8; out[4 * k + 3] = st[k]; }
}

/* ------------------------------------------------------------------ suffix array
 * Prefix doubling with qsort; O(n log^2 n). Order = unsigned bytes, shorter suffix first. */
static const u32* g_rank; static u32 g_h, g_n;
static int cmp_pair(const void* a, const void* b) {
  u32 x = *(const u32*)a, y = *(const u32*)b;
  if (g_rank[x] != g_rank[y]) return g_rank[x] < g_rank[y] ? -1 : 1;
  long long rx = x + g_h < g_n ? (long long)g_rank[x + g_h] : -1, ry = y + g_h < g_n ? (long long)g_rank[y + g_h] : -1;
  return rx < ry ? -1 : rx > ry;
}
int zqo_suffix_array(const u8* t, u32* sa, u32 n) {
  if (!n) return 0;
  u32* rank = (u32*)malloc(4 * (size_t)n), *tmp = (u32*)malloc(4 * (size_t)n);
  if (!rank || !tmp) return -1;
  for (u32 i = 0; i < n; ++i) sa[i] = i, rank[i] = t[i];
  for (u32 h = 1;; h *= 2) {
    g_rank = rank; g_h = h; g_n = n;
    qsort(sa, n, 4, cmp_pair);
    tmp[sa[0]] = 0;
    for (u32 i = 1; i < n; ++i) tmp[sa[i]] = tmp[sa[i - 1]] + (cmp_pair(&sa[i - 1], &sa[i]) < 0);
    memcpy(rank, tmp, 4 * (size_t)n);
    if (rank[sa[n - 1]] == n - 1 || h >= n) break;
  }
  free(rank); free(tmp);
  return 0;
}

/* ------------------------------------------------------------------ E8E9 (Z:19162) */
void zqo_e8e9(u8* buf, int n) {
  for (int i = n - 5; i >= 0; --i)
    if ((buf[i] & 254) == 0xe8 && ((buf[i + 4] + 1) & 254) == 0) {
      u32 a = (buf[i + 1] | buf[i + 2] << 8 | buf[i + 3] << 16) + i;
      buf[i + 1] = a; buf[i + 2] = a >> 8; buf[i + 3] = a >> 16;
    }
}

/* ------------------------------------------------------------------ LZ77 / BWT pre-pass */
static int lg(u32 x) { int r = 0; while (x) ++r, x >>= 1; return r; }

typedef struct {
  u8* out; u64 cap, len; int overflow;
  u32 bits, nbits;
} Sink;
static void put(Sink* s, int c) { if (s->len < s->cap) s->out[s->len++] = (u8)c; else s->overflow = 1; }
static void putb(Sink* s, u32 x, int k) {
  x &= (1u << k) - 1;  /* k < 32 always here */
  s->bits |= x << s->nbits; s->nbits += k;
  while (s->nbits > 7) put(s, s->bits & 255), s->bits >>= 8, s->nbits -= 8;
}
static void flushb(Sink* s) { if (s->nbits > 0) put(s, s->bits); s->bits = s->nbits = 0; }

typedef struct { int level; u32 minMatch, rb; const u8* in; } Coder;

static void write_literal(Sink* s, const Coder* c, u32 i, u32* lit) {
  if (c->level == 1) {
    if (*lit < 1) return;
    int ll = lg(*lit);
    putb(s, 0, 2);
    --ll;
    while (--ll >= 0) { putb(s, 1, 1); putb(s, (*lit >> ll) & 1, 1); }
    putb(s, 0, 1);
    while (*lit) { putb(s, c->in[i - *lit], 8); --*lit; }
  } else {
    while (*lit > 0) {
      u32 l1 = *lit > 64 ? 64 : *lit;
      put(s, l1 - 1);
      for (u32 j = i - *lit; j < i - *lit + l1; ++j) put(s, c->in[j]);
      *lit -= l1;
    }
  }
}
static void write_match(Sink* s, const Coder* c, u32 len, u32 off) {
  if (c->level == 1) {
    int ll = lg(len) - 1;
    off += (1u << c->rb) - 1;
    int lo = lg(off) - 1 - c->rb;
    putb(s, (lo + 8) >> 3, 2);
    putb(s, lo & 7, 3);
    while (--ll >= 2) { putb(s, 1, 1); putb(s, (len >> ll) & 1, 1); }
    putb(s, 0, 1);
    putb(s, len & 3, 2);
    putb(s, off, c->rb);
    putb(s, off >> c->rb, lo);
  } else {
    const u32 mm = c->minMatch;
    --off;
    while (len > 0) {
      const u32 l1 = len > mm * 2 + 63 ? mm + 63 : len > mm + 63 ? len - mm : len;
      if (off < (1u << 16)) { put(s, 64 + l1 - mm); put(s, off >> 8); put(s, off); }
      else if (off < (1u << 24)) { put(s, 128 + l1 - mm); put(s, off >> 16); put(s, off >> 8); put(s, off); }
      else { put(s, 192 + l1 - mm); put(s, off >> 24); put(s, off >> 16); put(s, off >> 8); put(s, off); }
      len -= l1;
    }
  }
}

/* Whole LZBuffer output for args[0..8] (the e8e9 step is the caller's: apply zqo_e8e9 first when
 * args[1]>4).  `sa_in` may be NULL (computed here).  Returns stream length, -1 alloc, -2 overflow.
 * If tok_out != NULL, every parse decision is recorded as (i, len, off) triples (len==0: literal step)
 * -- used by the GPU tests to localise a divergence. */
long long zqo_lz_stream(const u8* in, u32 n, const int* args, const u32* sa_in, u8* out, u64 cap,
                        u32* tok_out, u64 tok_cap, u64* ntok) {
  const int level = args[1] & 3;
  const int use_sa = (args[5] - args[0] >= 21) || level == 3;
  Sink s; memset(&s, 0, sizeof s); s.out = out; s.cap = cap;
  u64 nt = 0;
  u32* sa = 0; u32* isa = 0; u32* ht = 0;
  long long ret = -1;
  if (use_sa) {
    sa = (u32*)malloc(4 * (size_t)(n + 1));
    if (!sa) goto done;
    if (sa_in) memcpy(sa, sa_in, 4 * (size_t)n); else if (zqo_suffix_array(in, sa, n)) goto done;
  }
  if (level == 3) { /* BWT: last column with the EOS row coded as 255, then its index LSB first */
    u32 idx = 0;
    for (u32 i = 0; i < n + 5; ++i) {
      if (i == 0) put(&s, n > 0 ? in[n - 1] : 255);
      else if (i > n) put(&s, idx & 255), idx >>= 8;
      else if (sa[i - 1] == 0) idx = i, put(&s, 255);
      else put(&s, in[sa[i - 1] - 1]);
    }
    ret = s.overflow ? -2 : (long long)s.len;
    goto done;
  }
  {
    const int checkbits = use_sa ? 17 + args[0] : 12 - args[0];
    const u32 mask = (1u << checkbits) - 1;
    const u32 minMatch = args[2], minMatch2 = args[3], maxMatch = 3u << 14, maxLiteral = 1u << 12;
    const u32 lookahead = args[6], bucket = (1u << args[4]) - 1;
    const u32 htsize = use_sa ? 0 : 1u << args[5];
    const u32 shift1 = minMatch > 0 ? (args[5] - 1) / minMatch + 1 : 1;
    const u32 shift2 = minMatch2 > 0 ? (args[5] - 1) / minMatch2 + 1 : 0;
    const u32 mmb0 = minMatch > minMatch2 + lookahead ? minMatch : minMatch2 + lookahead;
    const int minMatchBoth = (int)mmb0 + 4;
    Coder cd; cd.level = level; cd.minMatch = minMatch; cd.rb = args[0] > 4 ? args[0] - 4 : 0; cd.in = in;
    if ((minMatch < 4 && level == 1) || (minMatch < 1 && level == 2)) { ret = -3; goto done; }
    if (use_sa) { isa = (u32*)calloc((size_t)mask + 1, 4); if (!isa) goto done; }
    else { ht = (u32*)calloc(htsize, 4); if (!ht) goto done; }
    u32 i = 0, lit = 0, h1 = 0, h2 = 0;
    while (i < n) {
      u32 blen = minMatch - 1, bp = 0, blit = 0; int bscore = 0;
      if (use_sa) {
        if (sa[isa[i & mask]] != i)
          for (u32 j = 0; j < n; ++j) if ((sa[j] & ~mask) == (i & ~mask)) isa[sa[j] & mask] = j;
        for (u32 h = 0; h <= lookahead; ++h) {
          u32 q = isa[(h + i) & mask];
          if (sa[q] != h + i) continue;
          for (int j = -1; j <= 1; j += 2) {
            for (u32 k = 1; k <= bucket; ++k) {
              u32 p, x = q + (u32)j * k;
              if (x < n && (p = sa[x] - h) < i) {
                u32 l, l1;
                for (l = h; i + l < n && l < maxMatch && in[p + l] == in[i + l]; ++l) {}
                for (l1 = h; l1 > 0 && in[p + l1 - 1] == in[i + l1 - 1]; --l1) {}
                int score = (int)(l - l1) * 8 - lg(i - p) - 4 * (lit == 0 && l1 > 0) - 11;
                for (u32 a = 0; a < h; ++a) score = score * 5 / 8;
                if (score > bscore) blen = l, bp = p, blit = l1, bscore = score;
                if (l < blen || l < minMatch || l > 255) break;
              }
            }
          }
          if (bscore <= 0 || blen < minMatch) break;
        }
      } else if (level == 1 || minMatch <= 64) {
        if (minMatch2 > 0) {
          for (u32 k = 0; k <= bucket; ++k) {
            u32 p = ht[h2 ^ k];
            if (p && (p & mask) == (in[i + 3] & mask)) {
              p >>= checkbits;
              if (p < i && i + blen <= n && in[p + blen - 1] == in[i + blen - 1]) {
                u32 l;
                for (l = lookahead; i + l < n && l < maxMatch && in[p + l] == in[i + l]; ++l) {}
                if (l >= minMatch2 + lookahead) {
                  int l1;
                  for (l1 = lookahead; l1 > 0 && in[p + l1 - 1] == in[i + l1 - 1]; --l1) {}
                  int score = (int)(l - l1) * 8 - lg(i - p) - 8 * (lit == 0 && l1 > 0) - 11;
                  if (score > bscore) blen = l, bp = p, blit = l1, bscore = score;
                }
              }
            }
            if (blen >= 128) break;
          }
        }
        if (!minMatch2 || blen < minMatch2) {
          for (u32 k = 0; k <= bucket; ++k) {
            u32 p = ht[h1 ^ k];
            if (p && i + 3 < n && (p & mask) == (in[i + 3] & mask)) {
              p >>= checkbits;
              if (p < i && i + blen <= n && in[p + blen - 1] == in[i + blen - 1]) {
                u32 l;
                for (l = 0; i + l < n && l < maxMatch && in[p + l] == in[i + l]; ++l) {}
                int score = (int)l * 8 - lg(i - p) - 2 * (lit > 0) - 11;
                if (score > bscore) blen = l, bp = p, blit = 0, bscore = score;
              }
            }
            if (blen >= 128) break;
          }
        }
      }
      const u32 off = i - bp;
      if (off > 0 && bscore > 0 &&
          blen - blit >= minMatch + (level == 2) * ((off >= (1u << 16)) + (off >= (1u << 24)))) {
        lit += blit;
        write_literal(&s, &cd, i + blit, &lit);
        write_match(&s, &cd, blen - blit, off);
        if (tok_out && nt + 3 <= tok_cap) { tok_out[nt] = i; tok_out[nt + 1] = blen - blit; tok_out[nt + 2] = off; }
        nt += 3;
      } else {
        blen = 1; ++lit;
        if (tok_out && nt + 3 <= tok_cap) { tok_out[nt] = i; tok_out[nt + 1] = 0; tok_out[nt + 2] = 0; }
        nt += 3;
      }
      if (use_sa) i += blen;
      else {
        while (blen--) {
          if ((long long)i + minMatchBoth < (long long)n) {
            u32 ih = ((i * 1234547u) >> 19) & bucket;
            const u32 p = (i << checkbits) | (in[i + 3] & mask);
            if (minMatch2) {
              ht[h2 ^ ih] = p;
              h2 = (((h2 * 9) << shift2) + (in[i + minMatch2 + lookahead] + 1) * 23456789u) & (htsize - 1);
            }
            ht[h1 ^ ih] = p;
            h1 = (((h1 * 5) << shift1) + (in[i + minMatch] + 1) * 123456791u) & (htsize - 1);
          }
          ++i;
        }
      }
      if (lit >= maxLiteral) write_literal(&s, &cd, i, &lit);
    }
    write_literal(&s, &cd, n, &lit);
    flushb(&s);
    ret = s.overflow ? -2 : (long long)s.len;
  }
done:
  if (ntok) *ntok = nt / 3;
  free(sa); free(isa); free(ht);
  return ret;
}

/* ------------------------------------------------------------------ block framing, unmodeled
 * tag | "zPQ" lvl 1 | header | 01 filename 00 comment 00 00 | chunks | 00 00 00 00 | FD sha1 / FE | FF
 * where the chunk stream carries  [00] or [01 len_lo len_hi pcomp...]  followed by `stream`,
 * cut into <= 65536-byte pieces each prefixed by its big-endian 32-bit length.
 * header/pcomp bytes come from the host assembler (validated separately against the reference). */
long long zqo_block_unmodeled(const u8* header, u32 hlen, const u8* pcomp, u32 plen,
                              const char* filename, const char* comment_full,
                              const u8* stream, u64 slen, const u8* sha1 /* or NULL */,
                              u8* out, u64 cap) {
  static const u8 tag[13] = {0x37, 0x6b, 0x53, 0x74, 0xa0, 0x31, 0x83, 0xd3, 0x8c, 0xb2, 0x28, 0xb0, 0xd3};
  Sink s; memset(&s, 0, sizeof s); s.out = out; s.cap = cap;
  for (int i = 0; i < 13; ++i) put(&s, tag[i]);
  put(&s, 'z'); put(&s, 'P'); put(&s, 'Q'); put(&s, 1 + (header[6] == 0)); put(&s, 1);
  for (u32 i = 0; i < hlen; ++i) put(&s, header[i]);
  put(&s, 1);
  for (const char* p = filename; p && *p; ++p) put(&s, (u8)*p);
  put(&s, 0);
  for (const char* p = comment_full; p && *p; ++p) put(&s, (u8)*p);
  put(&s, 0); put(&s, 0);
  /* virtual payload = selector bytes + stream */
  u8 sel[3]; u32 nsel;
  if (plen) sel[0] = 1, sel[1] = plen & 255, sel[2] = plen >> 8, nsel = 3; else sel[0] = 0, nsel = 1;
  const u64 total = nsel + plen + slen;
  for (u64 o = 0; o < total; o += 65536) {
    u64 c = total - o < 65536 ? total - o : 65536;
    put(&s, (c >> 24) & 255); put(&s, (c >> 16) & 255); put(&s, (c >> 8) & 255); put(&s, c & 255);
    for (u64 k = o; k < o + c; ++k)
      put(&s, k < nsel ? sel[k] : k < nsel + plen ? pcomp[k - nsel] : stream[k - nsel - plen]);
  }
  put(&s, 0); put(&s, 0); put(&s, 0); put(&s, 0);
  if (sha1) { put(&s, 253); for (int i = 0; i < 20; ++i) put(&s, sha1[i]); } else put(&s, 254);
  put(&s, 255);
  return s.overflow ? -2 : (long long)s.len;
}

/* ------------------------------------------------------------------ dedup fragmenter */
long long zqo_fragment(const u8* in, u64 n, int fragment, u32 blocksize, u32* frag_len,
                       u32* frag_hits, u64 cap) {
  u32 maxf = fragment <= 19 ? (8128u << fragment) : blocksize - 12;
  if (maxf > blocksize - 12) maxf = blocksize - 12;
  u32 minf = fragment <= 25 ? (64u << fragment) : maxf;
  if (minf > maxf) minf = maxf;
  u64 pos = 0, k = 0;
  while (pos < n) {
    u8 o1[256]; memset(o1, 0, 256);
    u32 h = 0, hits = 0, sz = 0; int c1 = 0;
    while (pos < n) {
      int c = in[pos++];
      if (c == o1[c1]) h = (h + c + 1) * 314159265u, ++hits; else h = (h + c + 1) * 271828182u;
      o1[c1] = (u8)c; c1 = c; ++sz;
      if (sz >= maxf || (fragment <= 22 && h < (1u << (22 - fragment)) && sz >= minf)) break;
    }
    if (k >= cap) return -2;
    frag_len[k] = sz; frag_hits[k] = hits; ++k;
  }
  return (long long)k;
}
