// oracle/ref_shim.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// Wraps the UNMODIFIED reference translation unit (zpaqfranz.cpp, found through -I<its directory>: ZPAQFRANZ_SRC
// names it -- no reference source is copied into this repository) behind a small C ABI so
// that tests and the bench's CPU-baseline leg can call the reference's own libzpaq::compressBlock,
// libzpaq::decompress, SHA1/SHA256, XXH3-128, BLAKE3, divsufsort, makeConfig/Compiler and LZBuffer.
// Built by __graft_entry__.build() / oracle/Makefile into oracle/_ref/libzpaqref.so (git-ignored).
#define main zpaqfranz_reference_main
#include "zpaqfranz.cpp"
#undef main
#include <pthread.h>
#include <atomic>

namespace {
struct VecWriter : public libzpaq::Writer {
  std::vector<unsigned char> v;
  void put(int c) { v.push_back((unsigned char)c); }
  void write(const char* buf, int n) { v.insert(v.end(), (const unsigned char*)buf, (const unsigned char*)buf + n); }
};
struct MemReader : public libzpaq::Reader {
  const unsigned char* p; size_t n, i;
  MemReader(const unsigned char* p_, size_t n_) : p(p_), n(n_), i(0) {}
  int get() { return i < n ? p[i++] : -1; }
  int read(char* buf, int len) {
    size_t r = n - i; if (r > (size_t)len) r = len;
    memcpy(buf, p + i, r); i += r; return (int)r;
  }
};
thread_local std::string g_lasterr;
// built with -DHWSHA2 like the reference's own Makefile on x86: use the SHA extensions where the host has them, as the
// command line does (Z:68513)
struct HwInit { HwInit() { flaghw = ihavehw(); } } g_hwinit;
}  // namespace

extern "C" {

const char* zref_last_error() { return g_lasterr.c_str(); }
void zref_set_nojit(int v) { flagnojit = v != 0; }

// == libzpaq::compressBlock (Z:20255). Returns bytes written, -1 on error, -2 if out too small.
long long zref_compress_block(const unsigned char* in, unsigned n, const char* method,
                              const char* filename, const char* comment, int dosha1,
                              unsigned char* out, unsigned long long cap) {
  try {
    libzpaq::StringBuffer sb;
    if (n) sb.write((const char*)in, n);
    VecWriter w;
    libzpaq::compressBlock(&sb, &w, method, filename, comment, dosha1 != 0);
    if (w.v.size() > cap) return -2;
    memcpy(out, w.v.data(), w.v.size());
    return (long long)w.v.size();
  } catch (std::exception& e) { g_lasterr = e.what(); return -1; }
}

// == libzpaq::Compressor driven directly (Z:15970-16187): one block, one segment, caller's model.
// level > 0: startBlock(level) (built-in models); else header = stored block header bytes.
// pcomp/plen: postProcess(pcomp, plen) when plen > 0, else postProcess() default.
long long zref_compress_segment(int level, const unsigned char* header, const unsigned char* pcomp, int plen,
                                const unsigned char* in, unsigned n, const char* filename, const char* comment,
                                const unsigned char* sha1, int tag, unsigned char* out, unsigned long long cap) {
  try {
    MemReader r(in, n);
    VecWriter w;
    libzpaq::Compressor co;
    co.setOutput(&w);
    co.setInput(&r);
    if (tag) co.writeTag();
    if (level > 0) co.startBlock(level); else co.startBlock((const char*)header);
    co.startSegment(filename, comment);
    if (plen > 0) co.postProcess((const char*)pcomp, plen); else co.postProcess();
    co.compress();
    co.endSegment((const char*)sha1);
    co.endBlock();
    if (w.v.size() > cap) return -2;
    memcpy(out, w.v.data(), w.v.size());
    return (long long)w.v.size();
  } catch (std::exception& e) { g_lasterr = e.what(); return -1; }
}

// One block holding nseg segments (what the streaming archiver writes; Compressor Z:15970-16187): segment k is
// in[off[k] .. off[k]+len[k]), named "<filename><k>", with the SHA-1 of its data stored when sha != 0.
long long zref_compress_multi(int level, const unsigned char* header, const unsigned char* pcomp, int plen, int nseg,
                              const unsigned char* in, const unsigned long long* off, const unsigned* len,
                              const char* filename, const char* comment, int sha, unsigned char* out, unsigned long long cap) {
  try {
    VecWriter w;
    libzpaq::Compressor co;
    co.setOutput(&w);
    co.writeTag();
    if (level > 0) co.startBlock(level); else co.startBlock((const char*)header);
    for (int k = 0; k < nseg; ++k) {
      MemReader r(in + off[k], len[k]);
      co.setInput(&r);
      const std::string name = std::string(filename ? filename : "") + std::to_string(k);
      co.startSegment(name.c_str(), comment);
      if (k == 0) { if (plen > 0) co.postProcess((const char*)pcomp, plen); else co.postProcess(); }
      co.compress();
      if (sha) {
        libzpaq::SHA1 s1; s1.write((const char*)in + off[k], (int64_t)len[k]);
        co.endSegment(s1.result());
      } else co.endSegment(0);
    }
    co.endBlock();
    if (w.v.size() > cap) return -2;
    memcpy(out, w.v.data(), w.v.size());
    return (long long)w.v.size();
  } catch (std::exception& e) { g_lasterr = e.what(); return -1; }
}

// The reference's own command line (its main(), Z:78458), for archive-level comparisons: run it in a child
// process -- it calls exit().
int zref_main(int argc, const char** argv) { return zpaqfranz_reference_main(argc, argv); }

// == libzpaq::decompress (Z:15536) over a whole stream of blocks.
long long zref_decompress(const unsigned char* in, unsigned long long n, unsigned char* out,
                          unsigned long long cap) {
  try {
    MemReader r(in, n);
    VecWriter w;
    libzpaq::decompress(&r, &w);
    if (w.v.size() > cap) return -2;
    memcpy(out, w.v.data(), w.v.size());
    return (long long)w.v.size();
  } catch (std::exception& e) { g_lasterr = e.what(); return -1; }
}

void zref_sha1(const unsigned char* in, unsigned long long n, unsigned char* out20) {
  libzpaq::SHA1 s; s.write((const char*)in, (int64_t)n); memcpy(out20, s.result(), 20);
}
void zref_sha256(const unsigned char* in, unsigned long long n, unsigned char* out32) {
  libzpaq::SHA256 s; s.write((const char*)in, (int64_t)n); memcpy(out32, s.result(), 32);
}
// XXH64, seed 0 (the archiver's default file hash), little-endian u64
void zref_xxh64(const unsigned char* in, unsigned long long n, unsigned char* out8) {
  XXHash64 x(0);            // the archiver's own wrapper (Z:27039) around XXH64_reset/update/digest
  x.add(in, n);
  const unsigned long long h = x.hash();
  for (int k = 0; k < 8; ++k) out8[k] = (unsigned char)(h >> (8 * k));
}
// CRC-32 as Jidac::updatehash computes it (crc32_16bytes, Z:30299), little-endian u32
void zref_crc32(const unsigned char* in, unsigned long long n, unsigned char* out4) {
  const unsigned int c = crc32_16bytes(in, n, 0);
  for (int k = 0; k < 4; ++k) out4[k] = (unsigned char)(c >> (8 * k));
}
// XXH3-128, seed 0; out = high64 then low64, big-endian hex order as the reference prints it
void zref_xxh3_128(const unsigned char* in, unsigned long long n, unsigned char* out16) {
  XXH3_state_t st; (void)XXH3_128bits_reset(&st);
  (void)XXH3_128bits_update(&st, in, n);
  XXH128_hash_t h = XXH3_128bits_digest(&st);
  for (int i = 0; i < 8; ++i) out16[i] = (unsigned char)(h.high64 >> (56 - 8 * i));
  for (int i = 0; i < 8; ++i) out16[8 + i] = (unsigned char)(h.low64 >> (56 - 8 * i));
}
// MD5 / SHA3-256 as Jidac::updatehash feeds them (MD5::add Z:21616, SHA3::add Z:21337); digests as raw bytes
void zref_md5(const unsigned char* in, unsigned long long n, unsigned char* out16) {
  MD5 h; h.add(in, n); h.getHash(out16);
}
void zref_sha3_256(const unsigned char* in, unsigned long long n, unsigned char* out32) {
  SHA3 h; h.add(in, n); const std::string x = h.getHash();
  for (int k = 0; k < 32; ++k) out32[k] = (unsigned char)strtoul(x.substr(2 * k, 2).c_str(), 0, 16);
}
void zref_blake3(const unsigned char* in, unsigned long long n, unsigned char* out32) {
  blake3_hasher h; blake3_hasher_init(&h); blake3_hasher_update(&h, in, n);
  blake3_hasher_finalize(&h, out32, 32);
}
int zref_divsufsort(const unsigned char* t, int* sa, int n) { return libzpaq::divsufsort(t, sa, n); }

// makeConfig (Z:19615): method "x..." -> config text + args[9]
int zref_make_config(const char* method, int* args9, char* out, int cap) {
  try {
    std::string s = libzpaq::makeConfig(method, args9);
    if ((int)s.size() + 1 > cap) return -2;
    memcpy(out, s.c_str(), s.size() + 1);
    return (int)s.size();
  } catch (std::exception& e) { g_lasterr = e.what(); return -1; }
}
// Compiler (Z:15904): config text -> COMP+HCOMP header bytes (as written to the block) and PCOMP bytes
int zref_compile(const char* config, int* args9, unsigned char* hdr, int* hlen,
                 unsigned char* pc, int* plen) {
  try {
    libzpaq::ZPAQL hz, pz;
    libzpaq::StringBuffer cmd;
    libzpaq::Compiler(config, args9, hz, pz, &cmd);
    VecWriter w; hz.write(&w, false);
    memcpy(hdr, w.v.data(), w.v.size()); *hlen = (int)w.v.size();
    int n = pz.hend - pz.hbegin; if (n < 0) n = 0;
    if (n) memcpy(pc, &pz.header[pz.hbegin], n);
    *plen = n;
    return 0;
  } catch (std::exception& e) { g_lasterr = e.what(); return -1; }
}
// The expanded method string compressBlock would use is not observable directly; tests derive it
// from the emitted header instead. LZBuffer (Z:19183) output stream for given args:
long long zref_lz_stream(const unsigned char* in, unsigned n, int* args9, unsigned char* out,
                         unsigned long long cap) {
  try {
    libzpaq::StringBuffer sb;
    if (n) sb.write((const char*)in, n);
    libzpaq::LZBuffer lz(sb, args9);
    unsigned long long k = 0; int c;
    while ((c = lz.get()) >= 0) { if (k >= cap) return -2; out[k++] = (unsigned char)c; }
    return (long long)k;
  } catch (std::exception& e) { g_lasterr = e.what(); return -1; }
}

// Dedup fragmenter exactly as in Jidac::add (Z:122457-122561; canonical form Z:95604-95633) with
// the constants of Z:121626-121631. Emits fragment lengths and per-fragment `hits`.
// (This loop has no callable symbol in the reference; it is restated here and cross-checked in
// tests against archives produced by the reference CLI.)
long long zref_fragment(const unsigned char* in, unsigned long long n, int fragment,
                        unsigned* frag_len, unsigned* frag_hits, unsigned long long cap) {
  const unsigned blocksize = (1u << 26) - 4096;  // default -m1..: "6" => 64 MiB blocks (Z:121605-121625)
  unsigned MAXF = fragment <= 19 ? (8128u << fragment) : blocksize - 12;
  if (MAXF > blocksize - 12) MAXF = blocksize - 12;
  unsigned MINF = fragment <= 25 ? (64u << fragment) : MAXF;
  if (MINF > MAXF) MINF = MAXF;
  unsigned long long pos = 0, k = 0;
  while (pos < n) {
    unsigned char o1[256] = {0};
    int c1 = 0; unsigned h = 0, hits = 0; unsigned sz = 0;
    while (pos < n) {
      int c = in[pos++];
      if (c == o1[c1]) h = (h + c + 1) * 314159265u, ++hits;
      else h = (h + c + 1) * 271828182u;
      o1[c1] = c; c1 = c; ++sz;
      if (sz >= MAXF || (fragment <= 22 && h < (1u << (22 - fragment)) && sz >= MINF)) break;
    }
    if (k >= cap) return -2;
    frag_len[k] = sz; frag_hits[k] = hits; ++k;
  }
  return (long long)k;
}

// Multi-threaded CPU baseline: T pthreads each looping compressBlock over a slice of equally
// sized units laid out back to back. Returns total compressed bytes (checks nothing else).
struct MtArg { const unsigned char* base; unsigned unit; int lo, hi; const char* method; long long out; };
static void* mt_worker(void* p) {
  MtArg* a = (MtArg*)p; a->out = 0;
  for (int u = a->lo; u < a->hi; ++u) {
    libzpaq::StringBuffer sb; sb.write((const char*)a->base + (size_t)u * a->unit, a->unit);
    VecWriter w;
    try { libzpaq::compressBlock(&sb, &w, a->method, "", "", true); } catch (...) { a->out = -1; return 0; }
    a->out += (long long)w.v.size();
  }
  return 0;
}
long long zref_compress_units_mt(const unsigned char* base, unsigned unit, int nunits,
                                 const char* method, int threads) {
  if (threads < 1) threads = 1;
  std::vector<pthread_t> th(threads); std::vector<MtArg> args(threads);
  for (int t = 0; t < threads; ++t) {
    args[t].base = base; args[t].unit = unit; args[t].method = method;
    args[t].lo = (int)((long long)nunits * t / threads);
    args[t].hi = (int)((long long)nunits * (t + 1) / threads);
    pthread_create(&th[t], 0, mt_worker, &args[t]);
  }
  long long tot = 0;
  for (int t = 0; t < threads; ++t) { pthread_join(th[t], 0); if (args[t].out < 0) tot = -1; else if (tot >= 0) tot += args[t].out; }
  return tot;
}


// Same pool over an arbitrary list of buffers (offset, length), handed out dynamically; optionally the SHA-256 and the
// length of every compressed block (bench.py's whole-batch parity check) and, with `roundtrip`, each block is also
// decompressed again by the reference's own decoder and compared with its input (configs[2]).
struct ListJob {
  const unsigned char* base; const unsigned long long* off; const unsigned* len; int n; const char* method;
  unsigned char* digests; unsigned* outlen; int roundtrip; std::atomic<int> next; std::atomic<long long> total; std::atomic<int> bad;
};
static void* list_worker(void* p) {
  ListJob* j = (ListJob*)p;
  for (;;) {
    const int u = j->next.fetch_add(1);
    if (u >= j->n) break;
    libzpaq::StringBuffer sb; sb.write((const char*)j->base + j->off[u], j->len[u]);
    VecWriter w;
    try { libzpaq::compressBlock(&sb, &w, j->method, "", "", true); } catch (...) { j->bad.fetch_add(1); continue; }
    j->total.fetch_add((long long)w.v.size());
    if (j->outlen) j->outlen[u] = (unsigned)w.v.size();
    if (j->digests) {
      libzpaq::SHA256 h; for (size_t k = 0; k < w.v.size(); ++k) h.put(w.v[k]);
      memcpy(j->digests + (size_t)u * 32, h.result(), 32);
    }
    if (j->roundtrip) {
      MemReader r(w.v.data(), w.v.size()); VecWriter back;
      try { libzpaq::decompress(&r, &back); } catch (...) { j->bad.fetch_add(1); continue; }
      if (back.v.size() != j->len[u] || memcmp(back.v.data(), j->base + j->off[u], j->len[u]) != 0) j->bad.fetch_add(1);
    }
  }
  return 0;
}
long long zref_compress_list_mt(const unsigned char* base, const unsigned long long* off, const unsigned* len, int n,
                                const char* method, int threads, unsigned char* digests, unsigned* outlen, int roundtrip) {
  if (threads < 1) threads = 1;
  ListJob j; j.base = base; j.off = off; j.len = len; j.n = n; j.method = method; j.digests = digests; j.outlen = outlen;
  j.roundtrip = roundtrip; j.next = 0; j.total = 0; j.bad = 0;
  std::vector<pthread_t> th(threads);
  for (int t = 0; t < threads; ++t) pthread_create(&th[t], 0, list_worker, &j);
  for (int t = 0; t < threads; ++t) pthread_join(th[t], 0);
  return j.bad.load() ? -1 : j.total.load();
}


// The chunker path on `threads` host threads, files handed out dynamically: fragment boundaries (zref_fragment's loop),
// libzpaq::SHA1 of every fragment, BLAKE3 of every file -- what Jidac::add + updatehash do per file (Z:122457-122573,
// Z:85948).  Returns the number of fragments (bench.py's CPU baseline of configs[3]).
struct FragJob { const unsigned char* base; const unsigned long long* off; const unsigned long long* len; int n, fragment; std::atomic<int> next; std::atomic<long long> frags; };
static void* frag_worker(void* p) {
  FragJob* j = (FragJob*)p;
  std::vector<unsigned> fl, fh;
  for (;;) {
    const int f = j->next.fetch_add(1);
    if (f >= j->n) break;
    const unsigned char* d = j->base + j->off[f]; const unsigned long long n = j->len[f];
    const unsigned long long cap = n / 4096 + 16;
    fl.resize(cap); fh.resize(cap);
    const long long k = zref_fragment(d, n, j->fragment, fl.data(), fh.data(), cap);
    unsigned long long o = 0; unsigned char dg[32];
    for (long long q = 0; q < k; ++q) { zref_sha1(d + o, fl[q], dg); o += fl[q]; }
    zref_blake3(d, n, dg);
    j->frags.fetch_add(k > 0 ? k : 0);
  }
  return 0;
}
long long zref_fragment_hash_mt(const unsigned char* base, const unsigned long long* off, const unsigned long long* len, int nfiles,
                                int fragment, int threads) {
  if (threads < 1) threads = 1;
  FragJob j; j.base = base; j.off = off; j.len = len; j.n = nfiles; j.fragment = fragment; j.next = 0; j.frags = 0;
  std::vector<pthread_t> th(threads);
  for (int t = 0; t < threads; ++t) pthread_create(&th[t], 0, frag_worker, &j);
  for (int t = 0; t < threads; ++t) pthread_join(th[t], 0);
  return j.frags.load();
}

}  // extern "C"
