/* zq_b200.h -- C ABI of libzqb200.so: the H100 (sm_90a) implementation of zpaqfranz's two
 * data-parallel hot paths (SURVEY.md §8): libzpaq block compression and the dedup fragmenter with
 * its fragment/file hashes.  Plain pointers and sizes only; no C++/torch types cross this line.
 *
 * Every entry point cites the reference interface it replaces ("Z:" = zpaqfranz.cpp line).
 * All functions return 0 on success and a negative code on failure; zq_last_error() gives the text
 * the reference would have passed to libzpaq::error() (Z:12560 / Z:27148).  There is NO CPU
 * fallback: without a usable CUDA device zq_create() fails and every compute entry point returns
 * ZQ_E_NODEVICE.
 */
#ifndef ZQ_B200_H
#define ZQ_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct zq_ctx zq_ctx;

enum {
  ZQ_OK = 0,
  ZQ_E_NODEVICE = -1,   /* no CUDA device / driver error                      */
  ZQ_E_ARG = -2,        /* bad argument                                       */
  ZQ_E_METHOD = -3,     /* libzpaq::error() text in zq_last_error()           */
  ZQ_E_NOMEM = -4,      /* device or host allocation failed ("Out of memory") */
  ZQ_E_OUTPUT = -5,     /* caller's output buffer too small                   */
  ZQ_E_UNSUPPORTED = -6 /* valid ZPAQ input this build has no device path for */
};

/* ---- lifetime ------------------------------------------------------------------------------- */
/* One context per host thread / CUDA device (mirrors "one Compressor per thread", ZSFX/libzpaq.h:56). */
zq_ctx* zq_create(int device);
void zq_destroy(zq_ctx* ctx);
const char* zq_last_error(zq_ctx* ctx);      /* ctx may be NULL: error of the last failed zq_create */
const char* zq_version(void);
/* Run all of this context's work on the caller's CUDA stream (a cudaStream_t, e.g. torch's current
 * stream) instead of the context's own; pass NULL to go back. The stream is not owned. */
int zq_set_stream(zq_ctx* ctx, void* cuda_stream);
/* Several contexts on one device (zq_pipe does this): fn(arg, 2) is called before a batch's input copy is queued and
 * fn(arg, 3) once it has landed; fn(arg, 1) after the batch's planning and before its first kernel, fn(arg, 0) after its
 * last kernel has finished and before the output copy.  Mutexes behind fn make the batches copy in and compute in
 * turns, so that one batch's copies always run under another's kernels instead of all copying and then all computing
 * at the same time.  fn = NULL removes the gate. */
int zq_set_compute_gate(zq_ctx* ctx, void (*fn)(void* arg, int acquire), void* arg);

/* ---- host-side planning (no GPU needed) ------------------------------------------------------ */
/* What libzpaq::compressBlock derives before touching data (Z:20262-20394): the expanded method,
 * makeConfig's args and the assembled block header / PCOMP bytes (Compiler, Z:15904).
 * Buffers may be NULL to query sizes.  data/n are only read for digit levels >= 5. */
int zq_plan_block(const char* method, const uint8_t* data, uint32_t n,
                  char* expanded, size_t expanded_cap, int args9[9],
                  uint8_t* header, uint32_t* header_len,   /* in: capacity, out: length */
                  uint8_t* pcomp, uint32_t* pcomp_len,
                  char* errbuf, size_t errcap);

/* ---- block compression ------------------------------------------------------------------------
 * Element-wise == libzpaq::compressBlock(StringBuffer* in, Writer* out, method, filename, comment,
 * dosha1) (Z:20255): unit u reads in_base[in_off[u] .. +in_len[u]) and produces one complete ZPAQ
 * block (tag .. 0xFF) at out_base[out_off[u] .. +out_len[u]).  Blocks are laid out back to back in
 * unit order, so the concatenation is a valid archive stream.
 *   method/filename/comment: arrays of n C strings, or NULL; if `uniform` != 0 only element [0] of
 *   each non-NULL array is read and applied to every unit.
 * Host variant: in_base/out_base are host pointers (pinned or pageable); H2D/D2H are part of the call. */
int zq_compress_blocks(zq_ctx* ctx, int n,
                       const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                       const char* const* method, const char* const* filename,
                       const char* const* comment, int uniform, int dosha1,
                       uint8_t* out_base, uint64_t out_cap,
                       uint64_t* out_off, uint32_t* out_len);

/* Device variant: in_base/out_base are device pointers on ctx's device; offsets/lengths stay on the
 * host.  Used for HBM-resident measurement and by callers that already staged data.
 * Like libzpaq::compressBlock, which filters its StringBuffer in place (E8E9, Z:19363 / Z:20414), a method whose type
 * has the exe bit set (args[1] & 4) REWRITES the unit's bytes in d_in_base: units of such a call must not overlap and
 * the buffer cannot be submitted a second time without being refilled.  (The host variant filters its staged copy;
 * the caller's bytes stay untouched.) */
int zq_compress_blocks_device(zq_ctx* ctx, int n,
                              const uint8_t* d_in_base, const uint64_t* in_off, const uint32_t* in_len,
                              const char* const* method, const char* const* filename,
                              const char* const* comment, int uniform, int dosha1,
                              uint8_t* d_out_base, uint64_t out_cap,
                              uint64_t* out_off, uint32_t* out_len);

/* ---- batches in flight ---------------------------------------------------------------------------------
 * The counterpart of CompressJob's block queue (appendz / compressThread / writeThread, Z:71364-71520): `depth`
 * lanes, each with its own context, stream and worker thread, so the copies and kernels of the next batch fill the
 * tail of the current one.  zq_pipe_submit takes the arguments of zq_compress_blocks (device_pointers = 0) or
 * zq_compress_blocks_device (= 1) and returns a ticket >= 0; all argument arrays and buffers must stay valid and
 * untouched until zq_pipe_wait(ticket) returns the call's result.  Batches run in submission order per lane;
 * results are those of the synchronous calls. */
typedef struct zq_pipe zq_pipe;
zq_pipe* zq_pipe_create(int device, int depth);
void zq_pipe_destroy(zq_pipe* pipe);
int zq_pipe_submit(zq_pipe* pipe, int n,
                   const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                   const char* const* method, const char* const* filename, const char* const* comment,
                   int uniform, int dosha1, int device_pointers,
                   uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len);
int zq_pipe_wait(zq_pipe* pipe, int ticket);
const char* zq_pipe_last_error(zq_pipe* pipe);
uint64_t zq_pipe_launch_count(zq_pipe* pipe);

/* ---- caller-supplied models ---------------------------------------------------------------------
 * == libzpaq::Compressor used directly (Z:15970-16187): writeTag / startBlock(hcomp) / startSegment(filename,
 * comment) / postProcess(pcomp, len) / compress(-1) / endSegment(sha1string) / endBlock, once per unit.
 *   header:  the block header exactly as it is stored (hsize[2] hh hm ph pm n comp.. 0 hcomp.. 0, Z:14084);
 *   pcomp:   PCOMP bytecode to announce to the decoder (NULL/0: "0" = no post-processing);
 *   the unit's bytes go to the coder AS THEY ARE (any pre-processing matching pcomp is the caller's);
 *   comment: stored verbatim (compressBlock's "<n> " prefix is compressBlock's own, Z:20404);
 *   sha1_digests: n x 20 bytes stored as the segments' checksums, or NULL for none;
 *   write_tag: emit the 13-byte locator tag in front of each block.
 * n == 0 components -> stored/unmodeled framing, else arithmetic coded with the given component chain. */
int zq_compress_segments(zq_ctx* ctx, int n,
                         const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                         const uint8_t* header, uint32_t header_len,
                         const uint8_t* pcomp, uint32_t pcomp_len,
                         const char* const* filename, const char* const* comment, int uniform,
                         const uint8_t* sha1_digests, int write_tag,
                         uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len);

/* == libzpaq::Compiler (Z:15904) as Compressor::startBlock(config, args, pcomp_cmd) uses it: ZPAQL source ->
 * stored block header + PCOMP bytecode (+ the text between "pcomp" and ";").  No GPU needed.
 * header_len / pcomp_len: in = capacity, out = length. */
int zq_assemble_config(const char* config, const int args9[9],
                       uint8_t* header, uint32_t* header_len, uint8_t* pcomp, uint32_t* pcomp_len,
                       char* pcomp_cmd, size_t pcomp_cmd_cap, char* errbuf, size_t errcap);

/* ZPAQL source of the built-in models Compressor::startBlock(int level) selects (Z:15989): 1 = min.cfg,
 * 2 = mid.cfg; NULL for other levels. */
const char* zq_model_config(int level);

/* ---- block decompression -------------------------------------------------------------------------
 * Element-wise == Decompresser::findBlock/findFilename/readComment/decompress/readSegmentEnd over every segment of
 * one block (Z:15418-15534) and libzpaq::decompress (Z:15536): unit u is a complete block at
 * in_base[in_off[u] .. +in_len[u]) (the 13-byte locator tag is optional); the restored bytes of all its segments,
 * concatenated, go to out_base[out_off[u] .. +out_len[u]), laid out back to back.  The expected size of each block is
 * taken from expect_len[u] or, when expect_len is NULL, from the decimal number that starts the FIRST segment's comment
 * (the archiver writes "<n> jDC\x01", Z:20404; a block of several segments needs expect_len, else ZQ_E_OUTPUT).  Every
 * stored SHA-1 is verified on the device.  Where the segments of the last call lie: zq_decompress_last_segments.
 * Host pointers. */
int zq_decompress_blocks(zq_ctx* ctx, int n,
                         const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                         const uint32_t* expect_len /* may be NULL */,
                         uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len);

/* Same, and additionally reports per block (either may be NULL): in_used[u] = offset, from the block's start, of
 * the byte that follows the segment trailer (the end-of-block 0xFF), and sha1_out[u*21 ..] = readSegmentEnd()'s
 * 21-byte answer (1 + stored SHA-1, or 0).  in_len[u] may run past the end of the block (e.g. to the end of
 * the stream): decoding stops at the segment's end. */
int zq_decompress_blocks_ex(zq_ctx* ctx, int n,
                            const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                            const uint32_t* expect_len /* may be NULL */,
                            uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len,
                            uint32_t* in_used, uint8_t* sha1_out);
/* The segments of the blocks of the last zq_decompress_* call on this context, ordered by block, then position:
 * restored bytes [out_begin, out_end) of the block's output, and the offset within the block of the segment's trailer
 * byte (253 + SHA-1, or 254); the next segment's header (1, filename, 0, comment, 0, 0) follows the trailer.  The table
 * belongs to the context and is valid until its next decompress call. */
typedef struct zq_segment { uint32_t block, out_begin, out_end, trailer; } zq_segment;
int zq_decompress_last_segments(zq_ctx* ctx, const zq_segment** segs, uint64_t* nsegs);

/* The first max_out[i] bytes of each block's first segment (== Decompresser::decompress(n), Z:15480: a caller that only
 * wants the head of a segment); stops there, looks at no trailer, verifies no checksum.  out_len[i] <= max_out[i]. */
int zq_decompress_prefix(zq_ctx* ctx, int n, const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len,
                         const uint32_t* max_out, uint8_t* out_base, uint64_t out_cap, uint64_t* out_off, uint32_t* out_len);

/* Upper bound of one block's compressed size for an n-byte input (any method, names <= 255 bytes). */
uint64_t zq_compress_bound(uint32_t n);

/* ---- hashes: n independent buffers -> n digests ----------------------------------------------
 * == libzpaq::SHA1::write+result (Z:12637), libzpaq::SHA256 (Z:12828), XXH3_128bits (Z:24710,
 * printed high64||low64, Z:67189), blake3_hasher_* (Z:22143-22221).  Host pointers. */
int zq_sha1(zq_ctx* ctx, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests20);
int zq_sha256(zq_ctx* ctx, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests32);
int zq_xxh3_128(zq_ctx* ctx, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests16);
int zq_blake3(zq_ctx* ctx, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests32);
/* device-pointer variants (digests also written to device memory) */
int zq_sha1_device(zq_ctx* ctx, int n, const uint8_t* d_base, const uint64_t* off, const uint64_t* len, uint8_t* d_digests20);

/* ---- dedup fragmenter --------------------------------------------------------------------------
 * == the content-defined chunker inlined in Jidac::add (Z:122180-122574; canonical loop
 * Z:95604-95633; constants Z:121626-121631): for each of nfiles independent byte streams emit the
 * fragment lengths, per-fragment `hits` and per-fragment SHA-1 (the dedup key, Z:122569).
 * Output arrays are filled file after file; frag_first[f] .. frag_first[f+1] index file f's fragments
 * (frag_first has nfiles+1 entries).  `fragment` is -fragment N (default 6); blocksize as in
 * Z:121622-121625.  Host pointers. */
int zq_fragment(zq_ctx* ctx, int nfiles, const uint8_t* base, const uint64_t* off, const uint64_t* len,
                int fragment, uint32_t blocksize,
                uint32_t* frag_len, uint32_t* frag_hits, uint8_t* frag_sha1 /* may be NULL */,
                uint64_t frag_cap, uint64_t* frag_first);

/* Same, plus frag_o1 (256 bytes per fragment, may be NULL): the chunker's order-1 prediction table as it stands
 * at the end of each fragment -- the input of the archiver's text/exe/redundancy heuristics (Z:122592-122634). */
int zq_fragment_ex(zq_ctx* ctx, int nfiles, const uint8_t* base, const uint64_t* off, const uint64_t* len,
                   int fragment, uint32_t blocksize,
                   uint32_t* frag_len, uint32_t* frag_hits, uint8_t* frag_sha1, uint8_t* frag_o1,
                   uint64_t frag_cap, uint64_t* frag_first);

/* ---- the archiver's add loop over files in memory ------------------------------------------------------
 * == the body of Jidac::add between "for each file" and the index blocks (Z:122113-122911) for a fresh archive:
 * fragment every file (device), look each fragment up by SHA-1, run the data-type heuristics on the new ones,
 * pack them into blocks by the reference's new-block rule and compress every block (device).  Files are taken
 * in the order given; the reference's order is ascending zq_file_sort_key(path, size), then path.
 *   method:   -method as typed ("2", "14", "x..."); fragment: -fragment N; date14: the version's date as 14 digits
 *   first_id: id of the first new fragment (1 for a new archive)
 *   d_out:    the "d" blocks back to back, as they follow the version's header block in the archive
 *   h_out:    the "h" blocks (compressed size + SHA-1/size per fragment of each data block), in order
 *   file_frags[file_first[f] .. file_first[f+1]): fragment ids of file f (what its index entry lists).
 * The "c" header and "i" index blocks of the transaction are written by zq_journal_header / zq_journal_index. */
int zq_add_files(zq_ctx* ctx, int nfiles, const uint8_t* base, const uint64_t* off, const uint64_t* len,
                 const char* method, int fragment, const char* date14, uint32_t first_id,
                 uint8_t* d_out, uint64_t d_cap, uint64_t* d_len,
                 uint8_t* h_out, uint64_t h_cap, uint64_t* h_len,
                 uint32_t* file_frags, uint64_t file_frags_cap, uint64_t* file_first /* nfiles+1 */,
                 uint32_t* nblocks);
uint64_t zq_file_sort_key(const char* path, int64_t size);

/* One stream hashed in pieces (what the streaming classes libzpaq::SHA1 / SHA256 do, zpaqfranz.cpp:12637 / 12828):
 * the compression function over nblocks whole 64-byte blocks of data, from and to the chaining value in state
 * (SHA-1: 5 words from 67452301 ...; SHA-256: 8 words from 6a09e667 ...).  Padding and the length field are the
 * caller's last block(s) (include/libzpaq_b200.h does it).  One dependency chain = one thread: this bounds the host
 * memory of a long stream, it is not the fast way to hash many buffers (zq_sha1 / zq_sha256 are). */
int zq_sha1_continue(zq_ctx* ctx, uint32_t state[5], const uint8_t* data, uint64_t nblocks);
int zq_sha256_continue(zq_ctx* ctx, uint32_t state[8], const uint8_t* data, uint64_t nblocks);

/* The fragment index (replaces HTIndex::find, zpaqfranz.cpp:71567-71604): first[i] = the smallest j <= i whose 20-byte
 * digest equals fragment i's, for n digests laid out back to back.  first[i] == i marks a fragment new to the set. */
int zq_dedup_first(zq_ctx* ctx, uint64_t n, const uint8_t* sha1, uint32_t* first);

/* The other two journaling blocks of a transaction (device compression, method "0" / "1", comment "jDC\x01").
 * zq_journal_header: the "c" block -- 8 bytes, cdata = size of the data blocks that follow, or -1 while the update is
 *   open; htsize = id of the first new fragment.  Replaces writeJidacHeader (zpaqfranz.cpp:71521-71540).
 * zq_journal_index: the "i" blocks -- per record date (0 = deletion), name, and for live files the attribute bytes
 *   (attr_base + attr_off[r], attr_len[r] bytes, as the front end's writefranzattr lays them out; opaque here) and the
 *   fragment ids frags[frag_first[r] .. frag_first[r+1]); a block closes once it passes 16 000 bytes.  Replaces the
 *   index loop of Jidac::add (zpaqfranz.cpp:122915-123100).  out: the blocks back to back. */
int zq_journal_header(zq_ctx* ctx, const char* date14, int64_t cdata, uint32_t htsize,
                      uint8_t* out, uint64_t cap, uint64_t* len);
int zq_journal_index(zq_ctx* ctx, const char* date14, int nrec, const int64_t* date, const char* const* name,
                     const uint8_t* attr_base, const uint64_t* attr_off, const uint32_t* attr_len,
                     const uint64_t* frag_first /* nrec+1 */, const uint32_t* frags,
                     uint8_t* out, uint64_t cap, uint64_t* len, uint32_t* nblocks);


/* ---- several GPUs (one process per GPU) -------------------------------------------------------------------------
 * Units shard over the ranks with no data-path collective (SURVEY.md section 8e): every rank runs the single-device
 * entry points above on its own units.  What is exchanged, through NCCL over NVLink, is small:
 *   zq_dist_exchange_sizes  the compressed size of every block (4 B each) -> global archive offsets on every rank;
 *                           replaces the running offset of the reference's single writer thread (Z:71445-71518)
 *   zq_dist_dedup           the 20-byte SHA-1 of every fragment -> which local fragments are new to the archive;
 *                           replaces the HTIndex lookup of Jidac::add (Z:122569-122573, Z:71567-71604)
 * Rank 0 calls zq_dist_unique_id and hands the 128 bytes to the other ranks (launcher's job: environment, file, MPI,
 * torch.distributed ...); every rank then calls zq_dist_create.  world == 1 needs neither NCCL nor an id.
 * zq_dist_create_cb runs the same logic over a caller-supplied all-gather (tests: gloo on CPUs). */
typedef struct zq_dist zq_dist;
/* every rank contributes `bytes` bytes at `in`; `out` receives world * bytes in rank order; returns 0 on success */
typedef int (*zq_allgather_fn)(void* user, const void* in, void* out, size_t bytes);
int zq_dist_unique_id(uint8_t out[128]);
zq_dist* zq_dist_create(int device, int rank, int world, const uint8_t id[128]);
zq_dist* zq_dist_create_cb(int rank, int world, zq_allgather_fn fn, void* user);
void zq_dist_destroy(zq_dist* d);
const char* zq_dist_last_error(zq_dist* d);     /* d may be NULL: error of the last failed create / unique_id */
uint64_t zq_dist_bytes_exchanged(zq_dist* d);   /* payload bytes received by this rank so far */
/* contiguous balanced shard [lo, hi) of `total` units; longest-first assignment for units of unequal cost */
int zq_dist_shard_range(uint64_t total, int rank, int world, uint64_t* lo, uint64_t* hi);
int zq_dist_shard_lpt(const uint64_t* cost, uint64_t n, int world, int32_t* owner);
/* local_sizes: compressed sizes of this rank's shard (zq_dist_shard_range order) -> all_sizes[total], offsets[total] */
int zq_dist_exchange_sizes(zq_dist* d, const uint32_t* local_sizes, uint64_t total, uint32_t* all_sizes, uint64_t* offsets);
/* local_digests: n_local x 20 bytes in archive order -> is_first[n_local] (1: store it, 0: reference an earlier one),
 * unique_total: fragments stored by all ranks together */
int zq_dist_dedup(zq_dist* d, const uint8_t* local_digests, uint64_t n_local, uint8_t* is_first, uint64_t* unique_total);

/* One stream (a file larger than one GPU's share, e.g. a disk image) cut across the ranks -- replaces, for that file,
 * the single sequential chunker loop of Jidac::add (zpaqfranz.cpp:122457-122561): rank r owns the bytes [lo, hi) of the
 * stream (hi of rank r == lo of rank r+1) and also holds the `overlap` bytes after hi, up to avail_end.  It runs
 * zq_fragment over [from, avail_end) with from = lo: a speculative chain.  zq_dist_stitch_fragments (collective: one
 * all-gather of the fragment end offsets, 8 B each) then finds where the real chain, coming from the left, lands on a
 * boundary this rank's chain shares; the chunker's state is reset at every boundary, so the chains are identical from
 * there on.  Result, the same fragments the reference cuts from the whole stream:
 *   again == 0: this rank's fragments first_keep .. first_keep + n_keep are the stream's fragments number
 *               global_first .. (of global_total), covering the bytes [begin, end); the fragment that straddles hi
 *               belongs to the left owner.  Their SHA-1s from zq_fragment are valid as they are.
 *   again == 1: some chain did not meet its neighbour's inside the overlap (constant runs -- zero pages -- never
 *               re-synchronise).  The rank with restart == 1 fragments [restart_at, avail_end) afresh (restart_at is
 *               the real boundary it has to start from); then EVERY rank calls again, the others with the arguments
 *               they used before.  At most world - 1 repetitions.
 * ZQ_E_UNSUPPORTED: the overlap is shorter than one fragment (choose overlap >= 8128 << fragment). */
typedef struct zq_stitch {
  uint64_t first_keep, n_keep;      /* this rank's fragments that are fragments of the stream */
  uint64_t global_first, global_total;
  uint64_t begin, end;              /* bytes of the stream they cover */
  uint64_t restart_at;
  int32_t again, restart;
} zq_stitch;
int zq_dist_stitch_fragments(zq_dist* d, uint64_t stream_total, uint64_t lo, uint64_t hi, uint64_t from, uint64_t avail_end,
                             const uint32_t* frag_len, uint64_t nfrag, zq_stitch* out);

/* ---- introspection for tests / bench ---------------------------------------------------------- */
/* number of kernel launches issued by this context since creation */
uint64_t zq_launch_count(zq_ctx* ctx);
/* elapsed device time (ms, CUDA events on the context's stream) of the stages of the most recent
 * zq_compress_blocks* call: [0] total, [1] sha1, [2] suffix sort + lcp, [3] lz parse, [4] framing/
 * gather, [5] modeling/coding, [6] h2d, [7] d2h.  Unused stages are 0. */
int zq_last_timings(zq_ctx* ctx, float ms[8]);
/* the same plus the stages of the LZ77 parse pipeline: [8] look-ahead-0 scan, [9] look-ahead-1 scan, [10] walk,
 * [11] emit; n <= 16 values are written. */
int zq_last_timings_ex(zq_ctx* ctx, float* ms, int n);
/* debugging aid for the parity tests: suffix array (u32[n]) of one buffer, computed on the device */
int zq_suffix_array(zq_ctx* ctx, const uint8_t* data, uint32_t n, uint32_t* sa_out);

/* CRC-32 (crc32_16bytes, Z:30299: always on in Jidac::updatehash, Z:85948) and XXH64 seed 0 (the archiver's default
 * file hash, XXH64 Z:24688) of n buffers: digests = 4 / 8 bytes per buffer, little-endian.  Bit-exact against zlib and
 * the reference's XXH64 under the emulator and on the GPU (SURVEY.md §8f rank 4). */
int zq_crc32(zq_ctx* ctx, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests);
int zq_xxh64(zq_ctx* ctx, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests);
/* MD5 (16 bytes) and SHA3-256 (32 bytes) of n buffers: the -md5 / -sha3 file hashes of updatehash (MD5::add Z:21616,
 * SHA3::add Z:21337; SURVEY.md section 8f rank 4). */
int zq_md5(zq_ctx* ctx, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests16);
int zq_sha3_256(zq_ctx* ctx, int n, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint8_t* digests32);

/* ---- ZPAQL -> CUDA C translation (host only, no GPU needed) -------------------------------------
 * libzpaq compiles a block's HCOMP/PCOMP to x86 when the block starts (ZPAQL::assemble, Z:16358, called from ZPAQL::run Z:17677).
 * zq_jit_context_source does the source-to-source equivalent for the HCOMP of a block header (hsize ..
 * hcomp 0, as zq_plan_block returns it): a translation unit with `zq_hcomp` (one run of the program) and the
 * kernel `zq_ctx_kernel` (one thread per block, H[0..n) after every byte).  zq_jit_compile runs NVRTC on such a
 * source for sm_90a and reports the cubin size.  Groundwork: the compress path still interprets (DESIGN.md §9).
 * src may be NULL to query the length.  ZQ_E_UNSUPPORTED: program outside the translator's cover / no NVRTC. */
int zq_jit_context_source(const uint8_t* header, uint32_t header_len, char* src, uint32_t src_cap, uint32_t* src_len,
                          char* errbuf, size_t errcap);
int zq_jit_compile(const char* src, uint32_t* cubin_size, char* log, size_t logcap);
/* Same translation unit plus `zq_encode_block`: the block's model written out as straight-line code (every
 * component in index order, sizes / masks / rates / table offsets as literals) -- Predictor::predict0/update0 and
 * Encoder::encode specialised for this header, the generalisation of the chain fast path. */
int zq_jit_coder_source(const uint8_t* header, uint32_t header_len, char* src, uint32_t src_cap, uint32_t* src_len,
                        char* errbuf, size_t errcap);

#ifdef __cplusplus
}
#endif
#endif /* ZQ_B200_H */
