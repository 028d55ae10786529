/*
 * include/smr_b200.h -- C ABI of the GPU-native (H100, sm_90a) alignment hot path (libsmr_b200.so).
 *
 * The reference (sortmerna v5.0.0) has no FFI; the seam this library replaces is the C++ call
 *     void align(Readfeed&, Readstats&, Index&, KeyValueDatabase&, Runopts&)
 *         (src/sortmerna/processor.cpp:173, called from src/sortmerna/main.cpp:88,99,105)
 * whose unit of work is
 *     void traverse(Runopts&, Index&, References&, Readstats&, Refstats&, Read&, bool)
 *         (src/sortmerna/paralleltraversal.cpp:81-90).
 * Each entry point below names the reference code it stands in for.  All functions return 0 on
 * success and a non-zero smr_status otherwise (the reference prints and exit()s; a host wrapper
 * maps non-zero to that).  Plain pointers and sizes only; no C++ or torch types.  Every compute
 * entry point requires a CUDA device: there is no CPU fallback.
 */
#ifndef SMR_B200_H
#define SMR_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct smr_ctx smr_ctx; /* opaque; one per GPU, driven by one host thread */

enum smr_status {
  SMR_OK = 0,
  SMR_ERR_CUDA = 1,        /* a CUDA call failed (smr_last_error has the text) */
  SMR_ERR_ARG = 2,         /* invalid argument */
  SMR_ERR_INDEX = 3,       /* malformed index file (index.cpp:282-286 is fatal in the reference too) */
  SMR_ERR_UNSUPPORTED = 4, /* option combination outside this build (see DESIGN.md) */
  SMR_ERR_CAPACITY = 5,    /* caller-provided output buffer too small */
  SMR_ERR_NO_DEVICE = 6    /* no CUDA device / extension cannot run: fail loudly, never fall back */
};

/* The opts.* fields that cross the seam (SURVEY 8(b)); defaults are those of
 * Runopts::validate (src/sortmerna/options.cpp:1684-1738). */
typedef struct {
  int32_t match, mismatch, score_N, gap_open, gap_ext; /* --match --mismatch -N --gap_open --gap_ext */
  int32_t num_seeds, min_lis, edges, edges_is_percent; /* --num_seeds --min_lis --edges */
  int32_t num_alignments, is_best;                     /* --num_alignments / --best / --no-best */
  int32_t is_forward, is_reverse, is_full_search;      /* -F -R --full_search */
  int32_t minoccur;                                    /* include/options.hpp:572 (no CLI option) */
} smr_params;

/* Per-read result = the fields Read::toBinString persists (src/sortmerna/read.cpp:429-462), i.e.
 * what the unchanged report stage reads back through Read::load_db. */
typedef struct {
  uint32_t lastIndex, lastPart;
  uint32_t hit_seeds;
  uint32_t min_index, max_index; /* alignment_struct2 (include/ssw.hpp:157-159) */
  uint32_t n_align;              /* alignv.size() */
  uint16_t max_SW_count;
  uint8_t is_done, is_hit;
} smr_read_result;

/* One stored alignment = s_align2 (include/ssw.hpp:44-56); slot (read * max(1,num_alignments) + k), or in the packed layout
 * (smr_set_aln_layout) sum_{j<read} n_align(j) + k */
typedef struct {
  uint32_t cigar_off, cigar_len; /* into the cigar pool; BAM style len<<4|op, op 0=M 1=I 2=D (ssw.c:750-758) */
  uint32_t ref_num;
  int32_t ref_begin1, ref_end1, read_begin1, read_end1;
  uint32_t readlen;
  uint16_t score1, part, index_num;
  uint8_t strand, pad;
} smr_aln;

/* Index builder (host code, no GPU needed; SURVEY 8(f)(3)).  Replaces build_index (src/sortmerna/indexdb.cpp:1119-2095): writes
 * <out_prefix>.kmer_P.dat / .bursttrie_P.dat / .pos_P.dat for every part P and <out_prefix>.stats in the reference's on-disk
 * format -- the files Index::load (index.cpp:143-357), Refstats::load (refstats.cpp:103-190) and smr_load_index_part read.
 * Content is that of the reference's builder (same windows, alphabet map, burst tries, counts, position lists, part split);
 * only the arbitrary numbering of the unique L-mers differs (order of first occurrence instead of a CMPH hash value).
 * lnwin = -L (18), interval = -interval (1), max_pos = -max_pos (10000; 0 = all), max_mb = -m (3072); threads: 2*threads
 * workers build the tries of disjoint 9-mer classes (0 = cores/8 clamped to 1..8); the files do not depend on it.
 * report6 (optional): parts, sequences, windows, unique L-mers, trie nodes, bytes written.  err: message buffer. */
int smr_build_index(const char* fasta_path, const char* out_prefix, uint32_t lnwin, uint32_t interval, uint32_t max_pos,
                    double max_mb, uint32_t threads, uint64_t* report6, char* err, size_t err_cap);

/* KVDB blob writer (host code; SURVEY 8(f)(4)): for every read of a batch the byte string Read::toBinString() would store
 * under its id (src/sortmerna/read.cpp:429-462; alignment_struct2::toString read.cpp:79-101; s_align2::toString
 * include/ssw.hpp:106-140), written straight from the result buffers, so Read::load_db (read.cpp:467-539) reads back what the
 * CPU path would have stored.  Reads without a stored alignment get an empty blob (read.cpp:431-432).
 * num_alignments = opts.num_alignments; denovo4 (optional) = per read {c_yid_ycov, n_yid_ncov, n_nid_ycov, n_denovo}
 * (zero while aligning; set by denovo_stats).  blob_off[0..nreads] receives the offsets; call with out == nullptr to size. */
int smr_pack_kvdb_blobs(const smr_read_result* results, const smr_aln* alns, const uint32_t* cigar_pool, uint32_t nreads,
                        uint32_t slots, int32_t num_alignments, const uint32_t* denovo4, uint8_t* out, uint64_t out_cap,
                        uint64_t* blob_off);
/* The same blobs from packed results (SMR_ALNS_PACKED): read r's alignments at sum_{j<r} results[j].n_align.  Gives the bytes
 * smr_pack_kvdb_blobs gives for the strided equivalent. */
int smr_pack_kvdb_blobs_packed(const smr_read_result* results, const smr_aln* alns, const uint32_t* cigar_pool, uint32_t nreads,
                               int32_t num_alignments, const uint32_t* denovo4, uint8_t* out, uint64_t out_cap, uint64_t* blob_off);

/* Report-side arithmetic of one stored alignment = Read::calc_miss_gap_match (src/sortmerna/read.cpp:547-589), computed on the
 * GPU from the CIGAR it has just produced (SURVEY 8(f)(1)): what %id / %cov / NM:i / BLAST columns 3,5,6 are derived from. */
typedef struct {
  uint32_t n_miss, n_gap, n_match;
  /* n_match as denovo_stats_run obtains it (src/sortmerna/processor.cpp:329-357): that caller does NOT reverse-complement
   * the read first, so for a reverse-strand alignment the CIGAR is walked over the forward read.  Reproduced as is, because
   * n_yid_ycov / n_yid_ncov / n_nid_ycov / n_denovo and aligned_denovo.* depend on it; equals n_match on the forward strand. */
  uint32_t n_match_denovo;
} smr_aln_stats;

/* Counters.  The first block is Readstats (include/readstats.hpp:77-84) as mutated by this path;
 * it is what the single NCCL all-reduce sums across GPUs.  The second block is instrumentation
 * used for the roofline arithmetic (SURVEY 8(d)). */
enum {
  SMR_CNT_NUM_ALIGNED = 0,   /* readstats.num_aligned (alignment.cpp:414) */
  SMR_CNT_NUM_SHORT = 1,     /* readstats.num_short of the LAST index pass (processor.cpp:109-114,228) */
  /* SW_CALLS, SW_CELLS, POS_ENTRIES and LIS_CALLS count the work done, so they also count the first (failed) pass of a read
   * that overflowed its scratch and was run again (smr_align_batch, smr_download_results). */
  SMR_CNT_SW_CALLS = 2,      /* ssw_align-equivalent calls */
  SMR_CNT_SW_CELLS = 3,      /* sum refLen*readLen over those calls (forward pass only) */
  SMR_CNT_WINDOWS = 4,       /* seed windows searched (speculative windows included) */
  SMR_CNT_TRIE_NODES = 5,    /* trie nodes visited */
  SMR_CNT_BUCKETS = 6,       /* buckets visited */
  SMR_CNT_BUCKET_ENTRIES = 7,/* bucket entries visited */
  SMR_CNT_POS_ENTRIES = 8,   /* position entries touched by candidate voting */
  SMR_CNT_LIS_CALLS = 9,     /* compute_lis_alignment-equivalent calls */
  /* 10..22: warp-cycle accounting of the candidate kernel (max per read, sum, kernel, then per phase) */
  SMR_CNT_FIXED = 32         /* reads_matched_per_db[i] lives at counters[SMR_CNT_FIXED + i] */
};

/* -- lifetime ------------------------------------------------------------------------------- */
int smr_init(int device, smr_ctx** out);
void smr_destroy(smr_ctx*);
const char* smr_last_error(const smr_ctx*); /* text of the last failure on this context */
int smr_device_count(void);                 /* number of visible CUDA devices (0 if none) */

/* -- index + references: Index::load (src/sortmerna/index.cpp:143-357) and References::load
 *    (src/sortmerna/references.cpp:55-164) for one (index_num, part), in --ref order.  Takes the
 *    raw bytes of <idx>.kmer_<p>.dat / .bursttrie_<p>.dat / .pos_<p>.dat, flattens them to
 *    contiguous HBM arrays and keeps them resident (all indexes stay loaded unless an index budget is
 *    set, smr_set_index_budget; the reference loads and unloads one at a time, processor.cpp:225-266).
 *    refseq_cat: reference sequences in the 0..4 alphabet (nt_table, common.hpp:68-77), concatenated;
 *    ref_off[nref+1] offsets.  minimal_score / lnwin / skiplengths come from Refstats
 *    (src/sortmerna/refstats.cpp:147-166,259-265). */
int smr_load_index_part(smr_ctx*, uint32_t index_num, uint32_t part,
                        const void* kmer_file, size_t kmer_bytes,
                        const void* bursttrie_file, size_t bursttrie_bytes,
                        const void* pos_file, size_t pos_bytes,
                        const uint8_t* refseq_cat, const uint64_t* ref_off, uint32_t nref,
                        uint32_t lnwin, uint32_t minimal_score, const uint32_t skiplengths[3]);
/* Index build on the device (SURVEY 8(f)(3)): what smr_build_index + smr_load_index_part do for every part of the index of
 * `fasta_path`, without the files -- the FASTA is parsed on the host (records, alphabet maps, the part split rule of
 * indexdb.cpp:1381-1431), then windows, unique L-mers, position lists and the burst-trie order of every list are computed on the
 * device with sorts (sortmerna_b200/csrc/smr_build_dev.cuh) and stay resident.  Replaces build_index (src/sortmerna/indexdb.cpp:
 * 1119-2095) + Index::load (index.cpp:143-357) + References::load (references.cpp:55-154) for this index.  The arrays equal those
 * smr_load_index_part makes from the reference builder's files up to the numbering of the L-mer ids.
 * *nparts = parts made (ordinals continue the context's part list); report6 as for smr_build_index (nodes: 0). */
int smr_build_index_device(smr_ctx*, uint32_t index_num, const char* fasta_path, uint32_t lnwin, uint32_t interval, uint32_t max_pos, double max_mb,
                           const uint32_t skiplengths[3], uint32_t minimal_score, uint32_t* nparts, uint64_t report6[6]);
/* Test hook: resident array `which` of loaded part `slot` (0 flookup, 1 flist, 2 pos_off, 3 pos, 4 refseq, 5 ref_off); the
 * host copy of a search array that an index budget holds on the host. */
int smr_debug_index_array(smr_ctx*, uint32_t slot, uint32_t which, void* out, uint64_t cap_bytes, uint64_t* nbytes);
/* refstats.minimal_score depends on the read set (refstats.cpp:247-265): update without reloading */
int smr_set_minimal_score(smr_ctx*, uint32_t index_num, uint32_t minimal_score);
int smr_set_params(smr_ctx*, const smr_params*);
/* out[0]=#parts loaded [1]=bytes resident in HBM [2]=trie nodes [3]=bucket entries [4]=ids [5]=positions.  out[1] counts what is
 * on the device now: under an index budget, the index arena and the parts that hold their own search arrays. */
int smr_index_info(const smr_ctx*, uint64_t out[6]);

/* -- index budget: bounded device memory for index sets larger than the GPU (the reference's one part at a time, -m).
 *    `bytes` limits the device bytes of the parts' SEARCH arrays (flookup, ftext, fid, pos_off, pos); 0 = no limit, the default.
 *    refseq, ref_off and the report names of every part stay resident (finalize, the scorer and pairwise BLAST read them).
 *    Groups are formed greedily from consecutive parts in load order (--ref order, then part), each within the budget.  If all parts
 *    fit in one group they stay resident, as without a budget.  Otherwise every part's search arrays are held in pinned host memory,
 *    the device holds one arena of at most `bytes`, and each run uploads the groups into it in order: for each group, every chunk
 *    of the batch is seeded and searched over its parts, the reads' state carrying from group to group as from part to part; every
 *    chunk is finalized after the last group.  Results, counts and counters equal those of a run without a budget; so do the work
 *    counters, except that a read whose seed scratch overflows in a later group has the candidate work of the earlier groups counted
 *    before it is retried.  Scratch-overflow retries and packed re-runs upload the groups again.
 *    May be called before or after loading and takes effect at the next run; loading under a budget keeps the device within the
 *    budget plus the part being loaded (parts built on the device go to the host once built).  A part whose search arrays alone
 *    pass the budget is SMR_ERR_CAPACITY (here for the loaded parts, with the budget unchanged, and when it is loaded), the message
 *    naming it and its size; a failed pinned allocation is SMR_ERR_CUDA. */
int smr_set_index_budget(smr_ctx*, uint64_t bytes);
/* out[0]=groups of the next run [1]=search-array bytes of its largest group [2]=search-array bytes on the device now (the arena
 * included) [3]=pinned host bytes of search arrays [4]=group uploads since smr_init [5]=bytes they uploaded [6]=microseconds of
 * group uploads in the last run of the resident batch, the retries of its download included (device events) */
int smr_index_residency(const smr_ctx*, uint64_t out[7]);

/* -- the hot path: align() (processor.cpp:173-285) over one batch of reads, read-major.
 *    For each read: for each loaded (index,part) in order: forward then reverse strand through
 *    traverse() with KVDB-equivalent carry-over (read.cpp:429-539).
 *    seq_cat: reads in 0..4 (4 = ambiguous, as nt_table yields), concatenated; seq_off[nreads+1].
 *    Host buffers; the call copies host->device, runs, and copies the results back.
 *    results[nreads]; alns[nreads * smr_aln_slots()] (= num_alignments per read; see smr_set_aln_slots for 0); cigar_pool[cigar_cap] u32 words;
 *    counters[SMR_CNT_FIXED + n_index_files] are ADDED to (caller zeroes them).
 *    *cigar_used = words of cigar_pool used.  If cigar_cap is too small the call fails with SMR_ERR_CAPACITY and *cigar_used names
 *    the words the batch needs (more than cigar_cap): call again with a pool at least that large.
 *    Scratch overflow: every read first runs with fixed scratch; a read that outgrows it (many seed hits, a wide traceback band,
 *    many CIGAR operations, a full device CIGAR pool) is run again with 8x the scratch, then 64x and 512x, in a batch of the
 *    flagged reads gathered on the device; after that the call fails with SMR_ERR_CAPACITY.  Results do not depend on it; the
 *    CIGARs of retried reads follow those of the others in cigar_pool.  smr_last_timings sums the kernel and D2H times of the first
 *    run and its retries.  Uploads the batch as the resident batch, with no text behind it (as smr_upload_batch). */
int smr_align_batch(smr_ctx*, const uint8_t* seq_cat, const uint64_t* seq_off, uint32_t nreads,
                    smr_read_result* results, smr_aln* alns,
                    uint32_t* cigar_pool, uint64_t cigar_cap, uint64_t* cigar_used,
                    uint64_t* counters, uint32_t n_counters);

/* "All alignments" (opts.num_alignments == 0, src/sortmerna/alignment.cpp:420-424: every accepted alignment is appended, nothing
 * stops the candidate loop, scripts/test.jinja t9): the number of alignments of a read is unbounded, so the flat result layout needs
 * a stride.  smr_set_aln_slots sets it (default 16); alns[] / stats then hold nreads * slots entries, results[r].n_align of them
 * used.  If a read accepts more, the call fails with SMR_ERR_CAPACITY and smr_aln_slots_needed() names the stride that batch
 * needs (nothing is truncated silently).  smr_aln_slots() = the stride in effect: num_alignments when > 0, else the value set. */
int smr_set_aln_slots(smr_ctx*, uint32_t slots);
uint32_t smr_aln_slots(const smr_ctx*);
uint32_t smr_aln_slots_needed(const smr_ctx*);

/* Result layout of a context (default SMR_ALNS_STRIDED; another value is SMR_ERR_ARG).
 * SMR_ALNS_STRIDED: alns[] / stats hold nreads * smr_aln_slots() entries, read r's at r * smr_aln_slots() (above).
 * SMR_ALNS_PACKED: read r's results[r].n_align alignments are contiguous, in read order, from sum_{j<r} results[j].n_align; the
 *   counts define the layout, so no offset array crosses the ABI.  Any num_alignments: with N > 0 it drops the empty slots, with
 *   N == 0 a read may store any number of alignments.  A run still stores at most smr_aln_slots() alignments per read; a read that
 *   accepts more finishes its search, counts them, and the download runs it again, with the other such reads, in batches of its
 *   own whose arenas are sized by those counts (at most 2^24 slots per batch, environment variable SMR_RETRY_SLOTS read at
 *   smr_init; a larger read runs alone).  Results do not depend on it.  SMR_CNT_NUM_ALIGNED and reads_matched_per_db count each
 *   read once; SW_CALLS and the other work counters count every run.
 *   In this layout smr_align_batch, smr_download_results and smr_set_stats_buffer are SMR_ERR_ARG (use the _packed calls), and the
 *   report-side calls (smr_format_reports[_gz], smr_format_blast_pairwise[_gz], smr_otu_add, smr_denovo_stats) read their alns
 *   and stats packed. */
enum { SMR_ALNS_STRIDED = 0, SMR_ALNS_PACKED = 1 };
int smr_set_aln_layout(smr_ctx*, uint32_t layout);
/* smr_align_batch in the packed layout.  alns[aln_cap]; stats (nullable) [aln_cap], indexed like alns (the device always computes
 * them in this layout: the pointer decides whether they are copied).  *aln_used = the alignments stored, *cigar_used = the CIGAR
 * words; if either array is too small the call fails with SMR_ERR_CAPACITY and both are exact.  The batch is then resident and
 * run: smr_download_results_packed with arrays that large writes the bytes the call would have written, without running it again.
 * The CIGARs follow read order in cigar_pool. */
int smr_align_batch_packed(smr_ctx*, const uint8_t* seq_cat, const uint64_t* seq_off, uint32_t nreads, smr_read_result* results,
                           smr_aln* alns, uint64_t aln_cap, uint64_t* aln_used, smr_aln_stats* stats, uint32_t* cigar_pool,
                           uint64_t cigar_cap, uint64_t* cigar_used, uint64_t* counters, uint32_t n_counters);
/* smr_download_results in the packed layout, with the arguments of smr_align_batch_packed.  The batch must have been run
 * (smr_run_resident) in this layout at the current stride; it never changes the resident batch, and may be called again.  The
 * first download after a run runs the reads that outgrew the stride and places every read on the device (smr_place_results_packed);
 * the library keeps that placement (device memory of the size of the returned arrays) until the batch is run again or replaced,
 * so a later download copies it. */
int smr_download_results_packed(smr_ctx*, smr_read_result* results, smr_aln* alns, uint64_t aln_cap, uint64_t* aln_used,
                                smr_aln_stats* stats, uint32_t* cigar_pool, uint64_t cigar_cap, uint64_t* cigar_used,
                                uint64_t* counters, uint32_t n_counters);

/* Instrumentation (default OFF; the environment variable SMR_INSTR=1 turns it on at smr_init).  With it, the seed kernel counts
 * SMR_CNT_WINDOWS / BUCKETS / BUCKET_ENTRIES and the candidate kernel accounts its phases with the cycle counter (the SMR_CNT_*
 * entries from DBG_MAX_READ_CYCLES on): separate instantiations of both kernels, 2-3 % slower.  Everything a caller of the
 * reference would see -- results, Readstats counters, SW_CALLS / SW_CELLS / POS_ENTRIES / LIS_CALLS -- is identical either way. */
int smr_set_instrumentation(smr_ctx*, int on);

/* Optional: where the next smr_align_batch / smr_download_results stores smr_aln_stats for every stored alignment (same
 * indexing as alns[]; nullptr = do not compute).  Host buffer of nreads * max(1,num_alignments) entries.  A non-null buffer is
 * SMR_ERR_ARG in the packed layout, whose calls take the stats array as an argument (smr_set_aln_layout). */
int smr_set_stats_buffer(smr_ctx*, smr_aln_stats* stats);

/* Input decode on the device (SURVEY 8(f)(2)): `text` = the bytes of an uncompressed FASTA or FASTQ file (or a record-aligned
 * piece of one).  Replaces, for the reads of this batch, the record split of Readfeed (src/sortmerna/readfeed.cpp:683-770),
 * Read::Read(readstr) (read.cpp:141-176) and the nt_table encoding of Read::init (read.cpp:264-288, common.hpp:68-77):
 * the text is copied to the device once and newline indexing, record split and 0-4 encoding run there; the decoded batch
 * becomes the resident batch (as after smr_upload_batch): follow with smr_run_resident / smr_download_results.
 * FASTQ: 4 lines per record; FASTA: '>' header + any number of sequence lines; CR LF tolerated; a missing final newline is
 * fine; trailing blank lines are ignored.  *nreads = records found. */
int smr_upload_fastx(smr_ctx*, const char* text, uint64_t nbytes, uint32_t* nreads);

/* The same from a gzip file: `gz` = the bytes of a .fastq.gz / .fasta.gz (one or several gzip members, RFC 1952).  Replaces the
 * inflate of the reference's read feed (Readfeed::next_gz, src/sortmerna/readfeed.cpp:683-770, izlib.cpp / rapidgzip): the
 * compressed bytes are copied to the device and inflated there -- block starts found speculatively in every 64 KB of the file, one
 * decoder thread per span, back-references into not-yet-known history resolved in a second step (sortmerna_b200/csrc/smr_inflate.h)
 * -- then decoded as in smr_upload_fastx.  The CRC-32 and ISIZE of every member are checked on the inflated bytes; a corrupt or
 * truncated file fails with SMR_ERR_ARG. */
int smr_upload_fastx_gz(smr_ctx*, const void* gz, uint64_t nbytes, uint32_t* nreads);
/* The text behind the resident batch (what smr_upload_fastx was given / what smr_upload_fastx_gz inflated): *nbytes = its size;
 * copied to `text` when that is not null (cap bytes available).  header_text_off of smr_resident_layout indexes it.  A batch
 * uploaded by smr_upload_batch or smr_align_batch has no text: *nbytes = 0. */
int smr_resident_text(smr_ctx*, char* text, uint64_t cap, uint64_t* nbytes);
/* Test hook: inflate only.  chunk_bytes = distance of the speculative block searches (>= 1024; 0 = the default of smr_upload_fastx_gz); info = {spans decoded,
 * candidates found, device time in us, H2D time in us}. */
int smr_debug_inflate(smr_ctx*, const void* gz, uint64_t nbytes, uint64_t chunk_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_bytes, uint32_t info[4]);

/* -- read stream: a reads file of any size, pushed piece by piece (sortmerna_b200/csrc/smr_stream.cuh) --
 * The caller pushes the file's bytes (compressed bytes with SMR_STREAM_GZ) in pieces of any size, such as 64-512 MB read from disk;
 * the library inflates them on the device as they arrive (one round of smr_upload_fastx_gz's inflate per push, resumed at the last
 * block boundary the pushed bytes reach; the CRC-32 and ISIZE of every member are checked as members complete) and hands back
 * record-aligned batches: each one is made resident as by smr_upload_fastx, so smr_run_resident, smr_download_results,
 * smr_resident_text and smr_format_reports[_gz] / smr_otu_add with text == nullptr work on it unchanged.  A batch holds the whole
 * records that fit in batch_bytes of text (FASTQ: 4 lines each; FASTA: a header line and the lines up to the next one), or one
 * record alone when that record is longer; the batches of a file, one after another, decode to exactly the reads of the whole file.
 * The stream's buffers (compressed bytes not yet inflated, text not yet in a batch) belong to the stream; opening a new stream
 * drops them.  A corrupt, truncated or non-gzip SMR_STREAM_GZ input (bad data, CRC-32 or ISIZE, EOF inside a header, block or
 * trailer) fails with SMR_ERR_ARG, at the push that shows it, and closes the stream; text that is neither FASTA nor FASTQ fails in
 * smr_stream_next with the refusals of smr_upload_fastx.
 *
 * Separately, every pushed byte of text is counted as the reference's Readfeed::count_reads_parallel counts a reads file
 * (src/sortmerna/readfeed.cpp:1486-1663; rule in sortmerna_b200/csrc/smr_stream.h): a fixed cycle of 4 lines (first byte '@') or 2
 * lines per record, every byte of a cycle-position-1 line before its '\n' counted ('\r' included), a last sequence line without
 * '\n' not counted, multi-line FASTA taken as 2-line records.  For a flat multi-line FASTA the reference's figures depend on its
 * -threads (each split restarts the cycle at a '>' line); these are the single-split figures, which -threads 1 and gzip input give.
 * They are what Refstats::minimal_score and the E-value read length are computed from.  SMR_STREAM_COUNT_ONLY counts and keeps no
 * text: the cheap first pass over a file. */
enum { SMR_STREAM_GZ = 1, SMR_STREAM_COUNT_ONLY = 2, SMR_STREAM_NEXT_FILE = 4, SMR_STREAM_MATES = 8 };
/* open (or reset) the context's read stream; batch_bytes = text bytes per batch, in [1, 0xF0000000) (ignored with COUNT_ONLY).  Every
 * batch but the file's last holds the whole records that fit in batch_bytes; before the end of the file, pending text that fits in
 * one batch waits for the next push.  SMR_STREAM_NEXT_FILE: the counts go on from the previous stream's, as the reference counts
 * the -reads files of one run (mates): totals add up, the line cycle of the first file holds, a gzip file updates the minimum read
 * by read and a flat file's own minimum is merged at its end (readfeed.cpp:1497-1662). */
int smr_stream_begin(smr_ctx*, uint32_t flags, uint64_t batch_bytes);
/* the next n bytes of the file; eof = 1 with the last piece (n may be 0).  SMR_ERR_ARG on a mate stream. */
int smr_stream_push(smr_ctx*, const void* bytes, uint64_t n, int eof);
/* SMR_STREAM_MATES: a stream of two mate files (-reads R1 -reads R2), records k of both files paired (sortmerna_b200/csrc/smr_stream.cuh,
 * DESIGN.md 5c).  Each mate is pushed on its own, mate = 1 or 2, in pieces of any size; SMR_STREAM_GZ applies to both, and each is
 * inflated and indexed as a single stream's file.  smr_stream_next makes a batch of k pairs resident: record k of mate 1 and then
 * record k of mate 2, as one interleaved text (records 2k and 2k+1), a last line without '
' given one.  k is the largest number
 * of pairs both files hold whose interleaved text fits in batch_bytes, or 1 when the first pair alone is longer; before both files
 * have ended, pairs that fit wait for more pushes.  The batch is then used as any resident batch; smr_format_reports[_gz] with text
 * == nullptr treats it as mates (smr_report_opts.mates).  SMR_ERR_ARG, closing the stream, for: one mate FASTQ and the other FASTA;
 * files that differ in record count (at the smr_stream_next that finds one file ended while the other holds a record); a corrupt
 * gzip input of either mate (the message names the mate); smr_stream_push_mate on a stream without SMR_STREAM_MATES.  A mate
 * stream counts nothing (smr_stream_counts stays 0): count the mate files one after another with SMR_STREAM_NEXT_FILE.  MATES with
 * COUNT_ONLY or NEXT_FILE is SMR_ERR_ARG. */
int smr_stream_push_mate(smr_ctx*, uint32_t mate, const void* bytes, uint64_t n, int eof);
/* make the next batch resident: *nreads > 0 = a batch is resident (as after smr_upload_fastx); *nreads == 0 and *done == 0 = push
 * more; *done == 1 = the file is exhausted */
int smr_stream_next(smr_ctx*, uint32_t* nreads, int* done);
/* count_reads_parallel over everything pushed so far: {num_reads_tot, length_all, min_read_len, max_read_len} */
int smr_stream_counts(smr_ctx*, uint64_t out[4]);

/* Where the resident reads are: header_text_off[r] = offset of record r's header line in the text given to
 * smr_upload_fastx (for Read::getSeqId / report writers; nullptr = skip; only after smr_upload_fastx), read_off[0..nreads] =
 * offsets into the concatenated 0-4 codes, seq04 (optional) = those codes (seq_cap bytes available). */
int smr_resident_layout(smr_ctx*, uint64_t* header_text_off, uint64_t* read_off, uint8_t* seq04, uint64_t seq_cap);

/* Same work with the batch already resident: upload once, run many times (bench `value` leg).
 * smr_download_results takes the arguments of smr_align_batch and behaves the same way: reads that overflowed their scratch are run
 * again in a batch of their own, and a cigar pool too small gives SMR_ERR_CAPACITY with *cigar_used = the words needed (download
 * again into a larger pool).  It never changes the resident batch or the device results of its run: it may be called any number
 * of times after one smr_run_resident, and a download that needs retries runs them again each time.  smr_upload_batch leaves no
 * text behind the resident batch (smr_resident_text: 0 bytes; smr_format_reports needs the text passed in). */
int smr_upload_batch(smr_ctx*, const uint8_t* seq_cat, const uint64_t* seq_off, uint32_t nreads);
int smr_run_resident(smr_ctx*);                       /* all kernels of one pass over the resident batch */
int smr_download_results(smr_ctx*, smr_read_result* results, smr_aln* alns, uint32_t* cigar_pool,
                         uint64_t cigar_cap, uint64_t* cigar_used, uint64_t* counters, uint32_t n_counters);

/* -- report writer on the device (sortmerna_b200/csrc/smr_report.cuh, DESIGN.md 5e): one batch's results + the FASTA / FASTQ text
 *    of its reads -> the bytes the reference's report stage writes for that batch: aligned.sam body rows (ReportSam::append,
 *    src/sortmerna/report_sam.cpp:64-152), tabular aligned.blast rows (ReportBlast::append, report_blast.cpp:99-346), and the records
 *    of aligned.*, other.* and aligned_denovo.* (ReportFastx / ReportFxOther / ReportDenovo, routing of output.cpp:117-142); and in a
 *    call of its own, the pairwise aligned.blast rows of -blast 0 (report_blast.cpp:136-251). */

/* The reference ids (BaseRecord::getId) of the loaded (index_num, part), concatenated: id k = names_cat[name_off[k] .. name_off[k+1]).
 * Uploaded once; they stay resident with the part.  Needed for SAM and BLAST. */
int smr_set_report_refs(smr_ctx*, uint32_t index_num, uint32_t part, const char* names_cat, const uint64_t* name_off, uint32_t nref);
/* The E-value inputs of index index_num (Refstats: gumbel lambda / K, the corrected full_ref / full_read of refstats.cpp:236-257).
 * The host computes the E-value and bit score of every score 0..65535 with the reference's expressions (report_blast.cpp:117-126)
 * and uploads the tables; the device only looks them up.  Needed for BLAST. */
int smr_set_report_scoring(smr_ctx*, uint32_t index_num, double lambda, double K, uint64_t full_ref, uint64_t full_read);

enum { SMR_BLAST_COL_CIGAR = 1, SMR_BLAST_COL_QCOV = 2, SMR_BLAST_COL_QSTRAND = 3 };
typedef struct {
  int32_t sam;                 /* -sam */
  int32_t blast;               /* -blast given */
  int32_t blast_format;        /* its first field: 1 = tabular; 0 = pairwise (smr_format_blast_pairwise; SMR_ERR_UNSUPPORTED in
                                  smr_format_reports) */
  int32_t blast_cols[4];       /* the optional columns in the order given (SMR_BLAST_COL_*), 0 ends the list */
  int32_t fastx, other;        /* -fastx, -other */
  int32_t denovo;              /* -de_novo_otu: aligned_denovo.* */
  double min_id, min_cov;      /* -id, -coverage (the aligned_denovo rule) */
  int32_t paired_in, paired_out; /* the batch is interleaved mates: records 2k and 2k+1 */
  int32_t out2, sout;          /* -out2, -sout: aligned / other / aligned_denovo each split into 2 files (4 with both), for a paired
                                  batch only (SMR_ERR_UNSUPPORTED otherwise); -sout with paired_in / paired_out is SMR_ERR_ARG */
  int32_t mates;               /* records 2k and 2k+1 are mates from two files (-reads R1 -reads R2): paired, as the reference
                                  makes every two-file run (options.cpp:1590-1592); forced on for the resident batch of a mate stream */
} smr_report_opts;

/* Format one batch.  text / nbytes: the FASTA or FASTQ text of the reads, in batch order; text == nullptr means the resident text of
 * smr_upload_fastx[_gz].  results / alns / cigar_pool (cigar_words used words) / stats: exactly what smr_align_batch or
 * smr_download_results returned for it (stats through smr_set_stats_buffer; required for SAM, BLAST and denovo).  SEQ is taken
 * from the text.  The number of records and every aligned read's length must agree with the results (SMR_ERR_ARG otherwise).
 * Output: the streams one after another, in this order: SAM rows of every loaded (index, part) group in (index, part) order, BLAST
 * rows of every group, aligned reads, other reads, aligned_denovo reads; stream k = out[stream_off[k] .. stream_off[k+1]),
 * stream_off has 2 * groups + 3 * num_out + 1 entries.  num_out = 1, or 2 with -out2 (_fwd, _rev) or -sout (_paired, _singleton),
 * or 4 with both (_paired_fwd, _paired_rev, _singleton_fwd, _singleton_rev): each of the three read files is num_out streams in
 * that order (report_fx_base.cpp:73-90), routed as ReportFastx / ReportFxOther / ReportDenovo::append at -threads 1.  A caller that feeds a file in several batches appends every stream to its own file and
 * concatenates them at the end, as the reference's merge does.  If out is null or cap is below the last entry of stream_off, the call
 * returns SMR_ERR_CAPACITY with stream_off filled. */
int smr_format_reports(smr_ctx*, const smr_report_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                       const smr_aln* alns, const uint32_t* cigar_pool, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                       char* out, uint64_t cap, uint64_t* stream_off);
/* The same streams, each non-empty one compressed on the device to one gzip member (RFC 1952) before the D2H: the reference's
 * -zip-out output (its report writers go through zlib's gzip wrapper, izlib.cpp).  An empty stream stays 0 bytes.  Arguments and
 * stream_off as for smr_format_reports, with the sizes of the members: if out is null or cap is below the last entry of stream_off, the
 * call returns SMR_ERR_CAPACITY with the exact compressed sizes in stream_off, and a retry gives the same bytes.  The members are not
 * zlib's bytes (sortmerna_b200/csrc/smr_deflate.h) but the same input always gives the same bytes. */
int smr_format_reports_gz(smr_ctx*, const smr_report_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                          const smr_aln* alns, const uint32_t* cigar_pool, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                          char* out, uint64_t cap, uint64_t* stream_off);
/* The pairwise BLAST rows of -blast 0 (BlastFormat::REGULAR, report_blast.cpp:136-251) of one batch: per stored alignment, in the row
 * order of tabular BLAST, "Sequence ID: ", "Query ID: ", "Score: <score1> bits (<bit score>)\tExpect: <E-value>\tstrand: <+|->" and a
 * blank line, then the CIGAR's columns in blocks of 60, each as a Target line (reference, '-' for I), a line of '|' (equal), '*'
 * (differ) and ' ' (I, D), and a Query line (the read as SAM's SEQ prints it, '-' for D), with the 1-based first and the last
 * positions of each.  Arguments as for smr_format_reports.  opts must hold blast = 1, blast_format = 0, no BLAST columns, and sam,
 * fastx, other and denovo off (SMR_ERR_ARG otherwise; the reference refuses -blast '0 cigar' as well); of the rest only paired_in,
 * paired_out and mates count, through the skip of empty reads.  stats may be null.  Needs smr_set_report_refs and
 * smr_set_report_scoring for every loaded part, as tabular BLAST does.  Output: one stream per loaded (index, part) group in (index,
 * part) order, stream_off has groups + 1 entries; SMR_ERR_CAPACITY as for smr_format_reports.  A CIGAR that runs past its read or
 * its reference is SMR_ERR_ARG. */
int smr_format_blast_pairwise(smr_ctx*, const smr_report_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                              const smr_aln* alns, const uint32_t* cigar_pool, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                              char* out, uint64_t cap, uint64_t* stream_off);
/* The same streams, each non-empty one as one gzip member, with stream_off and SMR_ERR_CAPACITY as for smr_format_reports_gz. */
int smr_format_blast_pairwise_gz(smr_ctx*, const smr_report_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                                 const smr_aln* alns, const uint32_t* cigar_pool, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                                 char* out, uint64_t cap, uint64_t* stream_off);
/* n host bytes compressed on the device into one gzip member (n == 0: an empty member).  *out_bytes = its size; if out is null or
 * cap is smaller, SMR_ERR_CAPACITY. */
int smr_gzip(smr_ctx*, const void* in, uint64_t n, void* out, uint64_t cap, uint64_t* out_bytes);
/* of the last smr_format_reports[_gz], smr_format_blast_pairwise[_gz], smr_denovo_stats or smr_gzip, milliseconds (CUDA events): out[0] = H2D of the input (text and results), [1] =
 * device work (layout, sizes, scans, writes, compression; includes the read-backs of the sizes), [2] = D2H of the output */
int smr_last_report_timings(const smr_ctx*, double out[3]);

/* -- OTU map on the device (sortmerna_b200/csrc/smr_otu.cuh, DESIGN.md 5e): the reference's otu_map.txt (fill_otu_map /
 *    fill_otu_map2 / OtuMap::write, src/sortmerna/otumap.cpp:84-281) at -threads 1, accumulated over the batches of one read file.
 *    A stored alignment of a read is an entry of the line of its reference id when the read counts as c_yid_ycov > 0 (one of its
 *    alignments passes -id and -coverage with floor(x * 1000 + 0.5) / 1000.0, processor.cpp:334-342) and the alignment itself passes
 *    them with floor(x * 1000 + 0.5) * 0.001 (otumap.cpp:160-163).  %id is taken from n_match_denovo.  Lines: one per reference id in
 *    unsigned byte order of the id, "id\tread\tread...\n"; within a line the (index, part) groups in order, reads in the order added. */
/* Paired reads: the reference's OTU pass reads readfeed slot 0 (otumap.cpp:144), which is every record of one interleaved file but
 * only the first file of two mate files.  In both, a pair (records 2k, 2k+1) whose second record is empty was skipped by the
 * denovo_stats pass, so neither of its mates is an entry. */
enum { SMR_OTU_SINGLE = 0, SMR_OTU_ONE_FILE = 1, SMR_OTU_TWO_FILES = 2 };
typedef struct {
  double min_id, min_cov;         /* -id, -coverage (the reference's default under -otu_map: 0.97, 0.97) */
  int32_t paired_in, paired_out;  /* with feed SMR_OTU_SINGLE, a paired batch: SMR_ERR_UNSUPPORTED (DESIGN.md 5e) */
  int32_t feed;                   /* SMR_OTU_SINGLE: single-end reads; SMR_OTU_ONE_FILE: one interleaved paired file, every record is
                                     looked at; SMR_OTU_TWO_FILES: two mate files (records 2k and 2k+1 of a batch), only records 2k
                                     can be entries -- the only feed that takes a mate stream's batch.  Paired feeds need even batches. */
} smr_otu_opts;
/* Open (or reset) the accumulator of this context.  SMR_ERR_ARG if params.is_best == 0 (the reference refuses -otu_map with
 * -no-best), a loaded part has no smr_set_report_refs or feed is unknown.  Loading a part or setting report ids afterwards makes the
 * next smr_otu_add / smr_otu_finish fail with SMR_ERR_ARG. */
int smr_otu_begin(smr_ctx*, const smr_otu_opts* opts);
/* Add one batch: text / nbytes / results / alns / stats as for smr_format_reports (text == nullptr: the resident text; a mate stream's
 * resident batch needs feed SMR_OTU_TWO_FILES, SMR_ERR_UNSUPPORTED otherwise).  *n_added = entries it added (optional). */
int smr_otu_add(smr_ctx*, const char* text, uint64_t nbytes, const smr_read_result* results, const smr_aln* alns, const smr_aln_stats* stats,
                uint32_t nreads, uint64_t* n_added);
/* The map: counts[0] = bytes, [1] = lines ("Total OTUs"), [2] = entries.  The reference writes no file when counts[2] == 0.  The
 * "passing %id and %coverage" figure of aligned.log is the n_yid_ycov total of smr_denovo_stats, which equals the entries for
 * single-end reads at ordinary thresholds but counts both files of two mate files.  If out is null or cap < counts[0]:
 * SMR_ERR_CAPACITY with counts filled and the accumulator kept; a successful call closes it (smr_otu_begin opens the next). */
int smr_otu_finish(smr_ctx*, char* out, uint64_t cap, uint64_t counts[3]);
/* milliseconds (CUDA events): out[0] = H2D of the smr_otu_add calls since smr_otu_begin, [1] = their device work (includes the one
 * read-back of the sizes per call), [2] = the last smr_otu_finish (sort, sizes, write, D2H) */
int smr_last_otu_timings(const smr_ctx*, double out[3]);

/* -- De novo statistics on the device (sortmerna_b200/csrc/smr_otu.cuh): the reference's denovo_stats pass (denovo_stats_run,
 *    processor.cpp:287-438, run under -otu_map or -de_novo_otu) at -threads 1.  Every stored alignment falls in one class by %id
 *    (from n_match_denovo) and %coverage, both rounded with floor(x * 1000 + 0.5) / 1000.0: c_yid_ycov (both pass), n_yid_ncov (%id
 *    only), n_nid_ycov (%coverage only) or n_denovo (neither). */
typedef struct {
  double min_id, min_cov;   /* -id, -coverage */
  int32_t paired;           /* records 2k and 2k+1 are mates (-paired_in / -paired_out / two mate files): a pair whose second record
                               is empty counts for neither mate (processor.cpp:323-327).  Implied for a mate stream's resident batch.
                               The last record of an odd batch has no mate and counts for nothing, as the reference skips the
                               last record of an odd interleaved file. */
} smr_denovo_opts;
/* One batch: text / nbytes / results / alns / stats / nreads as for smr_otu_add (text == nullptr: the resident text; stats required;
 * the record count and every alignment's readlen are checked against the text, SMR_ERR_ARG otherwise).  per_read (nullable) [nreads *
 * 4] = {c_yid_ycov, n_yid_ncov, n_nid_ycov, n_denovo} of every read, the denovo4 of smr_pack_kvdb_blobs.  totals[4] are ADDED TO
 * (so a run of batches sums itself): Readstats n_yid_ycov, n_yid_ncov, n_nid_ycov, num_denovo of aligned.log.  Timings through
 * smr_last_report_timings. */
int smr_denovo_stats(smr_ctx*, const smr_denovo_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                     const smr_aln* alns, const smr_aln_stats* stats, uint32_t nreads, uint32_t* per_read, uint64_t totals[4]);

/* -- results placed on the device (sortmerna_b200/csrc/smr_place.cuh, DESIGN.md 5g): the last smr_run_resident of the resident
 *    batch turned into the layout of smr_download_results (strided, smr_place_results) or of smr_download_results_packed (packed,
 *    smr_place_results_packed) in device memory, where the report-side _placed calls read it: nothing goes down to the host and
 *    comes back between the alignment and the report writers.  In the packed layout (smr_set_aln_layout) smr_place_results is
 *    SMR_ERR_UNSUPPORTED, and the _placed calls read the packed placement of the resident batch's last run. */
/* Whether every later run computes the smr_aln_stats a placement keeps (default 0).  The _placed calls that read stats (SAM,
 * tabular BLAST, aligned_denovo, the OTU map, the denovo statistics) need a placement of a run made with it on; a run made with a
 * host stats buffer (smr_set_stats_buffer) computes them too.  The scratch-overflow retries of a placement compute the stats when
 * the run being placed did. */
int smr_set_place_stats(smr_ctx*, int on);
/* Place the results of the resident batch's last smr_run_resident on the device: smr_read_result[n], smr_aln[n * smr_aln_slots()]
 * zeroed past n_align, the stats alike, the CIGARs compacted in read order -- the bytes smr_download_results would write, with the
 * same retries of reads that overflowed their scratch (8x, 64x, 512x; each retry batch is placed through its read map before it
 * frees itself; their CIGARs follow those of the others) and the same errors: a read that stores more alignments than the stride
 * gives SMR_ERR_CAPACITY and smr_aln_slots_needed(), a trace back error SMR_ERR_INDEX; an index budget runs the retries as
 * smr_download_results does.  counters[SMR_CNT_FIXED + n_index_files] are ADDED to as by smr_download_results (nullable).
 * *n_alns = the alignment rows (n * stride), *cigar_words = the CIGAR words placed (both nullable, 0 on failure).  The context keeps
 * the placed arrays until the batch is run again or replaced (keyed by the run); a second call for the same run places nothing
 * again and adds the same counters.  SMR_ERR_ARG if the batch was not run, or was run at another stride. */
int smr_place_results(smr_ctx*, uint64_t* counters, uint32_t n_counters, uint64_t* n_alns, uint64_t* cigar_words);
/* The packed layout's placement: the bytes smr_download_results_packed writes -- smr_read_result[n], smr_aln[sum n_align] and
 * the stats alike in read order, the CIGARs compacted in read order, with the same re-runs of reads that stored more alignments
 * than the stride or overflowed their scratch -- placed in device memory.  The first run stays on the device; only the flagged reads'
 * index, flags and n_align come to the host, which forms the re-runs; each re-run's results stay on the device until one count
 * pass, two scans and one scatter place every read from the run that stored it.  counters as smr_download_results_packed adds them
 * (nullable); *n_alns = the alignments placed (sum n_align), *cigar_words = the CIGAR words (both nullable).  A packed download
 * places the same way and keeps its placement here, so either serves the other and the _placed calls; a second call for the same
 * run places nothing and adds the same counters.  A trace back error gives SMR_ERR_INDEX after the results are placed (sizes set),
 * as the packed download does.  SMR_ERR_ARG in the strided layout (use smr_place_results), before a run, or after a run at
 * another stride. */
int smr_place_results_packed(smr_ctx*, uint64_t* counters, uint32_t n_counters, uint64_t* n_alns, uint64_t* cigar_words);
/* The placed arrays copied to the host (a caller that also wants smr_pack_kvdb_blobs): results[n], alns[n * stride] (packed:
 * alns[n_alns] of smr_place_results_packed), stats (nullable; SMR_ERR_ARG if the placed run computed none) and
 * cigar_pool[cigar_cap] (SMR_ERR_CAPACITY below *cigar_words). */
int smr_download_placed(smr_ctx*, smr_read_result* results, smr_aln* alns, smr_aln_stats* stats, uint32_t* cigar_pool, uint64_t cigar_cap);
/* milliseconds (CUDA events) of the last placement's count, scan and scatter passes over the resident batch (retries and packed
 * re-runs excluded) */
int smr_last_place_timing(const smr_ctx*, double* ms);
/* The report-side calls on the placed results of the resident batch's last run and its resident text: smr_format_reports[_gz],
 * smr_format_blast_pairwise[_gz], smr_otu_add and smr_denovo_stats without text, results, alns, cigar_pool or stats; everything else
 * (opts, out, cap, stream_off, SMR_ERR_CAPACITY, n_added, per_read, totals) as there.  SMR_ERR_ARG without a placement of the
 * resident batch's last run (none yet, or one of an earlier run or batch), or when the call reads stats the placement lacks.  In
 * the packed layout they read the packed placement (which always has the stats) and are SMR_ERR_UNSUPPORTED without one of the
 * resident batch's last run; SMR_ERR_INDEX if that placement met a trace back error. */
int smr_format_reports_placed(smr_ctx*, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off);
int smr_format_reports_placed_gz(smr_ctx*, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off);
int smr_format_blast_pairwise_placed(smr_ctx*, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off);
int smr_format_blast_pairwise_placed_gz(smr_ctx*, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off);
/* aligned.bam (SAMv1 4; not a reference output): the SAM rows of smr_format_reports_placed as BAM records, in the same order,
 * compressed on the device into BGZF blocks -- gzip members with the BC subfield, each of at most 65,280 input bytes and compressed
 * with no history before it.  One stream per loaded (index, part) group in (index, part) order, cut into blocks of exactly 65,280
 * bytes and the rest; stream_off has groups + 1 entries.  A record: refID = the references of the groups before plus ref_num (the
 * dictionary of smr_bam_header), pos = SAM POS - 1, mapq 255, flag 0 or 16, next_refID -1, next_pos -1, tlen 0, the bin of the
 * reference span, the CIGAR with its soft clips, SEQ as SAM prints it in 4-bit codes, QUAL as SAM prints it - 33 (0xFF for FASTA),
 * and AS and NM in the smallest of the types C, S, I.  opts must hold sam = 1 and blast, fastx, other and denovo off (SMR_ERR_ARG
 * otherwise); of the rest only paired_in, paired_out and mates count, through the skip of empty reads.  SMR_ERR_ARG, naming the read,
 * for a QNAME longer than 254 bytes, or a FASTQ quality line whose length differs from its sequence's or with a byte outside
 * '!'..'~'.  Placement and stats as for the other _placed calls; stream_off, SMR_ERR_CAPACITY and the retry as for
 * smr_format_reports_gz.  The file is smr_bam_header's blocks, each batch's streams, then the 28-byte BGZF EOF block.  Timings
 * through smr_last_report_timings. */
int smr_format_bam_placed(smr_ctx*, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off);
/* The BAM header of the loaded indexes as BGZF blocks (as smr_format_bam_placed cuts them): magic "BAM\1", l_text and `text` (the
 * SAM header, nbytes bytes, no NUL), n_ref and (l_name, name NUL, l_ref) of every reference of every loaded part in (index, part,
 * ref_num) order, the refIDs of smr_format_bam_placed.  Names from smr_set_report_refs (SMR_ERR_ARG for a part without them),
 * lengths from the resident reference offsets.  *out_bytes = the size; if out is null or cap is smaller, SMR_ERR_CAPACITY. */
int smr_bam_header(smr_ctx*, const char* text, uint64_t nbytes, char* out, uint64_t cap, uint64_t* out_bytes);
/* Coordinate-sorted aligned.bam and aligned.bam.bai (SAMv1 4, 5.2; not a reference output).  The records of smr_format_bam_placed,
 * stably sorted by samtools' coordinate key refID << 32 | (pos + 1) << 1 | reverse strand, so equal keys keep the order of the
 * unsorted file (batch, then the writer's row order).  The file: smr_bam_header's blocks with the text's SO:unsorted made
 * SO:coordinate, the windows' blocks in order, the BGZF EOF block.
 * begin: opens the accumulator (again: the open one is discarded).  SMR_ERR_UNSUPPORTED, naming it, for a reference of 2^29 bases
 *   or more, which BAI cannot address; SMR_ERR_ARG for a part without smr_set_report_refs.
 * add_placed: the placed batch's records (opts and refusals as smr_format_bam_placed) sorted into one run, uncompressed, into out;
 *   *nbytes = its size.  The run's keys and sizes go to the accumulator on the device (12 B per record).  If out is null or cap is
 *   smaller, SMR_ERR_CAPACITY with *nbytes set and the accumulator unchanged; a retry gives the same bytes and appends once.
 * plan: one stable sort of every run's records; windows of whole records of at most window_bytes each (a larger record alone) cut
 *   greedily; *n_windows = their number, and ranges[(w * runs + r) * 2 .. + 1] = [lo, hi), the bytes of run r (from the run's start)
 *   that window w holds (lo = hi = 0 for none).  header_bytes = the size of the header blocks, the compressed offset of the first
 *   window's.  SMR_ERR_CAPACITY if ranges is null or cap (uint64 entries) is below n_windows * runs * 2.
 * window: w = 0, 1, ... in order; staged = window w's ranges of the runs concatenated in run order (nbytes their sum, SMR_ERR_ARG
 *   otherwise, or when a record's block_size disagrees with the runs added).  Its records in sorted order, cut into BGZF blocks of
 *   65,280 bytes and the rest, into out; *out_bytes = their size (SMR_ERR_CAPACITY as smr_bam_header, the window not done).
 * index: after the last window, the BAI bytes into out (*nbytes = the size; SMR_ERR_CAPACITY as above): every reference, bins
 *   ascending with their chunks merged when one starts in the block where the one before ends, the pseudo-bin 37450, the linear index
 *   of 16 kb windows, n_no_coor = 0.  Closes the accumulator.
 * SMR_ERR_ARG without an open accumulator, before plan, out of order, and after an index part was loaded or its report ids set since
 * begin.  add_placed and window set smr_last_report_timings. */
int smr_bam_sort_begin(smr_ctx*);
int smr_bam_sort_add_placed(smr_ctx*, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* nbytes);
int smr_bam_sort_plan(smr_ctx*, uint64_t window_bytes, uint64_t header_bytes, uint64_t* ranges, uint64_t cap, uint64_t* n_windows);
int smr_bam_sort_window(smr_ctx*, uint64_t w, const void* staged, uint64_t nbytes, char* out, uint64_t cap, uint64_t* out_bytes);
int smr_bam_sort_index(smr_ctx*, char* out, uint64_t cap, uint64_t* nbytes);
int smr_otu_add_placed(smr_ctx*, uint64_t* n_added);
int smr_denovo_stats_placed(smr_ctx*, const smr_denovo_opts* opts, uint32_t* per_read, uint64_t totals[4]);

/* Device-side timings of the last smr_run_resident / smr_align_batch, CUDA events on the
 * library's stream, milliseconds: out[0]=total [1]=seed kernels [2]=candidate/SW kernels
 * [3]=finalize (reverse SW + traceback) [4]=h2d [5]=d2h; out[6]=number of kernel launches [7]=decode of the last text upload
 * (smr_upload_fastx[_gz], smr_stream_next).  Index uploads of a budgeted run: smr_index_residency out[6]. */
int smr_last_timings(const smr_ctx*, double out[8]);

/* -- multi-GPU: the only cross-read state is the counter vector (SURVEY 8(e)).  The library
 *    shards nothing itself: each rank calls smr_align_batch on its own reads and the host sums
 *    `counters` with one all-reduce (torch.distributed / NCCL, see INTEGRATION.md). */

/* -- unit-test entry points (run the same device functions the hot path uses) ------------------ */
/* seed search of explicit windows: for window k, sequence seq03 (0..3, length >= win_pos+lnwin) of
 * read read_of[k]; returns ids per window into ids[k*cap .. ), counts[k] (may exceed cap),
 * zero[k] = accept_zero_kmer.  Bit 31 of cap selects the per-lane fallback search instead of the cooperative one. */
int smr_debug_seed_windows(smr_ctx*, uint32_t part_slot, const uint8_t* seq_cat, const uint64_t* seq_off,
                           uint32_t nreads, const uint32_t* win_read, const uint32_t* win_pos, uint32_t nwin,
                           uint32_t* ids, uint32_t cap, uint32_t* counts, uint8_t* zero);
/* measured peak of dependent-free DPX (VIADDMNMX) thread-operations per second on this device, in 1e9/s:
 * the denominator of the Smith-Waterman roofline (SURVEY 8(d)) */
int smr_debug_dpx_peak(smr_ctx*, double* giga_ops_per_s);
/* ssw_align(flag=2) equivalents on explicit (query, target) pairs:
 * out[k*6..] = score1, ref_begin1, ref_end1, read_begin1, read_end1, cigar_len; cigars at k*cigar_cap */
int smr_debug_ssw(smr_ctx*, const uint8_t* q_cat, const uint64_t* q_off, const uint8_t* t_cat,
                  const uint64_t* t_off, uint32_t npairs, uint32_t filters, int32_t* out, uint32_t* cigars,
                  uint32_t cigar_cap);

#ifdef __cplusplus
}
#endif
#endif
