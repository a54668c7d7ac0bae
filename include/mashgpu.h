/*
 * mashgpu.h -- C ABI of the H100-native MinHash engine (libmashgpu.so, sm_90a).
 *
 * This is the drop-in boundary for the three data-parallel hot paths of marbl/Mash.  The reference has
 * no FFI; its seams are the ThreadPool worker functions and the pure-compute functions underneath them
 * (paths below are relative to the reference's src/mash/):
 *
 *   mashgpu_sketch_batch      replaces  sketchFile / sketchSequence      Sketch.cpp:1147-1365 (Sketch.h:229-234)
 *                                       addMinHashes                     Sketch.cpp:512-583   (Sketch.h:226)
 *                                       getHash                          hash.cpp:10-38       (hash.h:21)
 *                                       MinHashHeap::tryInsert/toHashList MinHashHeap.cpp:68-146, HashSet.cpp:78-118
 *   mashgpu_dist_*            replaces  compare / compareSketches / pValue CommandDistance.cpp:306-448 (CommandDistance.h:91-93)
 *   mashgpu_screen_*          replaces  hashSequence + the shared/median/identity/p-value reduce
 *                                       CommandScreen.cpp:93-114, 484-599, 288-355, 409-455, 463-482, 601-615
 *
 * Conventions: plain pointers and sizes only; the caller owns every buffer; every function returns an int
 * status (0 = MASHGPU_OK), never throws and never calls exit() (the reference prints to cerr and exit(1)s,
 * Sketch.cpp:1294-1312 -- the host shim maps statuses back to those messages); a context is bound to one
 * CUDA device and must not be used from two threads at once.  Hashes are always carried as uint64_t, 32-bit
 * hashes (use64 == 0) zero-extended, exactly as HashList stores hash_u (HashList.h:13-37, hash.h:15-19).
 * Unlike addMinHashes (Sketch.cpp:524-530) the sequence buffers are NOT modified.
 *
 * There is no CPU fallback: without a CUDA device mashgpu_create fails.
 */
#ifndef MASHGPU_H
#define MASHGPU_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

#define MASHGPU_OK 0
#define MASHGPU_ERR_INVALID 1      /* bad argument */
#define MASHGPU_ERR_CUDA 2         /* CUDA runtime error (message in mashgpu_last_error) */
#define MASHGPU_ERR_UNSUPPORTED 3  /* parameter combination outside the GPU path (see mashgpu_sketch_params) */
#define MASHGPU_ERR_NOMEM 4

typedef struct mashgpu_ctx mashgpu_ctx;

/* Sketch::Parameters (Sketch.h:34-109), the fields the hot path reads. */
typedef struct mashgpu_sketch_params {
    int32_t kmer_size;        /* kmerSize, 1..32 (Command.cpp:168) */
    uint32_t sketch_size;     /* minHashesPerWindow (s) */
    uint32_t seed;            /* hash seed (default 42) */
    int32_t use64;            /* alphabetSize^k > 2^32 (Sketch.cpp:1136); filled by mashgpu_set_alphabet */
    int32_t noncanonical;
    int32_t preserve_case;
    uint8_t alphabet[256];    /* Parameters::alphabet; filled by mashgpu_set_alphabet */
    uint32_t min_copies;      /* `-m`: MinHashHeap multiplicityMinimum (Sketch.cpp:1186, reads mode; MinHashHeap.cpp:96-118): a hash enters
                                 the sketch at its m-th occurrence.  0 or 1 = off.  The sketch is then the s smallest hashes seen at
                                 least m times, and the multiplicities follow the heap exactly (tests/test_gpu_sketch.py). */
    double target_cov;        /* `-c`: stop after the first read that brings the heap's average multiplicity to this value
                                 (Sketch.cpp:1258-1262).  Only the reads paths look at it; <= 0 = off. */
    uint64_t bloom_bytes;     /* `-b`: MinHashHeap memoryBoundBytes (Sketch.cpp:1186, MinHashHeap.cpp:19-41, 78-95): a hash enters the
                                 sketch with count 2 when a Bloom filter of bloom_bytes bytes already holds it, else it is added to the
                                 filter.  The filter is the reference's exactly: one hash function, 8 * bloom_bytes bits of which the
                                 32-bit index reaches the first 2^32, so min(bloom_bytes, 2^29) bytes of device memory.  0 = off.  Only
                                 the reads paths take it (every other entry point returns MASHGPU_ERR_UNSUPPORTED); together with
                                 min_copies > 1 it is MASHGPU_ERR_INVALID, as the reference CLI refuses -b with -m. */
} mashgpu_sketch_params;
/* GPU path coverage: alphabet == {A,C,G,T} (canonical or not, any k 1..32, either case mode) runs the 4-bit
 * packed DNA kernels; any other alphabet requires noncanonical != 0 (the protein setting of the reference,
 * sketchParameterSetup.cpp) and runs the byte-alphabet kernels.  Other combinations return
 * MASHGPU_ERR_UNSUPPORTED (never a CPU fallback). */

/* setAlphabetFromString (Sketch.cpp:1108-1137): fills alphabet[] and use64 from kmer_size/preserve_case.
 * Returns the alphabet size. */
uint32_t mashgpu_set_alphabet(mashgpu_sketch_params *p, const char *characters);

int mashgpu_device_count(void);
int mashgpu_create(int device, mashgpu_ctx **ctx);
void mashgpu_destroy(mashgpu_ctx *ctx);
/* Message of the last failure on this context (ctx == NULL: of the last failed mashgpu_create). */
const char *mashgpu_last_error(const mashgpu_ctx *ctx);

/* ---------------------------------------------------------------------------------------------------------
 * Hot path 1: sketching.
 *
 * n_records pre-parsed records (what kseq_read delivers: sequence bytes, kseq.h:170-208) are grouped into
 * n_units sketch units: unit_of_record[r] (non-decreasing; NULL = record r is unit r).  A unit is one
 * sketchFile job (all records of the listed files, k-mers never span records) or one sketchSequence job.
 * Records shorter than kmer_size are skipped and not counted in the length (Sketch.cpp:1222-1226,1251-1254).
 *
 * Outputs, per unit u, in input order (ThreadPool ordering contract, ThreadPool.hxx:87-118):
 *   out_hashes[u*sketch_size .. +out_n[u])  the min(s, #distinct) smallest distinct hashes, ascending
 *   out_counts (nullable)                    multiplicity of each hash (HashSet counts)
 *   out_n[u]                                 number of hashes
 *   out_length[u]                            sum of the kept records' lengths (Reference::length, non -r mode)
 * ------------------------------------------------------------------------------------------------------- */
int mashgpu_sketch_batch(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                         uint64_t n_records, const char *const *seq, const uint64_t *len,
                         const uint32_t *unit_of_record, uint64_t n_units,
                         uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_length);

/* One sketch of a read set, `mash sketch -r [-m min_copies] [-c target_cov] [-b bloom_bytes]` (sketchFile with parameters.reads,
 * Sketch.cpp:1186-1282): all records in the order given (the caller interleaves several files round robin as Sketch.cpp:1202-1270
 * does).  With target_cov > 0 the result is the heap as it stood after the first kept record that brought estimateMultiplicity()
 * to the target (Sketch.cpp:1258-1262) and *out_records_used (the "Reads used" line, :1324-1327) is the number of kept records up
 * to and including it; otherwise all kept records are used.  With target_cov > 0 or bloom_bytes, or with min_copies > 1 when the set
 * does not fit in half of the free device memory, this is mashgpu_reads_open + one mashgpu_reads_feed + mashgpu_reads_finish +
 * mashgpu_reads_close; otherwise the result does not depend on the order of the reads and the whole set is sketched in one parallel
 * pass (same result, faster: DESIGN.md 2.6), or, beyond that memory limit, streamed through a unit job (mashgpu_unit_*).
 * out_counts nullable.  DNA alphabet only. */
int mashgpu_sketch_reads(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                         uint64_t n_records, const char *const *seq, const uint64_t *len,
                         uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_records_used);

/* The same as a streaming job, for read sets of any size: records are fed in order, in any number of feeds, and the result does not
 * depend on how they are split.  Each staged buffer is scanned stretch by stretch with the heap's current top as threshold (a top
 * never rises once the heap is full, so it bounds every k-mer after it that can change the heap); those k-mers are sorted by
 * position and replayed through the reference's heap logic (MinHashHeap::tryInsert, the Bloom branch included) by one warp whose
 * state stays in device memory (DESIGN.md 2.6).  Device memory is fixed at open by the parameters -- staging
 * (MASHGPU_READS_STAGE_BYTES, default 128 MiB), events (MASHGPU_READS_EVENT_CAP, default 2^21), O(s + pending hashes) replay
 * tables and min(bloom_bytes, 2^29) bytes of filter -- never by the size of the read set.  DNA alphabet only. */
typedef struct mashgpu_reads_job mashgpu_reads_job;
int mashgpu_reads_open(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, mashgpu_reads_job **job);
/* The next n_records records, as mashgpu_sketch_reads takes them.  Records shorter than kmer_size are skipped; a record longer than
 * the staging buffer is split with a (kmer_size-1)-base overlap and each of its windows is counted once.  Returns once the
 * caller's buffers are free; *stopped (nullable) = 1 once the target coverage was reached, after which feeds are accepted and
 * ignored. */
int mashgpu_reads_feed(mashgpu_reads_job *job, uint64_t n_records, const char *const *seq, const uint64_t *len, int *stopped);
/* The sketch (sketch_size slots, ascending) and the kept records used, as mashgpu_sketch_reads returns them.  out_counts nullable. */
int mashgpu_reads_finish(mashgpu_reads_job *job, uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_records_used);
int mashgpu_reads_close(mashgpu_reads_job *job);

/* One sketch unit of any size as a streaming job: exactly one unit of mashgpu_sketch_batch (one sketchFile job with minCov 1 and no
 * Bloom filter, Sketch.cpp:1147-1336), with records fed in order, in any number of feeds; the result does not depend on how they are
 * split.  Every configuration mashgpu_sketch_batch takes (DNA and byte alphabets, k 1..32, any sketch size, either case mode,
 * canonical or not) except min_copies > 1, target_cov > 0 and bloom_bytes, which return MASHGPU_ERR_UNSUPPORTED (they need the
 * order of the records: mashgpu_reads_*).  The stream is sketched stage by stage -- with the running s-th smallest hash as the
 * threshold once s hashes are held -- and each stage's bottom-s merged into the running one, counts summed, the reference's
 * top-of-heap count included (DESIGN.md 2.7).  Device memory is fixed at open by the parameters: two staging buffers
 * (MASHGPU_UNIT_STAGE_BYTES each, default 128 MiB; the copy of one overlaps the scan of the other), a candidate table sized from s
 * and the stage, and O(s) state.  mashgpu_sketch_batch routes a unit whose stream exceeds half of the free device memory here,
 * and mashgpu_sketch_reads a read set without -m > 1, -c or -b beyond that limit. */
typedef struct mashgpu_unit_job mashgpu_unit_job;
int mashgpu_unit_open(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, mashgpu_unit_job **job);
/* The next n_records records of the unit.  Records shorter than kmer_size are skipped and not counted; a record longer than a stage
 * is split with a (kmer_size-1)-base overlap and each of its windows is counted once.  Returns once the caller's buffers are free.
 * MASHGPU_ERR_INVALID after mashgpu_unit_finish. */
int mashgpu_unit_feed(mashgpu_unit_job *job, uint64_t n_records, const char *const *seq, const uint64_t *len);
/* The unit's sketch (out_hashes: sketch_size slots, ascending; out_counts nullable: the HashSet counts), *out_length = sum of the kept
 * records' lengths, *out_records = their number.  May be called again; no feed is accepted after it. */
int mashgpu_unit_finish(mashgpu_unit_job *job, uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_length,
                        uint64_t *out_records);
int mashgpu_unit_close(mashgpu_unit_job *job);

/* Same computation on a sequence stream already resident in device memory.  d_stream holds the units back to
 * back; unit u occupies bytes [unit_start[u], unit_start[u+1]) (host array of n_units+1 offsets); records inside
 * a unit are separated by at least one byte outside the alphabet (e.g. 0).  d_stream must be readable up to
 * unit_start[n_units] rounded up to 16 bytes.  d_out_* are device pointers (d_out_counts nullable).
 * `stream` is a cudaStream_t (NULL = the context's stream).  All work is enqueued on that stream; the call synchronises
 * it once at the end (it has to read the per-unit status flags to decide whether a unit needs the exact re-run). */
int mashgpu_sketch_stream_dev(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                              const void *d_stream, const uint64_t *unit_start, uint64_t n_units,
                              uint64_t *d_out_hashes, uint32_t *d_out_counts, uint32_t *d_out_n, void *stream);

/* Host feed path, exposed for tests (no GPU involved): packs records the way mashgpu_sketch_batch does before the
 * H2D copy -- every record followed by one separator position -- into 2-bit codes (A0 C1 G2 T3, 32 positions per
 * uint64 word) plus the list of runs of positions that are not in the alphabet (upper-casing unless preserve_case;
 * separators included).  codes must hold ceil(stream_len/32) words with stream_len = sum(len[r] + 1); runs receives
 * up to runs_capacity {start, length} pairs; *n_runs is the number of runs found. */
int mashgpu_host_pack(const mashgpu_sketch_params *params, uint64_t n_records, const char *const *seq, const uint64_t *len,
                      int threads, uint64_t *codes, uint64_t *runs, uint64_t runs_capacity, uint64_t *n_runs);

/* Sketching from a stream the caller already keeps 2-bit packed (the format mashgpu_host_pack writes): a collection cached in
 * this form crosses PCIe at a quarter of a byte per base and no host thread touches the bases again, so the call runs at the
 * rate of the scan kernel instead of the rate of PCIe-ASCII.  codes: ceil(stream_len / 32) words, base p at bits 2 (p % 32) of
 * codes[p / 32] (A0 C1 G2 T3); runs: n_runs {start, length} pairs, ascending and disjoint, covering every position that is not
 * a base of the alphabet (the separator after each record included); unit u = positions [unit_start[u], unit_start[u+1])
 * (n_units + 1 ascending offsets, unit_start[n_units] <= stream_len).  Same outputs as mashgpu_sketch_batch (without
 * out_length: record lengths are the caller's).  Pinned host buffers make the copies asynchronous.  DNA alphabet only. */
int mashgpu_sketch_batch_packed(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                                const uint64_t *codes, uint64_t stream_len, const uint64_t *runs, uint64_t n_runs,
                                const uint64_t *unit_start, uint64_t n_units,
                                uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n);

/* getHash over every window (hash.cpp:10-38 applied as in Sketch.cpp:540-576): out_hash[i]/out_valid[i] for each
 * window start i in [0, len-k]; invalid windows (a byte outside the alphabet) have out_valid[i] == 0.
 * Host buffers.  Diagnostic/test entry point of the scan+hash kernel. */
int mashgpu_hash_windows(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                         const char *seq, uint64_t len, uint64_t *out_hash, uint8_t *out_valid);

/* Six-frame translation of one chunk, as the translated screen runs it: d_out receives the peptides of forward frames 0, 1, 2
 * and then of reverse-complement frames 0, 1, 2, frame f holding (len - f) / 3 amino acids followed by one 0 byte, a stop or a
 * codon with a byte outside {A,C,G,T} written as 0 -- 6 + 2 * sum_f (len - f) / 3 bytes in all.  Device buffers: d_seq must be
 * readable up to len rounded up to 16 when it is 16-byte aligned (the kernel then loads whole vectors).  Runs on the context's
 * stream and returns once the output is written.  Diagnostic/test entry point of the translation kernel. */
int mashgpu_translate6(mashgpu_ctx *ctx, const void *d_seq, uint64_t len, int preserve_case, uint8_t *d_out);

/* ---------------------------------------------------------------------------------------------------------
 * Hot path 2: all-pairs sketch comparison.
 * ------------------------------------------------------------------------------------------------------- */
/* A Sketch's reference list (Sketch.h:131-139): n rows of `stride` uint64 slots; row i holds n_hashes[i]
 * ascending distinct hashes (Reference::hashesSorted) and has sequence length length[i] (Reference::length).
 * on_device != 0: hashes/n_hashes/length are device pointers. */
typedef struct mashgpu_sketch_set {
    uint64_t n;
    uint64_t stride;
    const uint64_t *hashes;
    const uint32_t *n_hashes;
    const uint64_t *length;
    int32_t on_device;
} mashgpu_sketch_set;

/* Arguments of compareSketches (CommandDistance.h:92). */
typedef struct mashgpu_dist_params {
    uint64_t sketch_size;   /* min(s_query, s_ref)  (CommandDistance.cpp:313-315) */
    int32_t kmer_size;
    double kmer_space;      /* alphabetSize^k as double (Sketch.cpp:509) */
    double max_distance;    /* -d, < 0 disables (CommandDistance.cpp:409) */
    double max_pvalue;      /* -v, < 0 disables (CommandDistance.cpp:419) */
} mashgpu_dist_params;

typedef struct mashgpu_dist_job mashgpu_dist_job;

/* Uploads both sets (qry == NULL or qry == ref: all-vs-all of one set), builds the order-preserving 32-bit
 * dictionary of all hashes and keeps everything resident. */
int mashgpu_dist_open(mashgpu_ctx *ctx, const mashgpu_sketch_set *ref, const mashgpu_sketch_set *qry,
                      const mashgpu_dist_params *params, mashgpu_dist_job **job);

/* Compares queries [q_begin, q_begin+q_count) with every reference: pair (q, r) is written at index
 * (q - q_begin) * n_ref + r, the reference's query-major order (CommandDistance.cpp:213-232, 306-334).
 * Per pair (PairOutput, CommandDistance.h:63-70): numer (shared hashes), denom, distance, pvalue, pass.
 * Sketch sizes up to 1034 run the tiled lockstep merge (32 references per shared-memory tile); larger ones (`-s 10000`) a
 * warp-per-pair merge; beyond ~28 000 hashes per sketch one thread per pair from global memory.
 * Where the reference leaves numer/denom/distance/pValue unset (distance > max_distance, :409-412) this
 * engine still writes the computed numer/denom/distance and pvalue = 0, with pass = 0.
 * Any output pointer may be NULL.  Host buffers. */
int mashgpu_dist_run(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count,
                     uint32_t *numer, uint32_t *denom, double *distance, double *pvalue, uint8_t *pass);
/* Same with device output buffers, enqueued on `stream` (cudaStream_t, NULL = context stream).  A job holds one set of
 * scratch buffers (work lists, deferred p-value queue, pass list): at most ONE run of a job may be in flight -- enqueue the
 * runs of a job on a single stream, or synchronise between runs on different streams. */
int mashgpu_dist_run_dev(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count,
                         uint32_t *d_numer, uint32_t *d_denom, double *d_distance, double *d_pvalue, uint8_t *d_pass,
                         void *stream);
/* Filtered runs (-d / -v): only the pairs with pass == 1, which is all that writeOutput prints
 * (CommandDistance.cpp:270-287), as a compact list sorted by pair index (q - q_begin) * n_ref + r, i.e. in the
 * reference's output order.  *n_pass = number of passing pairs; if it exceeds `capacity` nothing is returned and the
 * caller retries with a larger capacity (or uses mashgpu_dist_run).  Host buffers of `capacity` entries. */
int mashgpu_dist_run_list(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count, uint64_t capacity,
                          uint64_t *pair_index, uint32_t *numer, uint32_t *denom, double *distance, double *pvalue, uint64_t *n_pass);
int mashgpu_dist_close(mashgpu_dist_job *job);

/* Lower-triangular enumeration for a self comparison (qry == NULL): `mash triangle` compares row i with rows 0..i-1 only
 * (CommandTriangle.cpp:200-214).  on != 0: pairs with r >= q are neither computed nor written and never enter a pass list;
 * whole reference tiles above the diagonal are skipped.  Their output slots are zero with mashgpu_dist_run (host buffers)
 * and keep whatever they held with mashgpu_dist_run_dev (device buffers). */
int mashgpu_dist_set_triangle(mashgpu_dist_job *job, int on);

/* Tile prefilter of the merge (no counterpart in the reference, which merges every pair, CommandDistance.cpp:347-365;
 * the results are identical).  Before a tile of 32 references is merged with a query, the query's hashes are looked up in
 * a filter built over the tile's hashes; a query that shares no hash with any of the 32 references gets the closed form
 * of an empty intersection (common 0, denom min(s, |A|+|B|), distance 1, p-value 1) for all 32 pairs and is not merged.
 * mode: -1 auto (default: on, and switched off for the rest of the job once more than half of the probed
 * (query, tile) combinations turned out to share hashes), 0 off, 1 on.  Environment MASHGPU_DIST_PREFILTER=0|1
 * overrides the default at mashgpu_dist_open. */
int mashgpu_dist_set_prefilter(mashgpu_dist_job *job, int mode);
/* Counters of the prefilter since the job was opened: (query, tile) combinations probed, those that went on to the merge,
 * and whether the next run would probe.  Synchronises the device.  Any pointer may be NULL. */
int mashgpu_dist_prefilter_stats(mashgpu_dist_job *job, uint64_t *combos_probed, uint64_t *combos_flagged, int *active);
/* The prefilter also learns WHICH references of a tile a query may share a hash with (one owner byte per filter slot).  A
 * combination with at most 4 candidate references (MASHGPU_DIST_PAIR_MAX, 0 = off) is not merged as a whole: its candidate
 * pairs go to a list and are merged one warp per pair, the other references of the tile get the closed form.  This keeps the
 * run fast when related sketches are scattered over the collection instead of stored next to each other.
 * *pairs_merged_from_lists: pairs that took this path since the job was opened.  Synchronises the device. */
int mashgpu_dist_pair_stats(mashgpu_dist_job *job, uint64_t *pairs_merged_from_lists);

/* Best hits: the n_best nearest references of every query, selected on the device (no counterpart in the reference, whose
 * users pipe `mash dist` into sort; `mash dist -B`).  A HIT of query q is a reference r whose pair (q, r) has pass == 1 in
 * mashgpu_dist_run (so max_distance, max_pvalue and mashgpu_dist_set_triangle apply unchanged) and numer > 0.  Pairs without a
 * shared hash all sit at distance 1 and p-value 1 and are left out on purpose; so is the pair of two EMPTY sketches, which has
 * numer == denom == 0 and distance 0.  The best list of q is its hits ordered by (distance ascending as a double, reference
 * index ascending), cut to n_best: the first n_best rows of a stable sort of q's row of the dense grid once the rows with
 * numer == 0 or pass == 0 are dropped.  numer, denom, distance and pvalue of a hit are bit-identical to what
 * mashgpu_dist_run returns for the pair from the same job.
 * Row (q - q_begin) of ref / numer / denom / distance / pvalue holds n_best entries in rank order, n_hits[q - q_begin] of them
 * valid (the entries past them are zero); n_total (may be NULL) is the number of hits the query has in all.  ref is relative
 * to the job's references (to ref_begin for mashgpu_dist_open_encoded), like the column of the grid.
 * 1 <= n_best <= 1024: 0 is MASHGPU_ERR_INVALID, more MASHGPU_ERR_UNSUPPORTED, both before any work.  In a self comparison
 * every non-empty sketch is its own nearest hit: ask for n_best + 1.
 * The output is q_count x n_best entries instead of q_count x n_ref, so a search of a large collection runs at the speed of
 * the kernels, not of the link to the host.  Works on every kind of job and every merge path.  Host buffers. */
int mashgpu_dist_run_best(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count, uint32_t n_best,
                          uint32_t *n_hits, uint32_t *n_total, uint32_t *ref, uint32_t *numer, uint32_t *denom, double *distance,
                          double *pvalue);
/* Same with device output buffers and a stream (NULL = context stream); entries past n_hits are zero here too.  The hits are
 * captured in a bounded candidate buffer, block of queries by block, and the call reads the candidate count of every block on
 * the host (it synchronises `stream`, as mashgpu_dist_run_list does): a block whose hits exceed the buffer is discarded and run
 * again as two halves, so no hit is ever dropped.  The rule of mashgpu_dist_run_dev holds: one run of a job in flight. */
int mashgpu_dist_run_best_dev(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count, uint32_t n_best,
                              uint32_t *d_n_hits, uint32_t *d_n_total, uint32_t *d_ref, uint32_t *d_numer, uint32_t *d_denom,
                              double *d_distance, double *d_pvalue, void *stream);
/* Capacity of the candidate buffer in entries (32 bytes each, held twice).  Default 2^25; never below the number of references,
 * so that the hits of one query always fit (smaller values are raised to it, 0 restores the default), and below 2^32. */
int mashgpu_dist_set_best_capacity(mashgpu_dist_job *job, uint64_t entries);
/* Counters of the best runs since the job was opened: blocks of queries run (the re-runs of split blocks included), blocks
 * discarded and split because their hits exceeded the candidate buffer, hits captured by the blocks that were kept, and, when
 * mashgpu_set_timing is on, the device time of grouping and selection.  Any pointer may be NULL. */
int mashgpu_dist_best_stats(mashgpu_dist_job *job, uint64_t *blocks_run, uint64_t *blocks_split, uint64_t *candidates, double *select_ms);

/* Connected components of the passing pairs that share a hash (DESIGN.md 3.8); no counterpart in the reference.
 * Self jobs (qry == NULL) and encoded jobs only; the pairs are enumerated in the lower triangle whatever
 * mashgpu_dist_set_triangle says.  labels[i] = smallest index of sketch i's component, n_qry entries.
 * The component graph has one vertex per query row and an edge {q, r'} for every pair (q, r) of the lower triangle with
 * pass == 1 in mashgpu_dist_run and numer > 0 (the hit rule of mashgpu_dist_run_best: max_distance and max_pvalue apply, two
 * empty sketches are not joined), where r' = r for a self job and ref_begin + r for an encoded one.  So an encoded job over a
 * shard of the reference axis yields the components of that shard's edges over all n_rows sketches; the union of the shards'
 * graphs is the whole graph (shard.merge_component_labels).  *n_edges = number of edges, every unordered pair once.  The labels
 * do not depend on the order in which the pairs were evaluated.  A job with a separate query set and NULL outputs are
 * MASHGPU_ERR_INVALID.  Synchronises the stream (the edge count is read on the host). */
int mashgpu_dist_components(mashgpu_dist_job *job, uint32_t *labels, uint64_t *n_edges);
int mashgpu_dist_components_dev(mashgpu_dist_job *job, uint32_t *d_labels, uint64_t *n_edges, void *stream);

/* Minimum spanning forest of the component graph above, weighted by distance (DESIGN.md 3.9); no counterpart in the reference.
 * Self jobs (qry == NULL) and encoded jobs only; the lower triangle whatever mashgpu_dist_set_triangle says.  The graph is the one of
 * mashgpu_dist_components: an edge {i, j}, j < i, for every pair (q = i, r) with pass == 1 and numer > 0, j = r for a self job and
 * ref_begin + r for an encoded one.  Edges are ordered by the strict total order (distance as a double, j, i), under which the forest
 * is unique: it equals Kruskal's algorithm over the dense grid under that order, whatever the evaluation order or the merge path.
 * For every t <= max_distance the forest edges with distance <= t have the components of mashgpu_dist_components at
 * max_distance t (the same max_pvalue): the forest is the single-linkage dendrogram of the passing pairs.
 * Outputs: *n_edges <= n_qry - 1 edges in that order (capacity n_qry - 1 each), row = i, col = j, and numer, denom, distance, pvalue
 * bit-identical to what mashgpu_dist_run returns for (q = i, r = j - ref_begin) of the same job.  *n_rounds = Boruvka rounds run
 * (at most ceil(log2 n_qry) + 1).  An encoded job over a shard of the reference axis yields the forest of that shard's edges; the
 * forest of the union of the shards' forests is the global one (shard.merge_spanning_forests).  0 or 1 sketches give 0 edges and
 * 0 rounds.  A job with a separate query set and NULL outputs are MASHGPU_ERR_INVALID.  Synchronises the stream. */
int mashgpu_dist_spanning_forest(mashgpu_dist_job *job, uint32_t *row, uint32_t *col, uint32_t *numer, uint32_t *denom, double *distance,
                                 double *pvalue, uint64_t *n_edges, uint64_t *n_rounds);
int mashgpu_dist_spanning_forest_dev(mashgpu_dist_job *job, uint32_t *d_row, uint32_t *d_col, uint32_t *d_numer, uint32_t *d_denom,
                                     double *d_distance, double *d_pvalue, uint64_t *n_edges, uint64_t *n_rounds, void *stream);

/* Greedy dereplication of the component graph above (DESIGN.md 3.12); no counterpart in the reference.  Self jobs (qry == NULL) only;
 * the lower triangle whatever mashgpu_dist_set_triangle says.  The graph is the one of mashgpu_dist_components: an edge {i, j}, j < i,
 * for every pair (q = i, r = j) with pass == 1 and numer > 0.  The greedy order is the index order (a caller that wants another order
 * opens the job over a permuted set):
 *   representatives: for v = 0 .. n-1, v is a representative iff no representative u < v has an edge {u, v} (the lexicographically
 *   first maximal independent set);
 *   assignment: a member m goes to the representative r adjacent to it with the least (distance as a double, min(m, r), max(m, r)),
 *   the spanning forest's edge order -- its nearest one, ties to the smaller index, later representatives included.  An earlier
 *   representative is always adjacent, so every member has one.
 * Outputs of n_qry entries: rep[i] = sketch i's representative, i itself for a representative; for a member, numer, denom, distance
 * and pvalue bit-identical to what mashgpu_dist_run returns for (q = max(i, rep[i]), r = min(i, rep[i])), for a representative zeros.
 * *n_reps = number of representatives, *n_rounds = resolution rounds over all blocks (at most the rows of each block).  The result
 * depends only on the grid: not on the merge path, the prefilter, the block size or the run.  Memory: O(n) plus one block's
 * rows x rows bit matrix.  0 or 1 sketches give the identity and 0 rounds.  A job with a separate query set and NULL outputs are
 * MASHGPU_ERR_INVALID, an encoded job MASHGPU_ERR_UNSUPPORTED.  Synchronises the stream. */
int mashgpu_dist_representatives(mashgpu_dist_job *job, uint32_t *rep, uint32_t *numer, uint32_t *denom, double *distance, double *pvalue,
                                 uint64_t *n_reps, uint64_t *n_rounds);
int mashgpu_dist_representatives_dev(mashgpu_dist_job *job, uint32_t *d_rep, uint32_t *d_numer, uint32_t *d_denom, double *d_distance,
                                     double *d_pvalue, uint64_t *n_reps, uint64_t *n_rounds, void *stream);
/* Rows of one block of the representatives' first pass (each block is one lower-triangle run followed by its resolve rounds).
 * 0 = default, min(2^31 / n, 32768); larger values are cut to 32768 (a 128 MiB bit matrix).  The result does not depend on it. */
int mashgpu_dist_set_representative_block(mashgpu_dist_job *job, uint64_t rows);

/* Neighbor joining (DESIGN.md 3.10); no counterpart in the reference.  Canonical Saitou-Nei / Studier-Keppler NJ over a symmetric
 * n x n float64 matrix D of which only the lower triangle (j < i) is read, with the operation order fixed so that it is
 * reproducible bit for bit (tests/nj_model.py):
 *   r_i = sum of D(i, k) over ascending k, D(i, i) = 0.  While m = |live| > 3, over live positions p < q (a = L[p], b = L[q]) the
 *   least (Q, q, p) with Q = ((m - 2) * D(a, b) - r_a) - r_b is joined into node u = n + s (join s):
 *   la = D(a, b) * 0.5 + (r_a - r_b) / (2 * (m - 2)), lb = D(a, b) - la, D(u, k) = ((D(a, k) + D(b, k)) - D(a, b)) * 0.5,
 *   r_k = ((r_k - D(a, k)) - D(b, k)) + D(u, k), r_u = ((r_a + r_b) - m * D(a, b)) * 0.5; u takes position p, q is removed.
 *   The last three x, y, z hang from the center 2n - 3 with lx = ((D(x, y) + D(x, z)) - D(y, z)) * 0.5 and so on.
 * Every step is one IEEE double operation, never fused.  Row sums are updated, not recomputed, so they drift from the exact sums
 * by rounding; negative branch lengths are returned as computed (no clamping).
 * Outputs of 2n - 2 entries, nodes 0..n-1 the leaves: parent[v] and length[v] of v's branch; the center has parent UINT32_MAX and
 * length 0.  Memory: the matrix plus O(n). */
/* NJ over the caller's n x n float64 device matrix (row i at d_matrix + i * ld, ld >= n; lower triangle read; the matrix is used as
 * scratch and overwritten).  Host outputs of 2n-2 entries; synchronises `stream` (NULL: the context's stream).  n < 3 or a
 * non-finite entry in the lower triangle: MASHGPU_ERR_INVALID (the entry is found on the device before the first join). */
int mashgpu_neighbor_joining_matrix(mashgpu_ctx *ctx, double *d_matrix, uint64_t n, uint64_t ld,
                                    uint32_t *parent, double *length, void *stream);
/* NJ over every pair's distance of a self job (qry == NULL): D(i, j), j < i, is the distance mashgpu_dist_run returns for
 * (q = i, r = j), whatever max_distance, max_pvalue and mashgpu_dist_set_triangle say (none of them is changed).  The job fills an
 * n x n device matrix with its own runs, then runs mashgpu_neighbor_joining_matrix on it.  n_qry < 3 and a job with a separate query
 * set: MASHGPU_ERR_INVALID.  Encoded (sharded) jobs: MASHGPU_ERR_UNSUPPORTED.  8 n^2 bytes beyond the device's free memory:
 * MASHGPU_ERR_NOMEM before anything is allocated. */
int mashgpu_dist_neighbor_joining(mashgpu_dist_job *job, uint32_t *parent, double *length);

/* Average (UPGMA) and complete linkage (DESIGN.md 3.11); no counterpart in the reference.  Hierarchical clustering of a symmetric
 * n x n float64 matrix D of which only the lower triangle (j < i) is read, with the merge order and the operation order fixed so
 * that it is reproducible bit for bit (tests/linkage_model.py):
 *   Clusters occupy slots; leaf i starts in slot i.  While more than one slot is live, the least (D(a, b), b, a) over live slots
 *   a < b is merged (ties go to the first pair of the lower triangle in row-major order).  Merge s makes node u = n + s with
 *   height D(a, b) and size n_a + n_b; u takes slot a, slot b dies, and for every other live k
 *     average:  D(u, k) = ((double)n_a * D(a, k) + (double)n_b * D(b, k)) / (double)(n_a + n_b)
 *     complete: D(u, k) = max(D(a, k), D(b, k)) (D(a, k) when they are equal).
 * Every step is one IEEE double operation, never fused.  Heights are returned as computed: rounding in the average can make a
 * later height smaller than an earlier one by an ulp.  The average is the size-weighted mean of scipy's `average` method, but scipy
 * merges in another order, so its values may differ in the last bits.
 * Outputs of n - 1 entries in merge order, scipy's Z layout (scipy.cluster.hierarchy.fcluster, cophenet and dendrogram take it
 * unchanged): id_lo[s] < id_hi[s] the merged node ids (0..n-1 the leaves), height[s], size[s] the leaves under n + s.
 * rows_rescanned (may be NULL): the rows whose nearest-neighbour cache was rebuilt, which is what the device work scales with
 * beyond its O(n) per merge.  Memory: the matrix plus O(n). */
#define MASHGPU_LINKAGE_AVERAGE 0
#define MASHGPU_LINKAGE_COMPLETE 1
/* Linkage over the caller's n x n float64 device matrix (row i at d_matrix + i * ld, ld >= n; lower triangle read; the matrix is
 * used as scratch and overwritten, columns past n are neither read nor written).  Host outputs of n - 1 entries; synchronises
 * `stream` (NULL: the context's stream).  n < 2, ld < n, NULL outputs, a method other than the two above, or a non-finite entry in
 * the lower triangle: MASHGPU_ERR_INVALID (the entry is found on the device before the first merge). */
int mashgpu_linkage_matrix(mashgpu_ctx *ctx, double *d_matrix, uint64_t n, uint64_t ld, int method, uint32_t *id_lo, uint32_t *id_hi,
                           double *height, uint32_t *size, uint64_t *rows_rescanned, void *stream);
/* Linkage over every pair's distance of a self job (qry == NULL): D(i, j), j < i, is the distance mashgpu_dist_run returns for
 * (q = i, r = j), whatever max_distance, max_pvalue and mashgpu_dist_set_triangle say (none of them is changed); pairs without a
 * shared hash have distance 1.  The job fills an n x n device matrix with its own runs, then runs mashgpu_linkage_matrix on it.
 * n_qry < 2, a job with a separate query set, NULL outputs or an unknown method: MASHGPU_ERR_INVALID.  Encoded (sharded) jobs:
 * MASHGPU_ERR_UNSUPPORTED.  8 n^2 bytes beyond the device's free memory: MASHGPU_ERR_NOMEM before anything is allocated. */
int mashgpu_dist_linkage(mashgpu_dist_job *job, int method, uint32_t *id_lo, uint32_t *id_hi, double *height, uint32_t *size,
                         uint64_t *rows_rescanned);
/* The flat clusters of mashgpu_dist_linkage's tree cut at height t (DESIGN.md 3.13), without the n x n matrix: memory and time scale
 * with the largest component of the graph below, not with n.  labels[i] (n_qry entries) = the smallest index in sketch i's flat
 * cluster, scipy's fcluster(Z, t, "distance") of the whole set's Z: a maximal subtree whose largest merge height is <= t.
 * With T = t (1 + 8 n 2^-53) rounded up and T < 1, the set splits into the components of the pairs at distance <= T: those that share
 * a hash (mashgpu_dist_components at max_distance T, no p-value test) and the pairs of empty sketches (distance 0); every other pair
 * is at distance 1.  No merge at height <= t joins two of these components, so the cut of each
 * component's own linkage (the same definition and arithmetic, over its members in index order) is the whole set's cut there, bit
 * for bit, ties included.  With T >= 1 the whole set is one component.  A component of up to a few hundred members is linked inside
 * one CTA; a larger one through an m x m device matrix and mashgpu_linkage_matrix, with the same merges.
 * Optional merge forest (id_lo, id_hi, height, size: all NULL or all given, max(n_qry - 1, 0) entries each): each component's own
 * linkage in scipy's Z layout, leaves = sketch indices, merge s = node n_qry + s; the first n_qry - *n_components entries are written,
 * grouped by component in the order of its smallest member and in merge order within one.  Merges at height <= t are the whole
 * set's merges (heights bit-identical); merges above t are the component's own linkage, not the whole set's.
 * *n_clusters = number of flat clusters, *n_components = components (singletons included), *largest_component = its members.
 * The job's max_distance, max_pvalue and mashgpu_dist_set_triangle are ignored and left unchanged.  0 or 1 sketches give the
 * identity.  A job with a separate query set, NULL required outputs, a partial forest, an unknown method, or t NaN or negative:
 * MASHGPU_ERR_INVALID; an encoded (sharded) job: MASHGPU_ERR_UNSUPPORTED; a component whose 8 m^2 bytes exceed the device's free
 * memory: MASHGPU_ERR_NOMEM before its matrix is allocated.  Synchronises the stream. */
int mashgpu_dist_linkage_cut(mashgpu_dist_job *job, int method, double t, uint32_t *labels, uint32_t *id_lo, uint32_t *id_hi, double *height,
                             uint32_t *size, uint64_t *n_clusters, uint64_t *n_components, uint64_t *largest_component);
/* The largest component mashgpu_dist_linkage_cut links inside one CTA (0 = default, the most that fits its shared memory, 238;
 * larger values are cut to it; 1 sends every component to the matrix tier).  The result does not depend on it. */
int mashgpu_dist_set_linkage_cut_cta_max(mashgpu_dist_job *job, uint64_t members);
/* Device time in ms of the last mashgpu_dist_linkage_cut's phases: components, grouping, CTA tier, matrix tier (4 entries). */
int mashgpu_dist_linkage_cut_stats(mashgpu_dist_job *job, double *phase_ms);

/* ---- Sharded dictionary build (multi-GPU all-vs-all; DESIGN.md 5).  With the reference axis sharded over G ranks the
 * dictionary of mashgpu_dist_open would be rebuilt in full on every rank.  These entry points split it by HASH RANGE
 * instead (a sample sort): a rank sorts only its own rows' hashes, the sorted keys are cut at G-1 splitters, every rank
 * receives one hash range from all ranks (the caller's all-to-all, NCCL), ranks the distinct values of its range, and the
 * 32-bit codes travel back; the owners scatter them into rows of sketch_size+1 codes which are then all-gathered (4 B per
 * hash instead of 8) and opened with mashgpu_dist_open_encoded.  Codes of range d are offset by the number of distinct
 * values in the ranges below it, so the encoding is order- and equality-preserving over the whole collection, which is
 * all the merge of compareSketches (CommandDistance.cpp:347-365) depends on.  All pointers named d_* are device memory;
 * `stream` is a cudaStream_t (NULL = the context's stream); the calls that return a host value synchronise it. */
/* Hashes i < min(n_hashes, sketch_size+1, stride) of every row, ascending, with their slot row * (sketch_size+1) + i.
 * d_keys / d_slots must hold set->n * min(stride, sketch_size+1) entries; *n_valid = number of entries written. */
int mashgpu_dict_local_sort(mashgpu_ctx *ctx, const mashgpu_sketch_set *set, uint64_t sketch_size,
                            uint64_t *d_keys, uint32_t *d_slots, uint64_t *n_valid, void *stream);
/* counts[p] = number of keys of the ascending list d_keys[0..n) in part p of n_parts: part p holds
 * splitters[p-1] <= key < splitters[p] (splitters: host array of n_parts-1 ascending values). */
int mashgpu_dict_split(mashgpu_ctx *ctx, const uint64_t *d_keys, uint64_t n, const uint64_t *splitters, uint32_t n_parts,
                       uint64_t *counts, void *stream);
/* d_codes[t] = number of distinct keys smaller than d_keys[t] (any order of d_keys; equal keys get equal codes);
 * *n_distinct = number of distinct keys. */
int mashgpu_dict_rank(mashgpu_ctx *ctx, const uint64_t *d_keys, uint64_t n, uint32_t *d_codes, uint64_t *n_distinct, void *stream);
/* Rows of sketch_size+1 codes from the codes of this rank's sorted keys: entry t (in the order of mashgpu_dict_local_sort)
 * belongs to segment g = the part it was sent to (seg_counts[g] consecutive entries, host arrays of n_segs) and becomes
 * d_rows[d_slots[t]] = d_codes[t] + seg_base[g]; every other position of the n_rows rows is the padding code 0xFFFFFFFF.
 * d_n_eff[row] = min(n_hashes, sketch_size+1, stride).  Fails when a code would reach the padding value. */
int mashgpu_dict_scatter(mashgpu_ctx *ctx, const uint32_t *d_codes, const uint32_t *d_slots, const uint64_t *seg_counts,
                         const uint64_t *seg_base, uint32_t n_segs, const mashgpu_sketch_set *set, uint64_t sketch_size,
                         uint32_t *d_rows, uint32_t *d_n_eff, void *stream);
/* A job over rows that are already dictionary-encoded (device memory, owned by the caller, must outlive the job):
 * n_rows rows of sketch_size+1 codes, d_n_eff / d_length per row.  The queries are all n_rows rows, the references rows
 * [ref_begin, ref_begin + ref_count): pair (q, r) of a run is query row q against row ref_begin + r, written at
 * (q - q_begin) * ref_count + r.  mashgpu_dist_set_triangle compares q with rows below it only (ref_begin + r < q). */
int mashgpu_dist_open_encoded(mashgpu_ctx *ctx, const uint32_t *d_rows, const uint32_t *d_n_eff, const uint64_t *d_length,
                              uint64_t n_rows, uint64_t ref_begin, uint64_t ref_count, const mashgpu_dist_params *params,
                              mashgpu_dist_job **job);

/* One-shot convenience: open + run over all queries + close (the whole `compare` grid). */
int mashgpu_dist(mashgpu_ctx *ctx, const mashgpu_sketch_set *ref, const mashgpu_sketch_set *qry,
                 const mashgpu_dist_params *params,
                 uint32_t *numer, uint32_t *denom, double *distance, double *pvalue, uint8_t *pass);

/* ---------------------------------------------------------------------------------------------------------
 * `mash within`: containment of query sketches in reference sketches, every pair (CommandContain.cpp:205-265).
 * ------------------------------------------------------------------------------------------------------- */
typedef struct mashgpu_within_job mashgpu_within_job;

/* Uploads both sets (qry == NULL or qry == ref: every sketch of one set against every other and itself) and encodes them with
 * the order-preserving 32-bit dictionary of mashgpu_dist_open.  Reference rows take part in full: unlike dist's rows they are not
 * cut to a sketch size (containSketches walks min(|R|, |Q|) query hashes but as many reference hashes as it needs,
 * CommandContain.cpp:231-258).  Each row r holds n_hashes[r] ascending distinct hashes; a row with n_hashes > stride is refused
 * (MASHGPU_ERR_INVALID) before any work.  length is not read (NULL allowed).  max_error: the -e threshold of writeOutput
 * (CommandContain.cpp:179-203), as the double the caller compares with -- the CLI passes (double)(float)e. */
int mashgpu_within_open(mashgpu_ctx *ctx, const mashgpu_sketch_set *ref, const mashgpu_sketch_set *qry, double max_error,
                        mashgpu_within_job **job);
/* containSketches(ref r, query q) for queries [q_begin, q_begin + q_count) and every reference, pair (q, r) written at
 * (q - q_begin) * n_ref + r (the query-major order of CommandContain.cpp:143-175):
 *   common    shared hashes among the query hashes examined
 *   examined  j, the query hashes examined: min(min(|R|, |Q|), #{query hashes <= the largest reference hash})
 *   score     common / j (CommandContain.cpp:264); for j == 0 the x86 result of 0.0 / 0, a NaN with the sign bit set
 *   error     1 / sqrt(j) (:262); +inf for j == 0
 *   pass      error <= max_error (writeOutput, :189)
 * score and error are bit-identical to the reference's.  Reference sketches of up to 1034 hashes run a tiled lockstep merge
 * (32 references per shared-memory tile), larger ones a warp-per-pair merge.  Any output pointer may be NULL.  Host buffers;
 * the device outputs are cut into chunks of 2^24 pairs. */
int mashgpu_within_run(mashgpu_within_job *job, uint64_t q_begin, uint64_t q_count, uint32_t *common, uint32_t *examined,
                       double *score, double *error, uint8_t *pass);
/* Same with device output buffers, enqueued on `stream` (cudaStream_t, NULL = context stream); runs of one job may be in flight
 * on several streams at once (the job keeps no per-run scratch). */
int mashgpu_within_run_dev(mashgpu_within_job *job, uint64_t q_begin, uint64_t q_count, uint32_t *d_common, uint32_t *d_examined,
                           double *d_score, double *d_error, uint8_t *d_pass, void *stream);
int mashgpu_within_close(mashgpu_within_job *job);

/* ---------------------------------------------------------------------------------------------------------
 * Hot path 3: screen (containment of reference sketches in a read stream).
 * ------------------------------------------------------------------------------------------------------- */
typedef struct mashgpu_screen_job mashgpu_screen_job;

/* Builds the distinct-hash table of the reference sketches with zeroed counters (CommandScreen.cpp:93-114).
 * The alphabet picks the mode, as in the reference (CommandScreen.cpp:120):
 *   {A,C,G,T}                        nucleotide k-mers of the reads (canonical unless noncanonical);
 *   exactly ACDEFGHIKLMNPQRSTVWY     translated screen: every chunk is translated in all six frames (standard genetic code;
 *                                    a stop codon or a codon with a byte outside {A,C,G,T} ends the peptide; 'U' counts as
 *                                    'A' on the reverse strand only, as the reference's complement table has it) and its
 *                                    non-canonical amino-acid k-mers are screened; kmer space 20^k;
 *   any other alphabet (-z)          byte k-mers of the reads as they stand.
 * Non-nucleotide jobs always upload ASCII (MASHGPU_SCREEN_HOST_PACK is ignored).
 * Refused before any table is built: sketch_size > 8192 (MASHGPU_ERR_UNSUPPORTED); a row with n_hashes[r] > stride
 * (MASHGPU_ERR_INVALID); a reference sketch of more than 32768 hashes (MASHGPU_ERR_UNSUPPORTED; the stride may be larger);
 * a reference hash >= 2^32 in a 32-bit job, i.e. when the k-mer space is at most 2^32 (MASHGPU_ERR_INVALID); the hash value
 * 2^64-1 (MASHGPU_ERR_UNSUPPORTED). */
int mashgpu_screen_open(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, const mashgpu_sketch_set *refs,
                        mashgpu_screen_job **job);
/* One HashInput (CommandScreen.h:104-133): a '*'-joined chunk of reads (CommandScreen.cpp:224-262; any byte
 * outside the alphabet separates reads).  Host buffer; chunks may be of any size: chunks below 4 MiB are joined before a kernel
 * pass, larger ones are pipelined (the copy of chunk i+1 overlaps the kernels of chunk i).  The call returns as soon as the
 * caller's buffer may be reused; results are complete at mashgpu_screen_finish.  (MASHGPU_SCREEN_HOST_PACK=1: the chunk is 2-bit
 * packed on the host threads and uploaded with an invalid-position mask instead of as ASCII.) */
int mashgpu_screen_feed(mashgpu_screen_job *job, const char *chunk, uint64_t len);
/* Same for a chunk already in device memory (readable up to len rounded up to 16), at any address: an untranslated job
 * scans a chunk that is not 16-byte aligned from an aligned device copy. */
int mashgpu_screen_feed_dev(mashgpu_screen_job *job, const void *d_chunk, uint64_t len);
/* Reduce (CommandScreen.cpp:288-355, 409-455): per reference sketch i the number of its hashes seen at least
 * once (shared), the median multiplicity depths[shared/2], identity (estimateIdentity, :463-482) and p-value
 * (pValueWithin, :601-615); *set_size = (uint64_t)estimateSetSize() of the mixture's bottom-s heap (:322).
 * mixture_hashes (nullable, sketch_size slots) / mixture_n receive that bottom-s list.  Host buffers. */
int mashgpu_screen_finish(mashgpu_screen_job *job, uint64_t *shared, uint64_t *median, double *identity,
                          double *pvalue, uint64_t *set_size, uint64_t *mixture_hashes, uint32_t *mixture_n);
/* `mash screen -w` ("winner take all", CommandScreen.cpp:357-407): on != 0 makes mashgpu_screen_finish re-assign every
 * reference hash seen in the mixture to the one sketch, among those containing it, with the highest identity estimate
 * (ties: the longer genome, refs->length at mashgpu_screen_open; a tie in both goes to the lowest index -- the reference
 * leaves it to the iteration order of a hash set) before shared / median / identity / p-value are computed. */
int mashgpu_screen_set_winner(mashgpu_screen_job *job, int on);
/* Screening samples one after another against one resident table (`mash screen -I`).  After mashgpu_screen_reset, every
 * finish of the job returns, bit for bit, what a fresh job over the same sketches fed only the chunks fed since would return.
 *
 * mashgpu_screen_finish_hits: the values of mashgpu_screen_finish at exactly the sketches with shared >= 1 (under -w: after
 * the reallocation), in ascending sketch index: ref[i], shared[i], median[i], identity[i], pvalue[i] for i < *n_rows.  Every
 * other sketch has shared 0, median 0, p-value 1.0 and identity 0 (1.0 for a sketch of 0 hashes).  Host buffers of n_ref
 * entries each (any of ref .. pvalue and set_size may be NULL); honours mashgpu_screen_set_winner; leaves the job unchanged,
 * like mashgpu_screen_finish.  The work follows the sample's hits through an inverted index (distinct hash -> sketches)
 * built at the first call and kept until close: 4 B per (sketch, hash) pair plus 4 B per distinct hash, with scratch of
 * another 4 B per pair so that no later call allocates.  MASHGPU_ERR_UNSUPPORTED for 2^32 or more pairs (32-bit segment
 * offsets), MASHGPU_ERR_NOMEM when the index does not fit on the device.
 *
 * mashgpu_screen_reset: starts a new sample and keeps the table, the bitmap and the -w setting.  Feeds the small chunks still
 * joined in the library and collects the chunk in flight (their counts are then dropped), zeroes the hit counters (only those
 * hit, when no chunk was fed since a mashgpu_screen_finish_hits) and empties the mixture's bottom-s list.  Allocates nothing.
 *
 * mashgpu_screen_hits_stats: for the last mashgpu_screen_finish_hits, the distinct reference hashes the sample hit, the
 * (hash, sketch) pairs expanded from them, the device time of the one-off index build and of the call's own device work
 * (CUDA events, ms).  Any pointer may be NULL. */
int mashgpu_screen_finish_hits(mashgpu_screen_job *job, uint32_t *ref, uint64_t *shared, uint64_t *median, double *identity,
                               double *pvalue, uint64_t *n_rows, uint64_t *set_size);
int mashgpu_screen_reset(mashgpu_screen_job *job);
int mashgpu_screen_hits_stats(mashgpu_screen_job *job, uint64_t *hit_hashes, uint64_t *hit_pairs, double *index_ms, double *finish_ms);
/* Multi-GPU screening (reads sharded over ranks, table replicated): the hit counters live in device memory as one
 * uint32 per distinct reference hash, in ascending hash order, so counter i means the same hash on every rank that
 * opened the job with the same sketches.  *d_counters / *n_counters expose that array for an all-reduce(sum) (NCCL via torch.distributed); the
 * mixture bottom-s lists of the other ranks are folded in with mashgpu_screen_merge_mixture (ascending distinct hashes,
 * host buffer) -- bottom-s of a union is the bottom-s of the union of bottom-s lists (the reference merges its
 * per-thread heaps the same way, CommandScreen.cpp:288-302).  Then mashgpu_screen_finish as usual. */
int mashgpu_screen_counters(mashgpu_screen_job *job, uint32_t **d_counters, uint64_t *n_counters);
int mashgpu_screen_merge_mixture(mashgpu_screen_job *job, const uint64_t *hashes, uint32_t n);
/* The same without a host round trip per rank: *d_mix / *d_mix_n expose the running bottom-s list (sketch_size uint64 slots,
 * ascending, *d_mix_n of them valid) for an all-gather; mashgpu_screen_merge_mixtures_dev folds n_lists lists lying in
 * device memory (list i = d_hashes[i * stride ...], d_n[i] ascending distinct hashes; the job's own list may be among
 * them) into the job's list with one kernel and one read-back of the new top. */
int mashgpu_screen_mixture_dev(mashgpu_screen_job *job, uint64_t **d_mix, uint32_t **d_mix_n);
int mashgpu_screen_merge_mixtures_dev(mashgpu_screen_job *job, const uint64_t *d_hashes, const uint32_t *d_n, uint32_t n_lists, uint64_t stride);
int mashgpu_screen_close(mashgpu_screen_job *job);

/* ---------------------------------------------------------------------------------------------------------
 * `mash taxscreen`: lowest-common-ancestor taxon of every distinct reference hash of a screen job, counted per taxon and
 * rolled up the tree (CommandTaxScreen.cpp:415-471, TaxDB::getLowestCommonAncestor taxdb.hpp:158-190).
 * ------------------------------------------------------------------------------------------------------- */
typedef struct mashgpu_taxonomy mashgpu_taxonomy;

/* A taxonomy of n_nodes dense nodes: parent[i] is the index of node i's parent, parent[i] == i marks a root, taxid[i] is its
 * taxID (distinct).  Nodes with taxID 0 or 1 end the LCA walks as roots do (the reference's walks stop there); the roll-up
 * still goes through them to their parent.  A parent cycle is refused (MASHGPU_ERR_INVALID).  The tree stays in device
 * memory until mashgpu_taxonomy_close. */
int mashgpu_taxonomy_open(mashgpu_ctx *ctx, uint64_t n_nodes, const uint32_t *parent, const uint64_t *taxid, mashgpu_taxonomy **tax);
int mashgpu_taxonomy_close(mashgpu_taxonomy *tax);

#define MASHGPU_TAX_NONE 0xFFFFFFFFu   /* ref_code of a sketch without a taxID (taxID 0) */

/* One key of the reference's `counts` map (TaxCounts, taxdb.hpp:40-46). */
typedef struct mashgpu_tax_row {
    uint64_t taxid;
    uint64_t tax_count;          /* hashes assigned to this taxon and seen in the reads at least once */
    uint64_t tax_hash_count;     /* hashes assigned to this taxon */
    uint64_t clade_count;        /* tax_count summed over the clade; 0 for taxIDs outside the taxonomy */
    uint64_t clade_hash_count;   /* tax_hash_count summed over the clade; 0 for taxIDs outside the taxonomy */
} mashgpu_tax_row;

/* After the last chunk was fed (and, across GPUs, after the counters were all-reduced): ref_code[r] for each of the job's
 * reference sketches is a node index, n_nodes + u for the unknown taxID unknown_taxid[u] (distinct, none of them 0 or in
 * the taxonomy), or MASHGPU_TAX_NONE.  Each distinct hash h gets the reference's fold of getLowestCommonAncestor over the
 * sketches holding it:
 *   no sketch with a taxID -> 0; one -> its taxID, known or not; two or more -> 1 if any is unknown, if the known taxa share no
 *   ancestor or if their LCA is a root (or has taxID 0 or 1); otherwise the LCA.
 * Rows: one per taxon with a nonzero clade hash count, plus taxIDs outside the taxonomy (0 and unknown ones included) that got
 * hashes; ascending node index, then unknown slots, then 0 and 1.  *n_rows is their number; they are copied only when it is at
 * most `capacity` (n_nodes + n_unknown + 2 is always enough).  total_count / total_hash_count (nullable): sums of tax_count
 * and tax_hash_count over the rows.  hash_taxid (nullable, one entry per distinct hash in ascending hash order): the taxID
 * assigned to it.  unknown_in_lca (nullable, n_unknown bytes): 1 when unknown taxID u took part in a fold of two or more
 * sketches (the reference prints "TaxID u not in database" then).  Host buffers. */
int mashgpu_screen_taxonomy(mashgpu_screen_job *job, const mashgpu_taxonomy *tax, const uint32_t *ref_code,
                            uint32_t n_unknown, const uint64_t *unknown_taxid,
                            mashgpu_tax_row *rows, uint64_t capacity, uint64_t *n_rows,
                            uint64_t *total_count, uint64_t *total_hash_count,
                            uint64_t *hash_taxid, uint8_t *unknown_in_lca);

/* ---------------------------------------------------------------------------------------------------------
 * Instrumentation (bench.py): kernel launch counter and device time of the dominant kernels.
 * ------------------------------------------------------------------------------------------------------- */
typedef struct mashgpu_stats {
    uint64_t kernel_launches;      /* kernels launched by this context since the last reset */
    double scan_kernel_ms;         /* accumulated device time of the sketch/screen scan kernel (CUDA events) */
    uint64_t scan_kernel_launches;
    double dist_kernel_ms;         /* accumulated device time of the merge kernel */
    uint64_t dist_kernel_launches;
    uint64_t exact_reruns;         /* units that needed the exact re-run path */
    double translate_kernel_ms;    /* accumulated device time of the six-frame translation kernel (translated screen) */
    uint64_t translate_kernel_launches;
    double taxonomy_ms;            /* accumulated device time of mashgpu_screen_taxonomy's kernels, copies and scans */
    uint64_t reads_events;         /* k-mers replayed through the heap by reads jobs */
    double reads_replay_ms;        /* accumulated device time of the replay kernel of reads jobs (with timing on) */
    uint64_t reads_peak_device_bytes;  /* largest device footprint of the last reads job opened (not cleared by reset) */
    uint64_t unit_stages;          /* stages merged by unit jobs (mashgpu_unit_*, and the units and read sets routed to them) */
    uint64_t unit_peak_device_bytes;   /* largest device footprint of the last unit job opened (not cleared by reset) */
} mashgpu_stats;
/* timing != 0 brackets the dominant kernels with CUDA events (adds a sync at mashgpu_get_stats). */
int mashgpu_set_timing(mashgpu_ctx *ctx, int timing);
int mashgpu_get_stats(mashgpu_ctx *ctx, mashgpu_stats *out, int reset);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* MASHGPU_H */
