/* include/kuq.h — C ABI of libkuq.so: KrakenUniq's per-read classification hot path on one NVIDIA H100 (sm_90a).
 *
 * The reference (fbreitwieser/krakenuniq v1.0.4) has no plugin / FFI interface; its drop-in surface is the
 * `classify` executable and the on-disk formats (SURVEY.md §8(b)).  Inside that executable the hot path is one
 * function, `classify_sequence()` (src/classify.cpp:897-1012), called per read from the work-unit loop of
 * `process_file()` (src/classify.cpp:487-564) with the global state `KrakenDatabases`, `Parent_map` and
 * `taxon_counts` (src/classify.cpp:78,109,113).  This header is the boundary a maintainer binds instead of that
 * loop body: plain pointers and sizes in, plain arrays out, int error codes, no C++ or torch types.
 * Citations are file:line under the reference's src/.
 *
 *   reference object / call                              → entry point here
 *   ---------------------------------------------------------------------------------------------------------
 *   QuickFile::open_file + load_file (-M), KrakenDB(ptr),   kuq_stage_db            (HBM takes the place of the
 *     KrakenDBIndex(ptr)   classify.cpp:176-200,             page cache; krakendb.cpp:60-78,534-544 validation)
 *   KrakenDB::prepare_chunking / load_chunk (-x)            kuq_stage_db with a minimizer range [bin_lo,bin_hi)
 *     krakendb.cpp:411-522
 *   KrakenDB::count_taxons  krakendb.cpp:90-113             kuq_db_taxids           (by-product of staging)
 *   TaxonomyDB::getParentMap → Parent_map                   kuq_set_taxonomy
 *     taxdb.hpp:383-398, classify.cpp:217-219
 *   process_file work-unit loop + classify_sequence         kuq_classify_batch / kuq_submit_batch+kuq_wait_batch
 *     classify.cpp:506-559, 897-1012                          (host buffers) and kuq_classify_device (HBM buffers)
 *   classify_sequence_with_db_chunk (per-chunk lookups)     kuq_lookup_device   (per-window taxa of one DB range)
 *     classify.cpp:1014-1056
 *   merge + final pass of the chunked mode                  kuq_resolve_device  (calls + counters from merged taxa)
 *     classify.cpp:390-485, 663-791
 *   taxon_counts (ReadCounts<HyperLogLogPlusMinus>)         kuq_read_counts / kuq_get_registers / kuq_state_ptrs
 *     classify.cpp:78, readcounts.hpp:32-129
 *
 * Threading: a context is bound to one CUDA device and is thread-compatible (one caller at a time).  Each of
 * its `n_slots` batch slots owns a CUDA stream plus device and pinned-host staging, so H2D copy, kernels and D2H
 * copy of consecutive batches overlap when the caller alternates slots.
 */
#ifndef KUQ_H
#define KUQ_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- error codes (0 = success).  The reference calls errx()/exit() in these situations. ---------------- */
#define KUQ_OK 0
#define KUQ_E_INVALID_ARG (-1)    /* NULL pointer, zero size, bad slot ... */
#define KUQ_E_CUDA (-2)           /* a CUDA runtime call failed (kuq_last_error has the text) */
#define KUQ_E_NO_DEVICE (-3)      /* no usable sm_90 device: there is no CPU fallback */
#define KUQ_E_DB_FORMAT (-4)      /* krakendb.cpp:64-74: not JFLISTDN / val_len != 4; :541: bad index magic */
#define KUQ_E_UNSUPPORTED_K (-5)  /* k > 31 (key_bits > 62): bits 62 / 63 of a staged key word are record flags */
#define KUQ_E_STATE (-6)          /* call order: DB and taxonomy must be set before classifying, ... */
#define KUQ_E_CAPACITY (-7)       /* batch larger than the configured slot capacity */
#define KUQ_E_NOMEM (-8)          /* host or device allocation failed */
#define KUQ_E_TAXA_OVERFLOW (-9)  /* pool for the hit tables of reads with > 32 distinct taxa exhausted */
#define KUQ_E_TAXONOMY (-10)      /* cyclic parent chain in the taxonomy */

/* per-window code for an ambiguous k-mer ("A:" in the Kraken hit list, classify.cpp:846-848) */
#define KUQ_CODE_AMBIG 0xFFFFFFFFu

/* HLL mode rule to reproduce (SURVEY.md §7.3 item 1, App. C) */
#define KUQ_HLL_PRELOAD 0   /* per-work-unit sketches merged into the global map (classify.cpp:525,542-544) */
#define KUQ_HLL_CHUNKED 1   /* one global sketch per taxon (classify.cpp:719) — the `-x` path */
#define KUQ_HLL_DENSE_ONLY 2 /* p=12 registers only, no sparse-tier emulation (fastest; estimates = dense Ertl) */
#define KUQ_HLL_EXACT 3     /* classifyExact (EXACT_COUNTING, classify.cpp:46-49): sets of k-mers instead of sketches;
                               `unique` of kuq_read_counts / kuq_clade_counts is the exact set / union size.  The
                               (taxon, k-mer) table starts with kuq_config.sparse_set_slots entries of 16 bytes and
                               grows before a batch whose windows could take it past a load factor of 0.8
                               (kuq_exact_info); kuq_merge_into unites the sets of two contexts, kuq_exact_partition
                               and the kuq_exact_*partitioned calls spread them over contexts by k-mer. */

/* flags of the classify calls */
#define KUQ_F_WANT_CODES 1u     /* also return the per-window codes (4 B per base position) */
#define KUQ_F_NO_RUNS 2u        /* skip the run-length-encoded hit lists */
#define KUQ_F_NO_COUNTS 4u      /* do not touch the per-taxon counters / sketches (pure lookups) */
#define KUQ_F_STATS 8u          /* measurement aid: accumulate the algorithmic probe counts (kuq_slot_stats) */

typedef struct kuq_ctx kuq_ctx;

typedef struct kuq_config {
  int32_t device;                /* CUDA device ordinal */
  uint32_t n_slots;              /* batch slots (streams) for copy/compute overlap; 0 → 2 */
  uint32_t max_reads_per_batch;  /* slot capacity in reads; 0 → 1<<20 */
  uint64_t max_bases_per_batch;  /* slot capacity in bases (bytes of sequence); 0 → 160 MiB */
  uint64_t work_unit_size;       /* classify -u (classify.cpp:38,1106); 0 → 500000 */
  uint32_t hll_mode;             /* KUQ_HLL_* */
  uint32_t reserved0;
  uint64_t sparse_set_slots;     /* capacity (slots of 8 B) of the device set that backs the sparse HLL tier;
                                    KUQ_HLL_EXACT: initial entries (16 B) of the exact k-mer set.  Both grow on
                                    demand.  0 → 1<<26 */
} kuq_config;

/* One run of the Kraken hit list: `code:count` (classify.cpp:826-861). code = taxid, 0 (miss) or KUQ_CODE_AMBIG */
typedef struct kuq_run {
  uint32_t code;
  uint32_t count;
} kuq_run;

/* Result of one batch; every pointer refers to pinned host memory owned by the slot and stays valid until the
 * slot is submitted again. */
typedef struct kuq_batch_result {
  uint32_t n_reads;
  uint32_t reserved0;
  const uint32_t *call;        /* [n_reads] taxon call (classify.cpp:965; 0 = unclassified) */
  const uint32_t *n_windows;   /* [n_reads] k-mer windows scanned (0 when the read is shorter than k, :913) */
  const uint32_t *run_start;   /* [n_reads] first run of the read in `runs` (undefined with KUQ_F_NO_RUNS) */
  const uint32_t *run_count;   /* [n_reads] number of runs (0 → the reference prints "0:0", :994-995) */
  const kuq_run *runs;         /* [n_runs] */
  uint64_t n_runs;
  const uint32_t *codes;       /* KUQ_F_WANT_CODES: code of window i of read r at codes[read_offsets[r] -
                                  read_offsets[0] + i]; NULL otherwise */
  uint64_t n_classified;       /* reads with call != 0 (total_classified, classify.cpp:541) */
  double kernel_ms;            /* device time of the batch's kernels (CUDA events on the slot's stream) */
  /* kuq_set_threshold (krakenuniq-filter): NULL when no threshold is set */
  const uint32_t *filtered_call; /* [n_reads] taxid the call moves up to; 0 = unclassified */
  const uint32_t *filter_hits;   /* [n_reads] P = filter_hits / filter_total of the last node the walk weighed ... */
  const uint32_t *filter_total;  /* [n_reads] ... (filter_total = the read's unambiguous k-mers); 0 / 0 = none, P 0 */
  /* kuq_set_extract (krakenuniq-extract-reads): NULL / 0 when no extraction is set */
  const uint8_t *extract_sel;    /* [n_reads] bit 0: the read's Kraken line is selected, XOR KUQ_EXTRACT_INVERT; bit 1: the
                                    read has no Kraken line (call 0 under KUQ_EXTRACT_CLASSIFIED_ONLY) */
  uint64_t n_extract;            /* reads of the batch whose Kraken line is selected (before the inversion) */
} kuq_batch_result;

/* Device-side view of a slot's outputs after kuq_classify_device / kuq_resolve_device (HBM pointers). */
typedef struct kuq_device_result {
  const uint32_t *d_call;      /* [n_reads] raw taxids */
  const uint32_t *d_n_windows; /* [n_reads] */
  const uint32_t *d_codes;     /* per window, indexed like the bases; taxids / KUQ_CODE_AMBIG (KUQ_F_WANT_CODES) */
  const uint32_t *d_run_start;
  const uint32_t *d_run_count;
  const kuq_run *d_runs;
  const uint64_t *d_n_runs;    /* device scalar */
} kuq_device_result;

/* Raw device pointers to the per-taxon state, for the cross-GPU merge the caller performs with NCCL
 * (allreduce MAX over regs, SUM over the counters) when reads or DB ranges are spread over GPUs (SURVEY §8(e)).
 * Write through them only while no call of the context is in flight: each counting launch takes a lower bound of every
 * sketch's registers when it starts and relies on the registers not shrinking until it ends. */
typedef struct kuq_state_ptrs {
  uint8_t *d_regs;             /* [n_sketch][4096] HLL registers, p = 12 (readcounts.hpp:40) */
  uint64_t regs_bytes;
  uint64_t *d_n_kmers;         /* [n_sketch] add_kmer count per taxon (readcounts.hpp:71-74) */
  uint64_t *d_n_reads;         /* [n_taxa]   incrementReadCount per taxon (readcounts.hpp:36) */
  uint8_t *d_dense_flag;       /* [n_sketch] 1 = some sketch of the taxon converted to dense (mode emulation) */
  uint32_t n_sketch;
  uint32_t n_taxa;
} kuq_state_ptrs;

void kuq_config_default(kuq_config *cfg);
int kuq_create(const kuq_config *cfg, kuq_ctx **ctx_out);
void kuq_destroy(kuq_ctx *ctx);
const char *kuq_strerror(int code);
const char *kuq_last_error(const kuq_ctx *ctx);
/* Build identification: "libkuq <version> sm_90a" */
const char *kuq_version(void);
/* Number of device ordinals [0, n) among which sm_90 devices were found (0 without a usable GPU). */
int kuq_device_count(void);

/* ---- database -------------------------------------------------------------------------------------------- */
/* Stage (a minimizer range of) the database into HBM.  kdb_image / idx_image are the bytes of database.kdb and
 * database.idx (mmap'ed files are fine).  Bins [bin_lo, bin_hi) are copied; bin_hi = 0 means "to the end".
 * Replaces a previously staged range (the `load_chunk` step of the chunked mode, krakendb.cpp:411-425).
 * Any k up to 31.  The file's records are key_len + 4 bytes (key_len = ceil(2k / 8): 12 bytes for k = 29..31,
 * 8 to 11 bytes below); in HBM every record takes 12 bytes {u64 key, u32 value}.  Shorter records are copied as they
 * are and widened on the device, through a landing zone of 64 MiB (environment variable KUQ_LANDING_BYTES overrides
 * its size) that exists only during the call. */
int kuq_stage_db(kuq_ctx *ctx, const void *kdb_image, uint64_t kdb_bytes, const void *idx_image,
                 uint64_t idx_bytes, uint64_t bin_lo, uint64_t bin_hi);
/* Adopt a database that already lives in HBM (records in on-disk layout, values still raw taxids; offsets =
 * the full 4^nt+1 table or, with bin_lo>0, the slice starting at bin_lo).  The buffers stay owned by the caller
 * but the record values are rewritten in place (taxid → dense id).  The on-disk layout is the staged layout only for
 * 12-byte records, so this call takes k = 29..31; stage other databases with kuq_stage_db. */
int kuq_attach_db_device(kuq_ctx *ctx, void *d_pairs, uint64_t key_ct, const uint64_t *d_offsets, uint32_t k,
                         uint32_t nt, uint32_t idx_type, uint64_t bin_lo, uint64_t bin_hi);
/* Several databases resident at once (`classify -d a -d b`, classify.cpp:928-936): stage one more WHOLE database behind
 * those already staged (with none staged, the call is kuq_stage_db of the whole database).  Staging order is the order
 * in which the databases are asked: every k-mer takes the value of the first one that holds the key, a stored taxon 0
 * included.  Records are widened and remapped like kuq_stage_db's; the databases share k (else KUQ_E_INVALID_ARG) and may
 * differ in minimizer length and index type.  kuq_stage_db drops every appended database again.
 * On a context with several databases kuq_submit_batch / kuq_classify_batch / kuq_classify_device run, on the slot's
 * stream and into its own buffers: k_scan, the in-order lookup (one launch per run of consecutive databases with the same
 * (nt, index type), up to 8 databases per launch; later runs fill only windows no earlier run answered), then the
 * resolve half.  Results take the same form as on one database; the sparse HLL tier is filled by the resolve half (no
 * record flags).  kuq_lookup_batch / kuq_lookup_device return the merged first-hit codes, a stored zero always as
 * KUQ_CODE_FOUND_ZERO.  kuq_db_taxids reports the union over the staged databases (record counts summed).  Shard
 * counting and kuq_lookup_device_peers are refused (KUQ_E_STATE); kuq_lookup_device_peers_run shards them.
 * kuq_stage_db_append = kuq_stage_db_append_range(..., 0, 0). */
int kuq_stage_db_append(kuq_ctx *ctx, const void *kdb_image, uint64_t kdb_bytes, const void *idx_image, uint64_t idx_bytes);
/* The same for the minimizer bins [bin_lo, bin_hi) of the database: (0, 0) = the whole database, bin_hi = 0 = to the
 * end, bin_lo == bin_hi != 0 = an empty slice (a GPU that holds none of this database's bins; pass 4^nt, 4^nt for an
 * empty slice at the start).  A range outside the 4^nt bins gives KUQ_E_INVALID_ARG and leaves the context as it was.
 * With nothing staged yet the range becomes the first database, an empty slice included. */
int kuq_stage_db_append_range(kuq_ctx *ctx, const void *kdb_image, uint64_t kdb_bytes, const void *idx_image,
                              uint64_t idx_bytes, uint64_t bin_lo, uint64_t bin_hi);
/* Runs of the staged databases: maximal groups of consecutive databases with equal (nt, index type).  Each run is one
 * phase of the sharded lookup (kuq_lookup_device_peers_run). */
int kuq_db_runs(kuq_ctx *ctx, uint32_t *n_runs);
/* Distinct taxids stored in the staged records with their record counts — what KrakenDB::count_taxons()
 * (krakendb.cpp:90-113) computes for database.kdb.counts.  Pass cap = 0 to query *n only. */
int kuq_db_taxids(kuq_ctx *ctx, uint32_t *taxid, uint64_t *count, uint32_t cap, uint32_t *n);
/* Optional: the taxids of ALL database records when only a range is staged (other chunks / other GPUs), so that
 * every participant numbers taxa identically.  Must precede the first classify/lookup call. */
int kuq_set_db_taxid_universe(kuq_ctx *ctx, const uint32_t *taxid, uint32_t n);
/* Several databases (`classify -d a -d b`): every k-mer takes the value of the FIRST database that holds the key,
 * even when that value is taxon 0 (classify.cpp:928-936).  With on != 0 the lookup calls report such a stored zero
 * as KUQ_CODE_FOUND_ZERO instead of 0, so that the caller's merge over databases can stop at it; the resolve calls
 * read KUQ_CODE_FOUND_ZERO as 0 in any case.  The caller stages the databases one after the other, runs
 * kuq_lookup_* against each, keeps the first non-zero code per position and hands the result to kuq_resolve_*. */
#define KUQ_CODE_FOUND_ZERO 0xFFFFFFFDu
int kuq_mark_zero_hits(kuq_ctx *ctx, int on);
/* Quick mode, `classify -q [-m min_hits]` (Quick_mode / Minimum_hit_count, classify.cpp:44-45; min_hits = 0 turns it
 * off).  Classification and resolve calls then skip resolve_tree: a read is called as soon as it has min_hits hits.
 *   stop_at_last_hit != 0 — the preloaded path (:943-944,963-964): the read ends at its min_hits-th hit; later
 *     k-mers are neither looked at nor counted; the call is that hit's taxon.  n_windows = windows visited.
 *   stop_at_last_hit == 0 — the -x path (:701-702,705-721,737-738): every k-mer is counted, hits stop counting at
 *     min_hits and the call is the taxon of the read's last unambiguous k-mer (0 if that one missed).
 * Either way run_count[r] (d_run_count) carries the "Q:<hits>" value of the Kraken line (:989-990), no runs are
 * produced (as with KUQ_F_NO_RUNS) and a read with fewer than min_hits hits stays unclassified. */
int kuq_set_quick_mode(kuq_ctx *ctx, uint32_t min_hits, int stop_at_last_hit);

/* ---- taxonomy: Parent_map (taxdb.hpp:383-398): taxid → parent taxid, 0 for the root / unknown parent --------- */
int kuq_set_taxonomy(kuq_ctx *ctx, const uint32_t *taxid, const uint32_t *parent_taxid, uint32_t n);
/* The confidence filter of krakenuniq-filter (scripts/krakenuniq-filter:87-132) on every read of later batches.  taxid /
 * parent are the taxDB rows in file order; they make the script's parent map F: F[t] = p unless p == t, a later row
 * with another parent overwrites, and p = 0 is a parent like any other.  A read's call moves up F until the hits at or
 * below the node (hit taxa whose F-chain passes through it, the node itself included) reach a fraction of at least
 * threshold - 1e-5 of its unambiguous k-mers (misses count); a node without an F entry ends the walk unweighed.
 * Quick mode weighs "Q:<hits>" as hits that lie below no node.  The results come in kuq_batch_result's filtered_call /
 * filter_hits / filter_total; nothing else a batch computes changes.  Call after kuq_set_taxonomy, before the first
 * batch.  KUQ_E_INVALID_ARG for a threshold outside [0, 1]; KUQ_E_TAXONOMY when F has a cycle (the script would never
 * end) or gives taxid 0 a parent (the script divides by zero on reads without unambiguous k-mers). */
int kuq_set_threshold(kuq_ctx *ctx, double threshold, const uint32_t *taxid, const uint32_t *parent, uint32_t n);
/* The read selection of krakenuniq-extract-reads (scripts/krakenuniq-extract-reads:60-127) on every read of later
 * batches.  A read is selected when its Kraken line's taxid (the call, or filtered_call with a threshold) is one of
 * list[0, n_list), or, with KUQ_EXTRACT_SUBTREE, is reachable from one of them through the taxDB's child graph: taxid /
 * parent are the taxDB rows in file order, and every row with taxid != parent is an edge parent -> taxid (a taxid with
 * two rows sits under both parents).  KUQ_EXTRACT_OTHERS (the script's "-1") selects every read that has a Kraken line.
 * KUQ_EXTRACT_CLASSIFIED_ONLY (`classify -c`): reads with call 0 have no line and are never selected.
 * KUQ_EXTRACT_INVERT flips bit 0 of extract_sel, not n_extract.  Results in kuq_batch_result's extract_sel /
 * n_extract; nothing else a batch computes changes.  Call after kuq_set_taxonomy (and kuq_set_threshold, if used),
 * before the first batch.  KUQ_E_TAXONOMY when KUQ_EXTRACT_SUBTREE is given and a cycle of the child graph is
 * reachable from a listed taxon (the script's recursion would never end). */
#define KUQ_EXTRACT_SUBTREE 1u
#define KUQ_EXTRACT_INVERT 2u
#define KUQ_EXTRACT_OTHERS 4u
#define KUQ_EXTRACT_CLASSIFIED_ONLY 8u
int kuq_set_extract(kuq_ctx *ctx, const uint32_t *list, uint32_t n_list, uint32_t flags, const uint32_t *taxid,
                    const uint32_t *parent, uint32_t n_rows);
/* The taxa kuq_set_extract would select (flags: KUQ_EXTRACT_SUBTREE matters), ascending, without a context or a device:
 * *n_out of them, the first cap written to out (cap = 0: count only).  KUQ_E_TAXONOMY on a reachable cycle. */
int kuq_extract_taxa(const uint32_t *list, uint32_t n_list, uint32_t flags, const uint32_t *taxid, const uint32_t *parent,
                     uint32_t n_rows, uint32_t *out, uint32_t cap, uint32_t *n_out);

/* ---- classification, host buffers (the call a user makes) ----------------------------------------------- */
/* bases: concatenated sequences exactly as DNASequence::seq holds them (seqreader.hpp:27-32), read r =
 * bases[read_offsets[r] .. read_offsets[r+1]).  unit_id: work-unit id per read for the HLL mode rule, or NULL to
 * let the library cut units like process_file does (classify.cpp:514-520, continuing across batches).
 * kuq_classify_batch = submit + wait on slot 0. */
int kuq_classify_batch(kuq_ctx *ctx, const char *bases, const uint64_t *read_offsets, uint32_t n_reads,
                       const uint32_t *unit_id, uint32_t flags, kuq_batch_result *out);
int kuq_submit_batch(kuq_ctx *ctx, uint32_t slot, const char *bases, const uint64_t *read_offsets,
                     uint32_t n_reads, const uint32_t *unit_id, uint32_t flags);
int kuq_wait_batch(kuq_ctx *ctx, uint32_t slot, kuq_batch_result *out);
/* The two halves with host buffers, for databases staged range by range (classify -x, classify.cpp:566-791):
 * kuq_lookup_batch    = classify_sequence_with_db_chunk (:1014-1056): per-window DENSE taxon ids of the staged range
 *                       into codes_out (host; indexed like the bases; 0 = no hit in this range, KUQ_CODE_AMBIG for
 *                       ambiguous windows, 0 at positions without a window).  Ranges are merged by the caller with
 *                       an element-wise max (a key hits in at most one range, :447).
 * kuq_resolve_batch   = the final pass (:663-791): calls, hit lists and counters from the merged ids. */
int kuq_lookup_batch(kuq_ctx *ctx, const char *bases, const uint64_t *read_offsets, uint32_t n_reads,
                     uint32_t *codes_out, uint32_t *n_windows_out);
int kuq_resolve_batch(kuq_ctx *ctx, const char *bases, const uint64_t *read_offsets, uint32_t n_reads,
                      const uint32_t *codes_in, const uint32_t *unit_id, uint32_t flags, kuq_batch_result *out);
/* Pinned host memory for callers that want zero-copy staging of their batches. */
void *kuq_host_alloc(uint64_t bytes);
void kuq_host_free(void *p);

/* ---- classification, device buffers (inputs already in HBM) ---------------------------------------------- */
/* d_bases must be 16-byte aligned with 32 readable bytes of slack after the last base (TMA bulk loads fetch
 * whole 16-byte blocks); d_read_offsets (16-byte aligned, n_reads + 2 entries readable) are relative to d_bases.  Asynchronous on the slot's stream;
 * kuq_sync_slot() waits.  d_unit_id: work-unit id of every read (device array) — required with KUQ_HLL_PRELOAD
 * (the per-unit sketches of classify.cpp:525 are what the mode rule is about), NULL otherwise. */
int kuq_classify_device(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                        uint32_t n_reads, uint64_t total_bases, const uint32_t *d_unit_id, uint32_t flags);
/* Stage 1 only (classify_sequence_with_db_chunk): per-window DENSE taxon ids of the staged DB range into
 * d_codes_out (indexed like the bases; 0 where the range has no hit; KUQ_CODE_AMBIG for ambiguous windows).
 * d_codes_out may be peer memory of another GPU (NVLink P2P stores) when only_hits != 0: then only hits are
 * written, so several ranges can be merged into one zero-initialised buffer without a reduction.
 * only_hits = KUQ_LOOKUP_FILL_EMPTY: write hits only, and skip windows whose code in d_codes_out is non-zero already
 * (answered by an earlier database) before any index fetch — the databases after the first of a streamed run of
 * several databases; a stored zero is written as KUQ_CODE_FOUND_ZERO. */
#define KUQ_LOOKUP_FILL_EMPTY 2u
int kuq_lookup_device(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                      uint32_t n_reads, uint64_t total_bases, uint32_t *d_codes_out, uint32_t only_hits);
/* Stage 2 only: calls, hit lists and counters from merged per-window dense ids (the final pass of the chunked
 * mode, classify.cpp:663-791). */
int kuq_resolve_device(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                       uint32_t n_reads, uint64_t total_bases, const uint32_t *d_codes_in,
                       const uint32_t *d_unit_id, uint32_t flags);
/* Fused lookup + scatter for a database sharded by minimizer range over the GPUs of one node: text positions
 * [base_bounds[j], base_bounds[j+1]) belong to the reads GPU j resolves; every hit of the staged range is stored
 * straight into d_codes_peers[j] (that GPU's zero-initialised buffer, mapped with kuq_ipc_open) over NVLink, so no
 * reduction is needed afterwards.  Synchronise the ranks (e.g. a barrier) before the owners call
 * kuq_resolve_device on their buffer. */
int kuq_lookup_device_peers(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                            uint32_t n_reads, uint64_t total_bases, uint32_t *const *d_codes_peers,
                            const uint64_t *base_bounds, uint32_t n_peers);
/* Several databases sharded by minimizer range over the GPUs of a node (`classify -d a -d b` when they fit the GPUs only
 * together).  Every database of a run (kuq_db_runs) holds the same bins [cut_r[g], cut_r[g + 1]) on GPU g: one cut per
 * run over the GPUs.  One call does one run: a window whose bin lies in this GPU's range asks the run's databases in
 * order and the first hit — a stored zero as KUQ_CODE_FOUND_ZERO — is stored into d_codes_peers[j] of the GPU j that
 * resolves the read (text positions [base_bounds[j], base_bounds[j + 1])).  Run 0 writes hits only; a later run first
 * reads the owner's word (a coherent system-scope load) and skips the window when an earlier run answered it on any GPU.
 * Sketches are the owners' business, in the resolve half, so shard counting stays refused (KUQ_E_STATE).
 * Before the first batch every GPU gets kuq_set_db_taxid_universe(taxids of all databases over all ranges), so that all
 * number taxa identically, and kuq_enable_peer_access to every other GPU.  Per batch, with flag arrays as for kuq_lookup_device_peers (done counters and ready counters, one per GPU):
 *     every GPU: the batch into its HBM (all reads: every GPU looks up every window of its ranges)
 *     for r in runs:  every GPU g:  kuq_wait_flags(ready >= step + 1)          when r == 0 (owners cleared the buffers)
 *                                   kuq_wait_flags(done >= step * R + r)       when r > 0  (every GPU finished run r - 1)
 *                                   kuq_lookup_device_peers_run(..., r)
 *                                   kuq_signal_peers(done, step * R + r + 1)
 *     every owner g:  kuq_wait_flags(done >= (step + 1) * R);  kuq_resolve_device(its share, with work-unit ids);
 *                     clear its slice of its buffer;  kuq_signal_peers(ready, step + 3)
 * (R = number of runs, ready starting at 2 with two id buffers alternating by step.)  Shares must hold whole work units:
 * the per-work-unit sketch rule (KUQ_HLL_PRELOAD) decides each unit on the GPU that resolves it.  At the end, kuq_finish
 * on every context and kuq_merge_into the first, as for replicas. */
int kuq_lookup_device_peers_run(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                                uint32_t n_reads, uint64_t total_bases, uint32_t *const *d_codes_peers,
                                const uint64_t *base_bounds, uint32_t n_peers, uint32_t run);
/* Device memory that other ranks can map (cudaMalloc + CUDA IPC); handles are 64 opaque bytes. */
void *kuq_device_alloc(kuq_ctx *ctx, uint64_t bytes);
void kuq_device_free(kuq_ctx *ctx, void *p);
int kuq_device_memset(kuq_ctx *ctx, uint32_t slot, void *p, int value, uint64_t bytes);   /* async on the slot's stream */
int kuq_ipc_export(kuq_ctx *ctx, void *d_ptr, uint8_t handle64[64]);
int kuq_ipc_open(kuq_ctx *ctx, const uint8_t handle64[64], void **d_ptr_out);
int kuq_ipc_close(kuq_ctx *ctx, void *d_ptr);
int kuq_sync_slot(kuq_ctx *ctx, uint32_t slot);
/* Helpers for callers that keep their batches in HBM across several passes (a database streamed in ranges): an
 * asynchronous host → device copy on the slot's stream (pageable memory is fine), the free device memory, and the
 * second half of kuq_classify_batch for device inputs: after kuq_classify_device / kuq_resolve_device on `slot`,
 * kuq_collect_device_batch copies the batch's calls / window counts / hit lists to the slot's pinned host buffers,
 * waits, and fills `out` exactly like kuq_wait_batch. */
int kuq_copy_to_device(kuq_ctx *ctx, uint32_t slot, void *d_dst, const void *h_src, uint64_t bytes);
uint64_t kuq_device_free_bytes(kuq_ctx *ctx);
int kuq_collect_device_batch(kuq_ctx *ctx, uint32_t slot, kuq_batch_result *out);
int kuq_slot_device_result(kuq_ctx *ctx, uint32_t slot, kuq_device_result *out);
/* With KUQ_F_STATS: number of non-ambiguous windows looked up by the slot's last batch and the sum over them of
 * ceil(log2(bin size + 1)) — the textbook probe count SURVEY.md §8(d) defines the algorithmic bytes with. */
int kuq_slot_stats(kuq_ctx *ctx, uint32_t slot, uint64_t *n_lookups, uint64_t *sum_probes);
/* Turn KUQ_F_STATS on / off for every later call, including those that take no flags (kuq_lookup_device_peers). */
int kuq_set_stats(kuq_ctx *ctx, int on);
/* CUDA stream (cudaStream_t) of a slot, so callers can order their own work (e.g. NCCL) against it. */
void *kuq_slot_stream(kuq_ctx *ctx, uint32_t slot);
/* Number of kernels this context has launched so far (for bench.py's gpu_launches). */
uint64_t kuq_launch_count(const kuq_ctx *ctx);
/* Device time in ms of the most recent batch's kernels on `slot` (all stages). */
double kuq_last_kernel_ms(kuq_ctx *ctx, uint32_t slot);
/* Device time in ms of the three stages of the slot's last batch: ms3[0] k_scan (k-mers + minimizers),
 * ms3[1] k_lookup (index + bin search + HLL), ms3[2] k_resolve (hit lists, tree resolution, counters). */
int kuq_last_stage_ms(kuq_ctx *ctx, uint32_t slot, double *ms3);

/* ---- per-taxon results --------------------------------------------------------------------------------- */
/* End of input: closes the open work unit (the flush the reference performs when the reader runs dry). */
int kuq_finish(kuq_ctx *ctx);
/* Number of taxa with a non-zero counter, then their rows sorted by taxid: reads (readCount), kmers (kmerCount)
 * and unique (uniqueKmerCount = ertlCardinality under the configured mode rule, hyperloglogplus.cpp:722-753). */
int kuq_counts_size(kuq_ctx *ctx, uint32_t *n);
int kuq_read_counts(kuq_ctx *ctx, uint32_t *taxid, uint64_t *n_reads, uint64_t *n_kmers, uint64_t *unique,
                    uint8_t *is_sparse, uint32_t cap);
/* Clade roll-up of the report (TaxReport ctor, taxdb.hpp:956-973): sums the counters and merges the sketches
 * of the listed taxa; returns reads / kmers / unique of the union. */
int kuq_clade_counts(kuq_ctx *ctx, const uint32_t *taxids, uint32_t n, uint64_t *n_reads, uint64_t *n_kmers,
                     uint64_t *unique);
/* The same roll-up for many clades in one call: clade(taxids[i]) = that taxon and all its descendants in the taxonomy
 * given to kuq_set_taxonomy (what the TaxReport constructor builds for every node, taxdb.hpp:928-982).  Counters by
 * one pass up the tree; dense clades (a member's sketch is dense: register-wise max, hyperloglogplus.cpp:604-621) by
 * one launch per 8192 clades; sparse clades (union of the members' code sets, :600-603) from ONE sort of the sparse
 * tier's keys by (code, preorder of the taxon) — a subtree is a preorder interval, so its distinct codes are its
 * keys minus the adjacent equal-code pairs whose lowest common ancestor lies inside it.  KUQ_HLL_EXACT: the same
 * identity over the (k-mer, taxon) pairs, from ONE sort of the table (the books of kuq_exact_summary), or from the
 * books summed over the parts once kuq_set_exact_summary installed them.  Results equal kuq_clade_counts() of the
 * member list, clade by clade.  Unknown taxids and taxa without counted descendants give 0. */
int kuq_clade_counts_tree(kuq_ctx *ctx, const uint32_t *taxids, uint32_t n, uint64_t *n_reads, uint64_t *n_kmers,
                          uint64_t *unique);
/* The 4096 p=12 registers of one taxon (all zero if it received no k-mer). */
int kuq_get_registers(kuq_ctx *ctx, uint32_t taxid, uint8_t *regs4096);
int kuq_state_ptrs_get(kuq_ctx *ctx, kuq_state_ptrs *out);
/* KUQ_HLL_PRELOAD: the work units a batch can hold before the (unit, taxon) pairs of further units spill from the
 * dense per-batch table into the per-batch hash map (min(max_bases / work_unit_size + 8, 64 Mi / taxa with a sketch)).
 * A batch of at most this many units only puts candidate pairs into the map, which cannot overflow it.
 * Needs the database and the taxonomy. */
int kuq_unit_table_rows(kuq_ctx *ctx, uint32_t *rows);
/* KUQ_HLL_PRELOAD expects the unit ids of a batch in ascending order (as kuq_*_batch cut them when unit_id is NULL);
 * ids out of order are accepted and give the same results, but each candidate pair then scans the whole batch. */
/* Sparse tier across GPUs (replicas / shards with the exact HLL rule): export the (taxon, encoded hash) keys of the
 * taxa that are still sparse into d_keys_out (HBM; pass NULL / cap 0 to query *n), all-gather them, and import the
 * peers' keys; together with allreduce(MAX) on d_dense_flag / d_regs and SUM on the counters this is the merge
 * `taxon_counts[t] += ...` of classify.cpp:542-544 across processes. */
int kuq_sparse_export(kuq_ctx *ctx, uint64_t *d_keys_out, uint64_t cap, uint64_t *n);
/* The sparse tier's device set: capacity in slots, keys held, how often a harvest re-allocated it, and the device time
 * of the last harvest.  Hits reach the set lazily: the fused lookup only flags the database records it counted (the
 * free top bit of the key word) and kuq_finish / kuq_read_counts / kuq_sparse_export / a re-stage turn the flagged
 * records into (taxon, encoded hash) keys, growing the set first when it would pass a load factor of 0.7. */
int kuq_sparse_tier_info(kuq_ctx *ctx, uint64_t *slots, uint64_t *keys, uint64_t *times_grown, double *last_harvest_ms);
int kuq_sparse_import(kuq_ctx *ctx, const uint64_t *d_keys, uint64_t n);
/* ---- the exact k-mer set (KUQ_HLL_EXACT) ----------------------------------------------------------------------------
 * One open-addressing table of (taxon, canonical k-mer) pairs holds the k-mer sets of all taxa.  Before each batch the
 * library bounds the pairs it could add (one per window); when the bound could take the table past a load factor of 0.8
 * it reads the real fill back, and only when that does not fit either does it re-allocate the table at a load of at most
 * 0.6 (all slots drained first).  A growth that finds no device memory fails with KUQ_E_NOMEM.
 * kuq_exact_info: the table's capacity in slots, the pairs it holds (= the sum of the per-taxon set sizes) and how often
 * it grew.  Not KUQ_HLL_EXACT: 0 slots, 0 pairs. */
int kuq_exact_info(kuq_ctx *ctx, uint64_t *slots, uint64_t *pairs, uint64_t *times_grown);
/* Pair layout of kuq_exact_export / kuq_exact_import: 16 bytes, 16-byte aligned,
 *     { uint64_t kmer_plus_1;    canonical k-mer + 1
 *       uint64_t taxon_plus_1; } dense taxon id + 1 (kuq_dense_taxids numbers them)
 * kuq_exact_export writes every pair of the table to d_pairs_out (HBM, order unspecified; pass NULL / cap 0 to query *n
 * first).  kuq_exact_import inserts pairs into this context's table, growing it first when they need room; a pair the
 * table holds already is not counted again, so importing is set union.  Dense ids only mean the same taxon in two
 * contexts that number their taxa identically: the same database ranges' taxids (kuq_set_db_taxid_universe) and the same
 * taxonomy, which kuq_merge_into checks and callers of these two calls must ensure. */
int kuq_exact_export(kuq_ctx *ctx, void *d_pairs_out, uint64_t cap, uint64_t *n);
int kuq_exact_import(kuq_ctx *ctx, const void *d_pairs, uint64_t n);
/* ---- the exact set partitioned by k-mer over GPUs / processes ---------------------------------------------------------
 * Distinct counts are additive over any partition of the k-mer space: all pairs of one k-mer live in one part, so a
 * taxon's set size and a clade's union size are sums over the parts.  The owner of a canonical k-mer among n_parts
 * parts (1..64) is kuq_exact_owner:
 *     x = kmer ^ 0x2545F4914F6CDD1D;  x ^= x >> 30;  x *= 0xbf58476d1ce4e5b9;  x ^= x >> 27;  x *= 0x94d049bb133111eb;
 *     x ^= x >> 31;                   owner = ((x >> 32) * n_parts) >> 32
 * (splitmix64's finalizer; the table's slot hash is a different function of (k-mer, taxon), so a part never crowds
 * into a subset of a table's slots).  The recipe for G processes (krakenuniq_b200/dist.py, merge_exact_partitioned):
 *   1. all-reduce SUM of the counters (kuq_state_ptrs: n_kmers, n_reads);
 *   2. kuq_exact_export_partitioned(G): the table's pairs grouped by owner, parts back to back, counts[part] pairs each
 *      (NULL / cap 0: counts only); _alloc sizes and allocates the buffer itself (release with kuq_device_free);
 *   3. an all-to-all of the parts (two int64 words per pair);
 *   4. kuq_exact_replace(received pairs): the context's table is rebuilt from them at a load of at most 0.6 (its old
 *      pairs are dropped, duplicates across senders collapse, count[] is recounted); it now holds only its part, and
 *      kuq_clade_counts refuses (KUQ_E_STATE) rather than return a partial union;
 *   5. kuq_exact_summary: the part's per-taxon set sizes ([n_sketch] uint64) and roll-up books ([n_taxa] int64, dense
 *      ids of kuq_dense_taxids) into device buffers → all-reduce SUM → kuq_set_exact_summary.  Until the next batch,
 *      kuq_read_counts' `unique` and kuq_clade_counts_tree then report the union over all parts.
 * books[d] = pairs of taxon d − pairs adjacent in (k-mer, preorder of the taxon) order with one k-mer whose lowest
 * common ancestor is d; summed over a subtree they give the subtree's distinct k-mers (kuq_clade_counts_tree computes
 * them on one context too, with one sort of the pairs in passes over the k-mer space sized to free device memory;
 * KUQ_EXACT_ROLLUP_BUDGET=<bytes> sets the sort's scratch budget, kuq_exact_rollup_passes reports the passes taken).
 * kuq_exact_partition does steps 2–5 for the contexts of one process: pairs move to their owner in rounds over slot
 * ranges with peer copies, each owner builds its part beside its old table (peak per device: old table + part + one
 * round of pairs each way), and the summed summary is installed on ctxs[0].  Step 1 there is kuq_merge_counters_into. */
uint32_t kuq_exact_owner(uint64_t kmer, uint32_t n_parts);
int kuq_exact_export_partitioned(kuq_ctx *ctx, uint32_t n_parts, void *d_pairs_out, uint64_t cap, uint64_t *counts);
int kuq_exact_export_partitioned_alloc(kuq_ctx *ctx, uint32_t n_parts, void **d_pairs_out, uint64_t *counts);
int kuq_exact_replace(kuq_ctx *ctx, const void *d_pairs, uint64_t n);
int kuq_exact_summary(kuq_ctx *ctx, uint64_t *d_count_out, int64_t *d_books_out);
int kuq_set_exact_summary(kuq_ctx *ctx, const uint64_t *d_count, const int64_t *d_books);
int kuq_exact_partition(kuq_ctx *const *ctxs, uint32_t n);
int kuq_exact_rollup_passes(kuq_ctx *ctx, uint32_t *passes);
/* ---- the exact set spilled to host memory by k-mer part ---------------------------------------------------------------
 * kuq_set_exact_spill(ctx, bytes > 0): when the table cannot grow before a batch (no device memory, or
 * KUQ_EXACT_MAX_SLOTS), its pairs move to host memory instead of the batch failing with KUQ_E_NOMEM.  They go in rounds
 * over slot ranges (KUQ_EXACT_MERGE_SLOTS, as kuq_merge_into) through a bounded device buffer and a pinned one, grouped
 * into the 64 parts of kuq_exact_owner(kmer, 64); the table is emptied and takes the batch at the same capacity (an
 * empty table that cannot take a batch's bound of one pair per window fails with KUQ_E_NOMEM).  The budget bounds the
 * bytes of spilled pairs (16 each) held by all contexts of the process together: a spill that would pass it fails with
 * KUQ_E_NOMEM.  0 (the default) turns spilling off.
 * kuq_exact_spill_info: the times the table spilled since the last kuq_reset_counts, and the pairs held on the host now.
 * From a context's first spill until kuq_exact_settle, every readout that would see a part of its set refuses with
 * KUQ_E_STATE: kuq_read_counts, kuq_clade_counts, kuq_clade_counts_tree, kuq_exact_export, kuq_exact_export_partitioned*,
 * kuq_exact_summary, kuq_exact_partition and the set union of kuq_merge_into (kuq_merge_counters_into still works).
 * kuq_exact_settle(ctxs, n >= 1): every context spills what its table still holds (under its budget too); the parts of
 * all contexts are cut into groups of consecutive parts that fit a table (a table smaller than the largest grows to it
 * first where its device keeps room beside it for a round and the roll-up's sort), and one host thread per context imports each of its groups into its emptied table in rounds —
 * duplicates from successive spills and from other contexts collapse — and sums the group's set sizes and roll-up books
 * (kuq_exact_summary).  The sums are installed on ctxs[0] as kuq_set_exact_summary does; the host parts are freed and
 * their bytes return to the budget.  A part whose pairs do not fit any table even with their duplicates collapsed fails
 * with KUQ_E_NOMEM.  A failed settle keeps every host part (the contexts stay spilled), so it can run again.  Round
 * buffers halve until they fit a full card.  The counters join ctxs[0] by kuq_merge_counters_into.  kuq_reset_counts drops the host parts. */
int kuq_set_exact_spill(kuq_ctx *ctx, uint64_t host_budget_bytes);
int kuq_exact_spill_info(kuq_ctx *ctx, uint64_t *spills, uint64_t *pairs_on_host);
int kuq_exact_settle(kuq_ctx *const *ctxs, uint32_t n);
/* ---- database sharded by minimizer range over the GPUs of a node (SURVEY.md §8(e).2) ------------------------------
 * Who counts: with kuq_set_shard_counting(on) the GPU that FINDS a hit does that hit's sketch work inside the lookup
 * half (kuq_lookup_device / kuq_lookup_device_peers): HLL register update and the record flag behind the sparse tier;
 * the resolve half on the GPU that owns the read then only adds the misses (taxon 0), the counters and the per-unit
 * bookkeeping.  Only valid when every looked-up window is counted exactly once (one database, no quick mode). */
int kuq_set_shard_counting(kuq_ctx *ctx, int on);
/* Step flags instead of host barriers.  A flag array is device memory of 8-byte counters that every peer has mapped
 * (kuq_device_alloc + kuq_ipc_export/open).  kuq_signal_peers: in stream order on the slot — i.e. after everything
 * queued before it, peer stores included, is complete — store `value` into d_flag_peers[j][my_index] for every
 * peer j (system-scope fence first).  kuq_wait_flags: in stream order, spin until d_flags[0..n) >= value; after
 * timeout_ms (0 → 20 s) it gives up and the next kuq_sync_slot returns KUQ_E_STATE instead of hanging the GPU. */
int kuq_signal_peers(kuq_ctx *ctx, uint32_t slot, uint64_t *const *d_flag_peers, uint32_t n_peers, uint32_t my_index,
                     uint64_t value);
int kuq_wait_flags(kuq_ctx *ctx, uint32_t slot, const uint64_t *d_flags, uint32_t n, uint64_t value, uint32_t timeout_ms);
/* End-of-run merge of the sparse tier across GPUs in O(keys / GPUs) per GPU (replicas or shards): the keys of the
 * still-sparse taxa are grouped by the GPU that owns their CODE (hash(code) % n_parts; counts[j] keys for part j,
 * parts stored back to back in d_keys_out; pass d_keys_out = NULL to get the counts only), exchanged with one
 * all-to-all, and kuq_sparse_replace makes the received keys this GPU's set (duplicates collapse there).  The export
 * covers the local set and the database records flagged since the last harvest; with a buffer it CONSUMES those
 * flags (their keys exist only in the buffer afterwards), so it must be followed by kuq_sparse_replace.  Every key
 * that can duplicate another — the same (taxon, code) from two GPUs, the same code under two taxa of a clade — lands
 * on one GPU, so global per-taxon numbers are SUMS: kuq_sparse_summary writes this GPU's rank histograms
 * ([n_sketch][64] uint32) and distinct counts ([n_sketch] uint32) to device buffers for an all-reduce(SUM), and
 * kuq_set_sparse_summary installs the sums, which kuq_read_counts then reports (until the next batch).  Clade
 * unions of several sparse taxa: sum kuq_clade_partial's hist64 over the GPUs and evaluate kuq_ertl_sparse /
 * kuq_ertl_dense_hist (is_dense is the same on every GPU once dense flags and registers were all-reduced). */
int kuq_sparse_export_partitioned(kuq_ctx *ctx, uint32_t n_parts, uint64_t *d_keys_out, uint64_t cap, uint64_t *counts);
/* the same with the buffer sized and allocated by the library after its counting pass (release with kuq_device_free) */
int kuq_sparse_export_partitioned_alloc(kuq_ctx *ctx, uint32_t n_parts, uint64_t **d_keys_out, uint64_t *counts);
int kuq_sparse_replace(kuq_ctx *ctx, const uint64_t *d_keys, uint64_t n);
int kuq_sparse_summary(kuq_ctx *ctx, uint32_t *d_hist_out, uint32_t *d_distinct_out);
int kuq_set_sparse_summary(kuq_ctx *ctx, const uint32_t *d_hist, const uint32_t *d_distinct);
int kuq_clade_partial(kuq_ctx *ctx, const uint32_t *taxids, uint32_t n, uint64_t *n_reads, uint64_t *n_kmers, int *is_dense,
                      uint32_t *hist64);
uint64_t kuq_ertl_sparse(const uint32_t *hist64, uint64_t n_observed);
uint64_t kuq_ertl_dense_hist(const uint32_t *hist64, uint64_t n_observed);
/* Stage 1 alone (KmerScanner + canonical_representation + bin_key, krakenutil.cpp:239-282, krakendb.cpp:200-246) on
 * device buffers: canonical k-mer and minimizer bin of every window, indexed like the bases (window i of read r at
 * d_read_offsets[r] + i; bins: 0xFFFFFFFE = ambiguous window, 0xFFFFFFFF = no window at this position).  Needs no
 * staged database; used by the database-build tools and the synthetic-workload generator. */
int kuq_scan_device(kuq_ctx *ctx, uint32_t slot, uint32_t k, uint32_t nt, uint32_t idx_type, const char *d_bases,
                    const uint64_t *d_read_offsets, uint32_t n_reads, uint64_t total_bases, uint64_t *d_canon_out,
                    uint32_t *d_bins_out);

/* ---- a database larger than HBM, streamed range by range (classify -x / --preload-size, krakendb.cpp:411-526) ------
 * kuq_stage_db replaces the staged range synchronously.  The stream calls keep TWO device buffers and a copy stream, so
 * the next minimizer range travels over PCIe while the lookups of the current one run:
 *     kuq_set_db_taxid_universe(all taxids of the database); kuq_set_taxonomy(...);
 *     kuq_stream_open(k, nt, idx_type, max records / bins of a range)
 *     kuq_stream_load(0, range 0)
 *     for r in ranges:  kuq_stream_use(r & 1);  kuq_stream_load((r + 1) & 1, range r + 1);      // order matters
 *                       kuq_lookup_device(... only_hits = 1 ...) for every batch, ids merged in the caller's buffers
 *     kuq_resolve_device(...) for every batch                                  // the final pass (classify.cpp:663-791)
 * host_records = the range's records (key_len + 4 bytes each for the k given to kuq_stream_open: 12 for k = 29..31; raw
 * taxids; as in database.kdb), host_offsets = the bin_hi -
 * bin_lo + 1 cumulative ABSOLUTE record offsets of its bins (a slice of database.idx); both should be pinned
 * (kuq_host_alloc / kuq_host_register) or the copy will not overlap.  kuq_stream_load waits, on the device, for the
 * work queued on the slots so far (the users of the buffer it overwrites), never for the host.  Record values are
 * rewritten to dense ids on arrival; kuq_stream_check reports a taxid outside the declared universe.  The buffers hold
 * max_records records of 12 bytes; records shorter than that (k <= 28) are widened on arrival, in pieces that pass
 * through one landing zone of 64 MiB (KUQ_LANDING_BYTES) on the copy stream.  kuq_stream_open may be called again once
 * the slots are idle (it waits for them): the next database of a streamed run may have another nt or index type.
 * Several GPUs of a node (one context each, the same universe and taxonomy, kuq_enable_peer_access between all of them):
 * GPU g streams a contiguous group of the ranges, every GPU holds every batch, and each batch has one owner whose
 * zero-initialised id buffer takes every GPU's hits (a peer pointer for the others):
 *     the owners zero their buffers; host barrier
 *     for each database d, in command-line order:
 *         every GPU g at once: the loop above over g's group of d's ranges, kuq_lookup_device(... owner's buffer,
 *                              only_hits = d == 0 ? 1 : KUQ_LOOKUP_FILL_EMPTY);  kuq_sync_slot(0), (1);  kuq_stream_check
 *         host barrier — KUQ_LOOKUP_FILL_EMPTY reads the owner's word with a plain load, which sees another GPU's stores
 *         only once that GPU has finished and a new launch has begun
 *     every owner: kuq_resolve_device(...) for its batches; at the end kuq_finish on every context and kuq_merge_into
 * kuq_host_register pins with cudaHostRegisterPortable, so one registered mapping counts as pinned for every device and
 * every GPU's copies from it overlap its lookups.
 * kuq_stream_close releases the two range buffers and the landing zone once the slots are idle (it waits for them),
 * so that their device memory serves other work between passes: the taxa numbering stays, kuq_resolve_device keeps
 * resolving ids looked up before, and kuq_stream_load refuses (KUQ_E_STATE) until the next kuq_stream_open. */
int kuq_stream_open(kuq_ctx *ctx, uint32_t k, uint32_t nt, uint32_t idx_type, uint64_t max_records, uint64_t max_bins);
int kuq_stream_load(kuq_ctx *ctx, uint32_t buf, const void *host_records, uint64_t n_records, const uint64_t *host_offsets,
                    uint64_t bin_lo, uint64_t bin_hi);
int kuq_stream_use(kuq_ctx *ctx, uint32_t buf);
int kuq_stream_check(kuq_ctx *ctx);
int kuq_stream_close(kuq_ctx *ctx);
/* Pin / unpin caller memory (e.g. an mmap'ed database.kdb) for asynchronous copies. */
int kuq_host_register(void *p, uint64_t bytes);
int kuq_host_unregister(void *p);

/* Several GPUs in one process (what the drop-in `classify` does when it sees more than one device: every GPU holds the
 * database, batches go round-robin): fold the per-taxon state of `src` into `dst` — counters add, registers max, dense
 * anywhere = dense, sparse-tier keys united (classify.cpp:542-544 across devices; cudaMemcpyPeer, no NCCL).  Both
 * contexts must have been given the same database and taxonomy.  `src` keeps its state. */
int kuq_merge_into(kuq_ctx *dst, kuq_ctx *src);
/* kuq_merge_into without the sets: counters add, registers max, dense flags or; the sparse-tier keys and the exact
 * pairs stay where they are (the partitioned merges move them: kuq_exact_partition, kuq_sparse_export_partitioned). */
int kuq_merge_counters_into(kuq_ctx *dst, kuq_ctx *src);
/* In one process the GPUs of a sharded database need no CUDA IPC: after kuq_enable_peer_access(ctx, peer) the device
 * pointers of `peer` (kuq_device_alloc) can be handed to kuq_lookup_device_peers / kuq_signal_peers of `ctx` as they are. */
int kuq_enable_peer_access(kuq_ctx *ctx, kuq_ctx *peer);

/* Dense id ↔ taxid tables (n_taxa entries) for callers that exchange dense ids between GPUs. */
int kuq_dense_taxids(kuq_ctx *ctx, uint32_t *taxid_of_dense, uint32_t cap, uint32_t *n);
/* Start a new run on the staged database(s): afterwards the context gives the same results for any later batches and
 * readouts as a context that was just staged and given the same taxonomy and quick-mode settings (one staging serves
 * many samples, `classify --sample-sheet`).  Cleared: registers, dense flags, per-taxon k-mer and read counters, the
 * sparse-tier set (keys, used counter) and the exact k-mer set, the summaries and partitions installed by
 * kuq_set_sparse_summary / kuq_set_exact_summary / kuq_exact_partition, the SEEN and KEPT bits of every staged record
 * (one streaming pass over the records, skipped when no record can carry one), the open work unit and the host
 * snapshot.  Kept, being functions of the staged database alone: the records, the collision table of the record tier
 * and the grown table capacities (results do not depend on table size).  All slots must be idle. */
int kuq_reset_counts(kuq_ctx *ctx);

/* Host-side estimator (no device needed): ertlCardinality over 4096 dense registers (hyperloglogplus.cpp:
 * 730-752) — exported so bindings and tests can call the exact code the report path uses. */
uint64_t kuq_ertl_dense(const uint8_t *regs4096, uint64_t n_observed);

/* ---- measurement aid: the random-access roofline of SURVEY.md §8(d) ------------------------------------------- */
/* Random 32-byte-sector gather ceiling of the device's HBM: a kernel with k_lookup's launch shape (256 threads,
 * 8 CTAs per SM) issues independent loads at hashed sector addresses of a freshly allocated buffer of buffer_bytes
 * (use several GB: far beyond L2) until n_sectors_to_read sectors were touched; bytes_per_access = 32 (whole
 * sector) or 8 (one word of it — the sector is still what HBM moves).  Best of three timed launches after one
 * warm-up, CUDA events.  Returns sectors/s (in 1e9) and the same as GB/s of 32-byte sectors.  Needs no context. */
int kuq_random_gather_peak(int device, uint64_t buffer_bytes, uint64_t n_sectors_to_read, uint32_t bytes_per_access,
                           double *gsectors_per_s, double *gbytes_per_s, double *kernel_ms);

/* ---- test aid: the record-tier harvest on caller-owned device buffers ------------------------------------------ */
/* The harvest kuq_finish runs on a resident range, on device memory the caller owns: n_rec 12-byte records at d_pairs
 * (4-byte aligned), n_secondaries (secondary, primary) record index pairs (2 x u32 each), d_dense_flag[n_sketch]; record taxa < n_sketch.
 * Flagged secondaries hand their flag to their primaries; then every flagged record that is neither kept nor of a dense
 * taxon becomes kept and adds 1 to d_distinct[taxon] and to *d_n_kept; every flag is cleared.  Synchronous. */
int kuq_harvest_keep_device(int device, void *d_pairs, uint64_t n_rec, const void *d_secondaries, uint64_t n_secondaries,
                            const uint8_t *d_dense_flag, uint32_t n_sketch, uint32_t *d_distinct, uint64_t *d_n_kept);

/* Record-layout / search-shape experiment for the bin search (kmer_query, krakendb.cpp:250-321) — measurement aid.
 * Transcodes the staged 12-byte records once into 8-byte minimizer-relative records (the 16 bases outside the bin's
 * minimizer + minimizer position / orientation + 24-bit dense taxon; k = 31, m = 15 only) and times a lookup-only
 * kernel over the windows the LAST batch of `slot` left in the slot's scratch (text positions [0, n_positions), i.e.
 * a batch whose first read starts at offset 0), for both layouts x {4, 8, 16}-ary narrowing x final scans of <= 8 /
 * <= 16 records.  Every variant's per-window dense ids are compared with the ids the product's k_lookup wrote for
 * that batch (mismatches[] must be 0).  On the product's layout and search it also times other launch SHAPES:
 * shape 0 = thread per window with the next window's scratch prefetched (the product's), 1 = the product's own
 * k_lookup<MODE_LOOKUP> in the same harness, 2 / 3 = the next window's index entry prefetched too (8 / 6 CTAs per SM),
 * 4 / 5 / 6 = two windows per thread in lock step (8 / 6 / 4 CTAs per SM), 7 = four windows per thread (4 CTAs),
 * 8 = the product's k_lookup<MODE_LOOKUP> with its launch-uniform switches compiled out, 9 / 10 = the product's
 * k_lookup<MODE_FUSED> (search + register update) with / without those switches — these two run only on a
 * KUQ_HLL_DENSE_ONLY context (they count the batch's windows into its sketches once per launch; use a throwaway
 * context) and are reported as 0 ms otherwise; 11 = shape 0 with the narrowing step as an if / else-if chain instead
 * of a count of the pivots <= key, 12 = shape 0 fed through the product's parameter block, 13 = shape 0 with the
 * first round's pivots loaded with the L2::256B prefetch-size qualifier, 14 / 15 = shape 0 on a copy of the records
 * with every bin laid out as a two-level search tree (its pivots at the bin's head, then the leaves in key order;
 * tree_ms times the copy, tree_unordered counts bins whose keys do not strictly increase) with the tree's header
 * loaded plainly / with the L2::256B qualifier.
 * Needs 20 bytes per record + 4 bytes per position of free device memory.
 * Times: CUDA events on the slot's stream, one warm-up launch then `reps` timed ones per variant. */
#define KUQ_LAYOUT_VARIANTS 25
typedef struct kuq_layout_result {
  uint64_t n_records, n_positions;
  uint64_t n_windows;                         /* windows looked up in the staged range */
  uint64_t sum_probes;                        /* sum of ceil(log2(bin size + 1)) over them (SURVEY.md §8(d)'s P) */
  uint64_t bin_class[6];                      /* windows whose bin holds <= 8, <= 16, <= 64, <= 256, <= 1024, more records */
  double transcode_ms;
  uint32_t n_variants;
  uint32_t rec_bytes[KUQ_LAYOUT_VARIANTS], arity[KUQ_LAYOUT_VARIANTS], window[KUQ_LAYOUT_VARIANTS];
  uint32_t shape[KUQ_LAYOUT_VARIANTS];        /* see below */
  double best_ms[KUQ_LAYOUT_VARIANTS], mean_ms[KUQ_LAYOUT_VARIANTS];
  uint64_t mismatches[KUQ_LAYOUT_VARIANTS];
  double tree_ms;
  uint64_t tree_unordered;
} kuq_layout_result;
int kuq_layout_experiment(kuq_ctx *ctx, uint32_t slot, uint64_t n_positions, uint32_t reps, kuq_layout_result *out);

/* ---- database build (SURVEY.md §8 f4) ---------------------------------------------------------------------- */
/* db_sort [-z] -n nt (db_sort.cpp:41-116 + KrakenDB::make_index, krakendb.cpp:118-148): unsorted Jellyfish-style
 * image → database.kdb image (kdb_out: header + key_ct * (key_len + 4) bytes) and KRAKIX2 index image (idx_out:
 * 8 + 8 * (4^nt + 1) bytes).  Needs no context.  err (optional) receives a message on failure.
 * kuq_db_sort = kuq_db_sort_budget with budget 0. */
int kuq_db_sort(int device, const void *jdb_image, uint64_t jdb_bytes, uint32_t nt, int zero_vals, void *kdb_out,
                void *idx_out, char *err, uint64_t err_cap);
/* db_sort within `budget` bytes of device memory (0 → environment variable KUQ_DB_SORT_BUDGET, else 3/4 of the free
 * device memory).  When the one-piece working set (about 2 * (key_len + 4) + 60 bytes per record plus 8 * (4^nt + 1)
 * for the index) does not fit, the sort runs in passes over the two host images: the input streams through the device
 * twice (bin histogram → index; grouping by minimizer range into the output image), then every range is sorted in
 * place.  The result is the same bytes; PCIe carries about five times the database.  *n_passes (optional) = 1 for the
 * one-piece sort, else the number of ranges.  KUQ_E_CAPACITY when the index or one minimizer bin does not fit. */
int kuq_db_sort_budget(int device, const void *jdb_image, uint64_t jdb_bytes, uint32_t nt, int zero_vals, uint64_t budget,
                       void *kdb_out, void *idx_out, uint32_t *n_passes, char *err, uint64_t err_cap);
/* db_sort on several devices: kuq_db_sort_budget is its one-device case.  A sort that fits devices[0] in one piece runs
 * there alone.  Otherwise every entry of devices[0, n_devices) is a worker (an ordinal may repeat: several workers on
 * one card), each with its own stream and pinned bounce buffers and `budget` bytes of its device's memory (0 →
 * KUQ_DB_SORT_BUDGET, else 3/4 of the device's free memory shared among the workers on it; the smallest share is every
 * worker's).  The ranges are planned from that budget as on one device, so the plan does not depend on n_devices:
 *   A. worker w streams the contiguous slice [n * w / G, n * (w + 1) / G) of the records for its bin histogram and
 *      keeps its running sum on the device; the index is the sum over the slices;
 *   cursors: a kernel on each device reduces the slice's counts over the ranges' bins; range r's records are laid out
 *      slice after slice, so that they keep input order;
 *   B. every worker groups its slice by range into the output image at its own cursors;
 *   C. the ranges, split into contiguous groups (one per worker), are sorted in place.
 * Workers write disjoint bytes of the host images; no peer access is needed.  The result is the bytes of the one-device
 * sort. */
int kuq_db_sort_devices(const int *devices, uint32_t n_devices, const void *jdb_image, uint64_t jdb_bytes, uint32_t nt,
                        int zero_vals, uint64_t budget, void *kdb_out, void *idx_out, uint32_t *n_passes, char *err,
                        uint64_t err_cap);
/* set_lcas (set_lcas.cpp:429-476): for every k-mer of the library pieces that the staged database holds,
 * value = lca(taxid of the piece, value).  A piece is a stretch of one library sequence; consecutive pieces of a
 * sequence overlap by k-1 bases (the reference's SKIP_LEN pieces, :363-364).  The context needs the database
 * (kuq_stage_db) and the taxonomy (kuq_set_taxonomy); every taxid must be in the taxonomy — the reference
 * skips other sequences (:336-341) and so must the caller.  *n_missing = k-mers of this batch the database lacks (set_lcas
 * without -x stops there, :441-443).  After the first call the context cannot classify any more.
 * With a minimizer range [bin_lo, bin_hi) staged, only the k-mers whose bin lies in the range are looked up; the others
 * are neither updated nor counted as missing.  A database larger than HBM is built range by range: declare the taxids
 * of all its records (kuq_set_db_taxid_universe) before the taxonomy, then per range kuq_stage_db, the same batches in
 * the same order, kuq_export_db_values; the missing counts of the ranges add up to the one-piece count.
 * flags: KUQ_LCA_FORCE_CONTAMINANT = set_lcas -T (what build_db.sh always passes: a value of 32630 'synthetic
 * construct' / 81077 'artificial sequences' sticks and a piece with such a taxid overwrites instead of taking the LCA,
 * :462-474; between those two taxids the first to arrive wins, so one batch may hold pieces of only one of them),
 * KUQ_LCA_RESET = -R (the value becomes 0, :458-459). */
#define KUQ_LCA_FORCE_CONTAMINANT 1u
#define KUQ_LCA_RESET 2u
int kuq_set_lcas_batch(kuq_ctx *ctx, const char *bases, const uint64_t *piece_offsets, uint32_t n_pieces,
                       const uint32_t *taxid, uint32_t flags, uint64_t *n_missing);
/* Copy the record values of the staged database (as taxids) into the value fields of a host database.kdb image
 * with the same records — what set_lcas leaves in the memory-mapped file.  Values are written at the file's record
 * stride (key_len + 4 bytes), whatever the staged layout.  A staged range writes only its own records, at their
 * positions in the file. */
int kuq_export_db_values(kuq_ctx *ctx, void *kdb_image, uint64_t kdb_bytes);
/* Records of the staged database (or range) per value, as taxids, value 0 included: what KrakenDB::count_taxons
 * (krakendb.cpp:90-113) writes to database.kdb.counts, for the values as they are now (kuq_db_taxids reports them as
 * staged).  Ascending by taxid, taxids with no record left out; cap = 0 queries *n only.  Once the context has numbered
 * its taxa (after the first kuq_set_lcas_batch or classification) one pass over the records in HBM counts them by dense
 * id; before that the values are those staging counted.  KUQ_E_STATE with appended databases. */
int kuq_db_value_counts(kuq_ctx *ctx, uint32_t *taxid, uint64_t *count, uint32_t cap, uint32_t *n);

/* k-mer set of a FASTA library: step 1 of build_db.sh (scripts/build_db.sh:116-147), `jellyfish count -m k -C` of
 * Jellyfish 1, whose output database_0 becomes database.jdb.  The set holds one record per distinct canonical k-mer
 * (canonical_representation, krakendb.cpp:238-246) of the windows KmerScanner (krakenutil.cpp:239-282) yields over each
 * sequence: key_len(k) = ceil(2k / 8) little-endian key bytes + the u32 number of occurrences (saturated at 2^32 - 1),
 * the records of database.kdb.  Records come in ascending key order; Jellyfish writes them in hash order, which only
 * db_shrink depends on.  Needs no context.
 *
 * kuq_kmer_set_create: device ordinal, k = 1..31, budget = bytes of HBM for the packed library and one pass over a
 *   range of k-mers (0 → environment variable KUQ_KMER_SET_BUDGET, else 3/4 of the free device memory).  Batches of
 *   KUQ_KMER_SET_BATCH bases (default 256 Mi) are staged through two pinned buffers; their device buffers come on top
 *   of the budget until the first kuq_kmer_set_next / _info.  err (optional) receives a message on failure.
 * kuq_kmer_set_add: sequences r = bases[offsets[r] .. offsets[r + 1]) — what FastaReader::next_sequence
 *   (seqreader.cpp:34-79) returns; any letter but ACGTacgt makes its windows ambiguous, windows never cross sequences,
 *   and a '\n' / '\r' (CRLF files) is left out of the k-mers but costs the window KmerScanner then skips
 *   (krakenutil.cpp:265-269; sequences holding them take a slower host path).  Copies the bases; asynchronous on the device, so the caller can
 *   parse the next batch while this one is packed.  A sequence longer than a batch is cut into pieces overlapping by
 *   k - 1 bases (set_lcas.cpp:363-364), which keeps the multiset of windows.
 * kuq_kmer_set_next: up to cap_records records into records_out (cap_records * (key_len + 4) bytes), continuing in
 *   ascending key order; *n_out = 0 at the end.  The first call plans the passes from a histogram of the top 16 key
 *   bits (KUQ_E_CAPACITY when one histogram bucket alone exceeds a pass under the budget); every pass extracts, sorts and
 *   collapses one range of keys, so the whole set never sits in host memory.
 * kuq_kmer_set_info: *key_ct = records produced so far (the set's size once kuq_kmer_set_next returned 0 records),
 *   *n_passes = planned passes.
 * kuq_kmer_set_stats (measurement aid): device time in ms of the stages so far — [0] pack + histogram, [1] extract,
 *   [2] sort, [3] collapse, [4] record copy to the host —, the number of windows, the planner's estimate of the device
 *   bytes a pass needs (library included), the measured drop of free device memory at the passes' peak, and whether the
 *   packed library is in HBM (1) or pinned host memory (0). */
typedef struct kuq_kmer_set kuq_kmer_set;
int kuq_kmer_set_create(int device, uint32_t k, uint64_t budget, kuq_kmer_set **out, char *err, uint64_t err_cap);
int kuq_kmer_set_add(kuq_kmer_set *h, const char *bases, const uint64_t *offsets, uint32_t n_seqs);
int kuq_kmer_set_next(kuq_kmer_set *h, void *records_out, uint64_t cap_records, uint64_t *n_out);
int kuq_kmer_set_info(kuq_kmer_set *h, uint64_t *key_ct, uint32_t *n_passes);
int kuq_kmer_set_stats(kuq_kmer_set *h, double *stage_ms5, uint64_t *windows, uint64_t *ws_estimate_bytes,
                       uint64_t *peak_bytes, int *lib_on_device);
const char *kuq_kmer_set_last_error(const kuq_kmer_set *h);
void kuq_kmer_set_destroy(kuq_kmer_set *h);

/* Distinct k-mers of a FASTA library by HyperLogLog: count_unique (src/count_unique.cpp:51-79), which
 * krakenuniq-build runs when --jellyfish-hash-size is not given (scripts/build_db.sh:125-129).  Every sequence is cut
 * into pieces [i, i + 50000 + k - 1), i = 0, 50000, ...; a fresh KmerScanner (krakenutil.cpp:208-282) runs over each,
 * and every window whose k bases are ACGTacgt goes into a dense HyperLogLog sketch of 2^p registers as its forward
 * (not canonical) 2-bit k-mer: hash = murmur3 finalizer, register = top p bits, rank = leading zeros of the rest + 1
 * (hyperloglogplus.cpp:485-523).  Pieces merge by register max; n_observed counts every valid window of every piece.
 * Needs no context.
 *
 * kuq_count_unique_create: device ordinal, k = 1..31, precision p = 4..18 (KUQ_E_INVALID_ARG otherwise), batch_bases =
 *   bases per staged batch (0 → 256 Mi), staged through two pinned buffers.  err (optional) receives a message on
 *   failure; KUQ_E_NO_DEVICE without a GPU (there is no CPU path).
 * kuq_count_unique_add: sequences r = bases[offsets[r] .. offsets[r + 1]) — what FastaReader::next_sequence
 *   (seqreader.cpp:34-79) returns, a '\r' of CRLF files included.  The library cuts the pieces; a '\n' / '\r' is left
 *   out of the k-mers but costs the window KmerScanner then skips, and near a piece's end the scanner may read into the
 *   next piece, which can count a window twice in n_observed (sequences holding them take a slower host path).  Copies
 *   the bases; asynchronous on the device.  May be called again after kuq_count_unique_result.
 * kuq_count_unique_result: *estimate = what count_unique prints, ertlCardinality (hyperloglogplus.cpp:722-753) at p:
 *   n_observed when that is below the estimate, else the rounded estimate, and 0 when no window was valid;
 *   *n_observed = valid windows; regs_out (optional, 2^p bytes) = the registers.
 * kuq_count_unique_stats (measurement aid): device time in ms of the sketch kernel so far, valid windows as of the last
 *   kuq_count_unique_result, and bases staged (line breaks left out). */
typedef struct kuq_count_unique kuq_count_unique;
int kuq_count_unique_create(int device, uint32_t k, uint32_t p, uint64_t batch_bases, kuq_count_unique **out, char *err,
                            uint64_t err_cap);
int kuq_count_unique_add(kuq_count_unique *h, const char *bases, const uint64_t *offsets, uint32_t n_seqs);
int kuq_count_unique_result(kuq_count_unique *h, uint64_t *estimate, uint64_t *n_observed, uint8_t *regs_out);
int kuq_count_unique_stats(kuq_count_unique *h, double *sketch_ms, uint64_t *windows, uint64_t *bases);
const char *kuq_count_unique_last_error(const kuq_count_unique *h);
void kuq_count_unique_destroy(kuq_count_unique *h);

#ifdef __cplusplus
}
#endif
#endif /* KUQ_H */
