/*
 * fgumi_b200.h — C-ABI of the H100-native UMI-consensus engine.
 *
 * This is the drop-in boundary for fgumi's consensus hot path.  The reference (fgumi 0.2.0,
 * pure Rust, `#![deny(unsafe_code)]`) has no FFI; its only boundary is the trait
 *     crates/fgumi-consensus/src/caller.rs:205-234   trait ConsensusCaller
 *         fn consensus_reads(&mut self, records: Vec<RawRecord>) -> Result<ConsensusOutput>
 * whose per-family inner loops are
 *     vanilla_caller.rs:1260-1358  create_consensus_from_source_reads   -> fgb_vote_* / fgb_submit
 *     base_builder.rs:295-458      ConsensusBaseBuilder::{add,call}      -> (inside the vote kernel)
 *     duplex_caller.rs:838-1015    DuplexConsensusCaller::duplex_consensus -> fgb_duplex_combine_*
 *     codec_caller.rs:1029-1212    build_duplex_consensus_from_padded +
 *                                  mask_consensus_quals_query_based      -> fgb_codec_combine_*
 *     caller.rs:238-286            ConsensusCallingStats                 -> fgb_stats
 * A Rust maintainer binds these entry points with a `extern "C"` block behind a
 * `ConsensusCaller` impl (INTEGRATION.md shows the stub).  Everything here is plain pointers
 * and sizes; no C++/torch types cross the boundary.  Errors are status codes — no exceptions,
 * no aborts across the ABI (anyhow::Error maps to a non-zero fgb_status + fgb_last_error()).
 *
 * Data model ("SoA base/qual byte columns with per-family offsets"):
 *   unit   = one sub-family = one consensus read (Fragment / R1 / R2 of an MI group;
 *            vanilla_caller.rs:1124 process_subgroup).  Its reads are the SourceRead rows
 *            (vanilla_caller.rs:129-146) AFTER host prep: oriented, quality-masked, clipped,
 *            CIGAR-filtered, in reference order (order matters: the f64 Kahan vote is
 *            order-dependent, base_builder.rs:312-324).
 *   bases[], quals[]  two byte columns; read r occupies bytes
 *            [off_r, off_r+len_r) of BOTH columns, off_r % FGB_READ_ALIGN == 0, len_r >= 1,
 *            rows ascending and non-overlapping.
 *   reads[r] = FGB_READ_DESC(off_r, len_r); reads of a unit are consecutive.
 *   units[u] = {out_off, read_begin, cons_len}; units[U] is a sentinel
 *            {n_out, n_reads, 0}.  cons_len = min_reads-th longest read
 *            (vanilla_caller.rs:1269-1277), out_off % FGB_OUT_ALIGN == 0.
 *   tiles[t] = a run of consecutive units that fits one shared-memory stage; produced by
 *            fgb_plan_tiles() — part of the packed batch, like the offsets.
 *   output   four columns cons_base/cons_qual (u8) and cons_depth/cons_errors (u16); unit u
 *            owns elements [out_off, out_off+cons_len).
 */
#ifndef FGUMI_B200_H
#define FGUMI_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FGB_ABI_VERSION 4
#define FGB_READ_ALIGN 8u   /* byte alignment of every read row in bases[]/quals[]          */
#define FGB_OUT_ALIGN 8u    /* element alignment of every unit's output row                 */
#define FGB_MAX_READ_LEN 65535u
#define FGB_MAX_PHRED 93u   /* phred.rs:28 */
#define FGB_NTABLE 94u      /* tables are indexed by input quality 0..=93, base_builder.rs:258 */

typedef int32_t fgb_status;
enum {
  FGB_OK = 0,
  FGB_ERR_INVALID_ARG = 1,   /* null pointer, bad size, bad params                           */
  FGB_ERR_CUDA = 2,          /* a CUDA runtime call failed; see fgb_last_error()              */
  FGB_ERR_NO_DEVICE = 3,     /* no usable sm_90 device — the engine has NO CPU fallback       */
  FGB_ERR_LAYOUT = 4,        /* batch violates the layout rules above (alignment, ranges)     */
  FGB_ERR_UNIT_TOO_LARGE = 5,/* a single unit exceeds fgb_tile_capacity_bytes()               */
  FGB_ERR_NOMEM = 6,
  FGB_ERR_BUSY = 7,          /* fgb_submit while a previous submit has not been waited on     */
  FGB_ERR_MISSING_TAG = 8,   /* first record of a group lacks the UMI tag (vanilla_caller.rs:1493) */
  FGB_ERR_NOT_ENCODABLE = 9  /* fgb_pack8_encode: an observation outside the PACK8 alphabet     */
};

typedef struct fgb_handle fgb_handle;   /* one per GPU; thread-compatible, not thread-safe    */

/* Mirrors the arithmetic-relevant part of VanillaUmiConsensusOptions
 * (vanilla_caller.rs:284-341; CLI defaults common.rs:225-249).  Host-prep options
 * (min_input_base_quality, trim, max_reads) live in the host caller, not here. */
typedef struct fgb_params {
  uint8_t error_rate_pre_umi;          /* -1, default 45 */
  uint8_t error_rate_post_umi;         /* -2, default 40 */
  uint8_t min_consensus_base_quality;  /* default 2 (CLI) / 40 (library default)              */
  uint8_t reserved0;
  uint32_t min_reads;                  /* per-position depth gate, vanilla_caller.rs:1345     */
} fgb_params;

typedef uint64_t fgb_read_desc;        /* (byte_off << 16) | len                              */
#define FGB_READ_DESC(off, len) ((((uint64_t)(off)) << 16) | ((uint64_t)(len) & 0xFFFFu))
#define FGB_READ_OFF(d) ((uint64_t)(d) >> 16)
#define FGB_READ_LEN(d) ((uint32_t)((d) & 0xFFFFu))

typedef struct fgb_unit {
  uint64_t out_off;     /* first output element of this unit                                  */
  uint32_t read_begin;  /* index of its first read in reads[]; n_reads = next.read_begin - it */
  uint32_t cons_len;    /* consensus length (positions to call)                               */
} fgb_unit;

typedef struct fgb_tile {
  uint64_t byte_begin;  /* 16-aligned start of the tile's byte range in bases[]/quals[]       */
  uint32_t byte_len;    /* multiple of 16                                                     */
  uint32_t unit_begin;
  uint32_t n_units;
  uint32_t read_begin;
  uint32_t n_reads;
  uint32_t flags;       /* bit0: oversize unit voted straight from HBM; bits 8..31: 8-position items
                           per unit when every unit of the tile has the same count (else 0)    */
} fgb_tile;

typedef struct fgb_batch {
  uint64_t n_units;     /* U */
  uint64_t n_reads;     /* R */
  uint64_t n_bytes;     /* valid bytes in bases[]/quals[]; allocation must be padded to 16    */
  uint64_t n_out;       /* elements in each output column                                     */
  uint64_t n_tiles;     /* T */
  const uint8_t* bases;
  const uint8_t* quals;
  const fgb_read_desc* reads;  /* [R]   */
  const fgb_unit* units;       /* [U+1] */
  const fgb_tile* tiles;       /* [T]   */
  /* since ABI 2: tiles come in three classes (flags bits 4..5: general, shallow = every unit has at most 4
   * reads, deep = every unit has at least 24), each with its own kernel.  When the tile array is sorted by
   * class (fgb_sort_tiles_by_class) these are the three run lengths; all zero = not sorted, the general
   * kernel votes every tile (correct, slower on shallow and deep units).  The host-buffer calls
   * (fgb_submit*) sort their tiles themselves and ignore this field. */
  uint64_t class_tiles[3];
} fgb_batch;

typedef struct fgb_columns {   /* consensus output columns, [n_out] each                      */
  uint8_t* base;
  uint8_t* qual;
  uint16_t* depth;
  uint16_t* errors;
} fgb_columns;

/* Device-side counters accumulated over every launch on a handle (the part of
 * ConsensusCallingStats / CodecConsensusStats that is computed inside the kernels; the
 * host-side read/rejection counters live in the host caller).  These are what the multi-GPU
 * driver all-reduces (sum) over NCCL at end of run. */
enum {
  FGB_CTR_UNITS = 0,            /* units voted                                                */
  FGB_CTR_POSITIONS = 1,        /* consensus positions emitted                                */
  FGB_CTR_EXACT_POSITIONS = 2,  /* positions that took the exact f64 path (diagnostic)        */
  FGB_CTR_NOCALL_POSITIONS = 3, /* positions emitted as N                                     */
  FGB_CTR_INPUT_READS = 4,      /* source reads consumed                                      */
  FGB_CTR_DUPLEX_BASES = 5,     /* codec_caller.rs:1157 consensus_duplex_bases_emitted        */
  FGB_CTR_DUPLEX_DISAGREE = 6,  /* codec_caller.rs:1158 duplex_disagreement_base_count        */
  FGB_CTR_COMBINED = 7,         /* strand-combine jobs processed                              */
  FGB_CTR_FILTER_RECORDS = 8,   /* consensus reads seen by the filter epilogue                */
  FGB_CTR_FILTER_PASSED = 9,    /* ... that passed every read-level gate                      */
  FGB_CTR_FILTER_BASES_MASKED = 10, /* bases newly masked to N by the filter                  */
  FGB_NCOUNTERS = 12
};

/* ---- lifecycle ------------------------------------------------------------------------ */
/* Builds the two 94-entry f64 likelihood tables (base_builder.rs:252-278) and the
 * single-input quality LUT (vanilla_caller.rs:463-482) with the host libm, uploads them, and
 * creates the streams/events the handle owns.  Fails with FGB_ERR_NO_DEVICE if `device` is not
 * a CUDA device of compute capability 10.x. */
fgb_status fgb_create(int device, const fgb_params* params, fgb_handle** out);
void fgb_destroy(fgb_handle* h);
const char* fgb_strerror(fgb_status s);
/* Copies the last detailed error text of this handle (e.g. the CUDA error string). */
size_t fgb_last_error(const fgb_handle* h, char* buf, size_t buf_len);
uint32_t fgb_abi_version(void);

/* The host-computed tables, for inspection/tests: correct[94], err_alt[94], *ln_pre,
 * single_input_q[94] (any pointer may be NULL). */
fgb_status fgb_get_tables(const fgb_handle* h, double* correct, double* err_alt, double* ln_pre,
                          uint8_t* single_input_q);

/* Pure host function (no device): the same tables fgb_create builds, for any (pre, post).
 * qt[256] is the fast-path quality threshold by depth (255 = never); any pointer may be NULL. */
fgb_status fgb_host_tables(uint8_t error_rate_pre_umi, uint8_t error_rate_post_umi,
                           double* correct, double* err_alt, double* ln_pre,
                           uint8_t* single_input_q, uint8_t* qt, uint32_t* fast_qual);

/* Pure host function: the integer "dominant winner" proof tables the kernel uses to skip the f64
 * path (fgumi_b200/csrc/host_tables.cpp): dfix[96] = round((correct[q]-err_alt[q])*65536) with
 * INT32_MIN marking unusable qualities, *g2fix the fixed-point gap threshold, *nmax2 the largest
 * pileup the proof covers.  Exposed so the proof can be tested against the oracle on the CPU. */
fgb_status fgb_host_proof_tables(uint8_t error_rate_pre_umi, uint8_t error_rate_post_umi,
                                 int32_t* dfix, int32_t* g2fix, uint32_t* nmax2);

/* Pure host function: the step table the shallow vote kernel uses for UNANIMOUS pileups whose likelihood gap is below
 * the reference's fast path (base_builder.rs:338-379): the called quality as a function of the fixed-point gap
 * g = sum round((correct[q]-err_alt[q])*65536).  gap_begin[128] ascending (unused entries INT32_MAX), quality[128]:
 * a gap in [gap_begin[k], gap_begin[k+1]) calls quality[k].  The kernel accepts the answer only when the interval
 * g +- (2 * depth + 1 + *guard) lies inside one step; anything else is evaluated literally.  Exposed so the table can
 * be tested against the oracle on the CPU. */
fgb_status fgb_host_unanimous_steps(uint8_t error_rate_pre_umi, uint8_t error_rate_post_umi,
                                    int32_t* gap_begin, uint8_t* quality, uint32_t* n_steps, int32_t* guard);

/* ---- batch planning (pure host code, no device needed) -------------------------------- */
/* Bytes of one column that a tile may span. */
uint32_t fgb_tile_capacity_bytes(void);
uint32_t fgb_tile_max_units(void);
uint32_t fgb_tile_max_reads(void);
/* Greedy segmentation of units[0..n_units) into tiles.  Writes at most `cap` tiles to `out`
 * (may be NULL to count) and returns the number of tiles needed through *n_tiles.  Validates the
 * layout rules (FGB_ERR_LAYOUT) and the capacity (FGB_ERR_UNIT_TOO_LARGE). */
fgb_status fgb_plan_tiles(const fgb_unit* units, uint64_t n_units, const fgb_read_desc* reads,
                          uint64_t n_reads, fgb_tile* out, uint64_t cap, uint64_t* n_tiles);

/* Stable partition of a tile array by class (general, shallow, deep); class_tiles receives the run lengths
 * to put in fgb_batch.class_tiles.  The order of the tiles is immaterial to the kernels. */
fgb_status fgb_sort_tiles_by_class(fgb_tile* tiles, uint64_t n_tiles, uint64_t class_tiles[3]);

/* ---- the vote (simplex / single-strand consensus), K1 --------------------------------- */
/* Device-resident form: every pointer in `in`/`out` is a DEVICE pointer on the handle's GPU.
 * Enqueues ONE kernel launch on `stream` (a cudaStream_t passed as void*; NULL = default
 * stream) that calls every position of every unit.  Asynchronous.
 * Pointer alignment (the kernels read their inputs with bulk copies and write 8 positions at a time):
 * in->bases, in->quals, in->reads, in->units and in->tiles 16-byte aligned; out->base and out->qual 8-byte
 * aligned; out->depth and out->errors 16-byte aligned.  Anything else returns FGB_ERR_LAYOUT (fgb_last_error
 * names the pointer) and enqueues nothing. */
fgb_status fgb_vote_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* out,
                           void* stream);

/* Host-buffer form — the call a ConsensusCaller implementation makes.  Every pointer is a HOST
 * pointer (pinned memory makes the copies asynchronous; pageable memory works).  The library
 * owns the device buffers, chunks the batch at tile boundaries and overlaps H2D copy / vote /
 * D2H copy on its own streams.  Returns after enqueueing; fgb_wait() blocks until the output
 * columns are complete.  The caller owns all host buffers and must keep them alive until
 * fgb_wait() returns. */
fgb_status fgb_submit(fgb_handle* h, const fgb_batch* in, const fgb_columns* out);

/* ---- compact transfer formats (the PCIe link bounds end-to-end throughput) ------------------
 * PACK8: ONE byte per observation of a prepared SourceRead row instead of a base byte and a quality
 * byte: bits 7..6 = A,C,G,T (0..3), bits 5..0 = quality 0..61; 0x3E = (N, Q2), the masked base of
 * create_source_read (vanilla_caller.rs:908-916).  Row offsets and lengths are those of the
 * two-column layout, so units/reads/tiles are unchanged.  fgb_pack8_encode converts n bytes of a
 * (bases, quals) column pair; FGB_ERR_NOT_ENCODABLE (nothing useful in `out`) when a row holds a
 * lower-case or IUPAC base, an N whose quality is not 2, or a quality above 61 -- such batches go
 * through fgb_submit.  Row padding bytes (base 0, quality 0) are accepted and encode as 0x00. */
fgb_status fgb_pack8_encode(const uint8_t* bases, const uint8_t* quals, uint64_t n, uint8_t* out);
/* fgb_submit with `in->bases` holding the PACK8 column (in->quals is ignored): the column is
 * copied host->device and expanded to the two byte columns by an unpack kernel in front of the
 * vote.  Same chunking, ordering and completion rules as fgb_submit. */
fgb_status fgb_submit_pack8(fgb_handle* h, const fgb_batch* in, const fgb_columns* out);

/* BAM4: the records' own payload -- 4-bit packed sequence (raw-bam sequence.rs:9-35) and raw quality
 * bytes -- plus what the host decided per read.  The device does the per-base part of
 * create_source_read (vanilla_caller.rs:893-916): decode, orientation (reverse-complement and
 * reversed qualities for a reverse-strand read) and the min-input-quality mask, writing the
 * SourceRead rows straight into the HBM columns the vote reads.  The host keeps the per-read
 * decisions: which reads survive, the kept raw span (CODEC's virtual clip, codec_caller.rs:414-469)
 * and the row length after quality trim / mate-overlap clip / trailing-N strip (:899-927).
 * 1.5 bytes per raw base cross the link instead of 2 per row byte. */
typedef struct fgb_raw_read {    /* 16 bytes; entry r belongs to read r of the batch (fgb_batch.reads[r]) */
  uint64_t src_off;              /* index of the first kept raw base in the raw columns; even           */
  uint32_t raw_len;              /* kept raw bases (l_seq unless clipped in raw coordinates)            */
  uint32_t flags;                /* FGB_RAW_REVERSE                                                     */
} fgb_raw_read;
enum { FGB_RAW_REVERSE = 1 };

typedef struct fgb_raw_columns {
  uint64_t n_raw;                /* raw bases in the columns                                            */
  const uint8_t* seq4;           /* (n_raw + 1) / 2 bytes, base i in the high (i even) / low nibble     */
  const uint8_t* quals_raw;      /* n_raw bytes                                                         */
  const fgb_raw_read* raw_reads; /* n_reads entries in read order (chunks are cut along it, so spans
                                    should ascend); src_off even, inside the columns, and
                                    reads[r] length <= raw_len -- checked on the device where the
                                    span is read: a violation skips the read and makes the next
                                    fgb_wait return FGB_ERR_LAYOUT                                      */
  uint8_t min_input_base_quality;/* 0 = no masking (CODEC)                                              */
  uint8_t reserved[7];
} fgb_raw_columns;

/* RECORDS: the BAM records themselves (raw-bam fields.rs:6-23), shipped as they are -- one DMA from pinned
 * memory, no per-base host work.  raw_reads[r] describes read r of the batch: src_off = byte offset of the
 * record's packed-sequence field inside `records`, raw_len = the record's l_seq (its quality bytes start
 * (l_seq + 1) / 2 bytes after src_off), flags = FGB_RAW_REVERSE for a reverse-strand read.  The device does
 * the per-base part of create_source_read (vanilla_caller.rs:893-916) / to_source_read_for_codec_raw
 * (codec_caller.rs:414-469): row position p is raw base p (forward) or l_seq - 1 - p complemented (reverse),
 * q < min_input_base_quality -> (N, Q2).  The host keeps the per-read decisions; the row length in
 * fgb_batch.reads[r] is the length after mate clip / quality trim / trailing-N strip (<= raw_len).  Every
 * sequence field must start at least 16 bytes into `records` (it always does: a record's fixed fields come
 * first); spans are checked on the device, a violation skips the read and fails the next fgb_wait with
 * FGB_ERR_LAYOUT. */
typedef struct fgb_record_columns {
  uint64_t n_bytes;               /* bytes in `records`                                                   */
  const uint8_t* records;
  const fgb_raw_read* raw_reads;  /* n_reads entries                                                      */
  uint8_t min_input_base_quality; /* 0 = no masking (CODEC)                                               */
  uint8_t reserved[7];
} fgb_record_columns;

/* ---- overlapping-bases pre-pass (OverlappingBasesConsensusCaller, overlapping.rs:79-337) ---- */
enum { FGB_OVERLAP_AGREE_CONSENSUS = 0, FGB_OVERLAP_AGREE_MAX_QUAL = 1, FGB_OVERLAP_AGREE_PASS_THROUGH = 2 };
enum { FGB_OVERLAP_DISAGREE_CONSENSUS = 0, FGB_OVERLAP_DISAGREE_MASK_BOTH = 1,
       FGB_OVERLAP_DISAGREE_MASK_LOWER_QUAL = 2 };
/* One stretch of an R1 / R2 overlap, co-called by the device IN PLACE on the uploaded records before the rows
 * are built (OverlappingBasesConsensusCaller::call, overlapping.rs:236-337; the host decides the stretches from
 * the headers and CIGARs, the device applies the per-base rule): `len` bases of the record whose packed sequence
 * starts at seq1_off (l_seq1 bases, qualities behind them) from read offset o1, against the record at seq2_off
 * from o2.  The runs of one pair are consecutive; all but the first carry FGB_RUN_CONTINUES (one thread walks a
 * pair, so two runs never write the same packed byte at once).  A run may touch records that yield no row (a pair
 * whose reads the group rules rejected: the reference co-calls every pair and counts it): the call keeps every
 * run's sequence and quality fields resident next to the reads' and applies and counts every run.  A batch with no
 * tiles enqueues nothing, so its runs are neither applied nor counted; count those on the host. */
typedef struct fgb_overlap_run {
  uint64_t seq1_off, seq2_off;
  uint32_t l_seq1, l_seq2;
  uint32_t o1, o2, len;
  uint32_t flags;                 /* FGB_RUN_CONTINUES */
} fgb_overlap_run;
enum { FGB_RUN_CONTINUES = 1 };

/* fgb_submit for a batch whose rows are built on the device: `in` carries units / reads / tiles /
 * n_* as usual (row offsets and lengths describe the rows to build), in->bases and in->quals are
 * ignored.  Same chunking, ordering and completion rules as fgb_submit. */
fgb_status fgb_submit_bam4(fgb_handle* h, const fgb_batch* in, const fgb_raw_columns* raw,
                           const fgb_columns* out);
/* The general form: any input format, optionally NARROW outputs.  With FGB_OUT_U8, out->depth and
 * out->errors are treated as uint8_t columns of n_out elements (cast the pointers): the link then
 * carries 4 instead of 6 bytes per consensus position.  Allowed only when no unit has more than
 * 255 reads (FGB_ERR_INVALID_ARG otherwise); the record builder widens to i16 for the cd/ce tags. */
/* ---- consensus filter epilogue (single-strand reads) ----------------------------------------
 * What `fgumi filter` applies to a simplex consensus read, run on the columns right after the vote:
 * mask_bases (filter.rs:655-696), filter_read on the cD / cE the caller derives (filter.rs:453-471,
 * caller.rs:322-329), then the mean-quality and no-call gates (commands/filter.rs:909-929). */
typedef struct fgb_filter_params {      /* FilterThresholds (filter.rs:31-40) + command options   */
  uint32_t min_reads;                   /* -M: per-base depth gate and per-read cD gate            */
  int32_t min_base_quality;             /* -N; -1 = none                                           */
  double max_read_error_rate;           /* -E                                                      */
  double max_base_error_rate;           /* -e                                                      */
  double min_mean_base_quality;         /* -q; negative = none                                     */
  double max_no_call_fraction;          /* -n; >= 1.0 is an absolute count (commands/filter.rs:921) */
  uint8_t per_base_tags;                /* 0: the read would carry no cd/ce arrays, so every base
                                           has depth 0 for the mask (filter.rs:677)               */
  uint8_t reserved[7];
} fgb_filter_params;
enum {                                  /* per-unit result                                         */
  FGB_FILTER_PASS = 0,
  FGB_FILTER_INSUFFICIENT_READS = 1,    /* FilterResult::InsufficientReads                         */
  FGB_FILTER_EXCESSIVE_ERROR_RATE = 2,  /* FilterResult::ExcessiveErrorRate                        */
  FGB_FILTER_LOW_MEAN_QUALITY = 3,
  FGB_FILTER_TOO_MANY_NO_CALLS = 4,
  FGB_FILTER_NO_RECORD = 255            /* unit without a consensus read (cons_len 0)              */
};
/* `fgumi filter` on DUPLEX consensus reads: three tiers of thresholds (filter.rs:120-215) -- `cc` for
 * the final consensus, `ab` (the stricter tier) for the better strand of each metric, `ba` for the
 * worse one -- and optional single-strand agreement masking (filter.rs:702-806).  `cc` also carries
 * the options shared with the simplex filter (min_base_quality, min_mean_base_quality,
 * max_no_call_fraction; per_base_tags is ignored: the record says what it carries). */
typedef struct fgb_duplex_filter_params {
  fgb_filter_params cc;
  uint32_t ab_min_reads;
  uint32_t ba_min_reads;
  double ab_max_read_error_rate;
  double ba_max_read_error_rate;
  double ab_max_base_error_rate;
  double ba_max_base_error_rate;
  uint8_t require_ss_agreement;         /* --require-single-strand-agreement                       */
  uint8_t reserved[7];
} fgb_duplex_filter_params;
/* ---- the on-disk framing of the output (SURVEY §8f N4; host code) ----------------------------------- */
/* The ConsensusOutput stream is the record section of a BAM file as it stands.  fgb_bam_header writes
 * "BAM\1" | l_text | text | n_ref = 0 (consensus reads are unmapped); fgb_bgzf_compress cuts a byte
 * stream into BGZF members (<= 0xFF00 input bytes each, SAM spec §4.1) on n_threads threads and, when
 * asked, appends the 28-byte EOF member.  `out` must hold fgb_bgzf_bound(len) bytes.  Level 1 is the library's
 * own DEFLATE encoder (csrc/host/fast_deflate.h: greedy one-probe LZ77 + per-block Huffman codes, ~200-260 MB/s per
 * thread on consensus BAM bytes, a little smaller than zlib -1's output; own CRC-32); the other levels are zlib's,
 * looked up at call time (libz.so.1) -- if it is missing they return FGB_ERR_INVALID_ARG.  FGB_BGZF_ZLIB=1 in the
 * environment sends level 1 to zlib too (A/B runs). */
size_t fgb_bgzf_bound(size_t len);
/* ---- since ABI 3: BGZF members inflated on the device (K0z) ----------------------------------------------
 * The input side of a file-level run: the host frames the members (fgb_bgzf_scan_members: one pass over the 18-byte
 * headers and 8-byte trailers, no inflate), the COMPRESSED stream crosses the link, and fgb_bgzf_inflate_device
 * writes the inflated stream -- BAM header and records -- into device memory, one member per warp
 * (csrc/inflate_kernel.cuh; the decoder is csrc/inflate_core.h, the same code the CPU tests run against zlib).
 * status[m] = 0 or an error code of the decoder (1 input exhausted, 2 more output than ISIZE, 3 block type,
 * 4 stored length, 5 code lengths, 6 symbol / distance, 7 short output, 8 CRC mismatch): a corrupt member never
 * touches memory outside its own [out_off, out_off + out_len). */
typedef struct fgb_bgzf_member {
  uint64_t in_off;      /* first byte of the member's DEFLATE payload in the compressed stream      */
  uint64_t out_off;     /* where its output starts in the inflated stream (sum of the ISIZEs before) */
  uint32_t in_len;      /* payload bytes                                                           */
  uint32_t out_len;     /* ISIZE                                                                   */
  uint32_t crc;         /* CRC-32 of the output, from the member's trailer                         */
  uint32_t reserved;
} fgb_bgzf_member;
/* Host: fills members[0 .. *n_members) (call with members == NULL to count) and *out_len = total inflated size.
 * FGB_ERR_LAYOUT on a malformed header, a member that runs past `len`, or an ISIZE above 65536. */
fgb_status fgb_bgzf_scan_members(const uint8_t* data, size_t len, fgb_bgzf_member* members, uint64_t cap,
                                 uint64_t* n_members, uint64_t* out_len);
/* Device pointers throughout; `status` holds n_members bytes; *n_bad (device, optional) is incremented per failed member. */
fgb_status fgb_bgzf_inflate_device(fgb_handle* h, const uint8_t* data, const fgb_bgzf_member* members,
                                   uint64_t n_members, uint8_t* out, uint8_t* status, int check_crc,
                                   unsigned long long* n_bad, void* stream);
/* The same decoder on the host, one member (tests, and callers without a device): returns the status code above. */
uint32_t fgb_host_inflate_member(const uint8_t* payload, uint32_t in_len, uint8_t* out, uint32_t out_len);
fgb_status fgb_bgzf_compress(const uint8_t* data, size_t len, int level, uint32_t n_threads, int append_eof,
                             uint8_t* out, size_t cap, size_t* out_len);
fgb_status fgb_bam_header(const char* sam_text, size_t l_text, uint8_t* out, size_t cap, size_t* out_len);
/* The input side of a file-level run (the reference's fgumi-bgzf reader.rs and raw-bam record framing; host code):
 *   fgb_bgzf_uncompressed_size  sum of the members' ISIZE fields
 *   fgb_bgzf_decompress         every member inflated at its place in `out` (cap >= that sum) on n_threads threads,
 *                               CRC32 / ISIZE checked; FGB_ERR_LAYOUT for a stream that is not BGZF
 *   fgb_bam_read_header         locates the SAM text and the first record of an uncompressed BAM stream
 *   fgb_bam_split_records       [u32 block_size][record]... -> record bodies back to back + rec_off[0..n], the form
 *                               fgb_host_group_by_mi and fgb_caller_add_groups take; `bodies` may be `stream` */
fgb_status fgb_bgzf_uncompressed_size(const uint8_t* data, size_t len, size_t* size);
fgb_status fgb_bgzf_decompress(const uint8_t* data, size_t len, uint32_t n_threads, uint8_t* out, size_t cap,
                               size_t* out_len);
fgb_status fgb_bam_read_header(const uint8_t* bam, size_t len, size_t* text_off, size_t* text_len, uint32_t* n_ref,
                               size_t* records_off);
fgb_status fgb_bam_split_records(const uint8_t* stream, size_t len, uint8_t* bodies, uint64_t* rec_off,
                                 uint64_t cap_records, uint64_t* n_records, size_t* consumed);

/*   fgb_host_duplex_record  duplex_read_into (duplex_caller.rs:1048-1285, methylation off): the BAM record
 *                           (block_size word included) of one duplex consensus read.  `ab` / `ba` are the
 *                           single-strand consensuses it was built from (ba may be absent: ba_len = 0 and
 *                           NULL columns with ba_present = 0); rx / rx_first: n_rx RX values of the source
 *                           reads with their FIRST_SEGMENT flag (RX halves are swapped for reads of the
 *                           other segment, :1187-1211).  The flush of the duplex caller runs the same code. */
typedef struct fgb_strand_columns {
  const uint8_t* bases; const uint8_t* quals; const uint16_t* depths; const uint16_t* errors; uint32_t len;
  uint32_t present;
} fgb_strand_columns;
fgb_status fgb_host_duplex_record(const char* read_name_prefix, const char* read_group_id, const char* base_mi,
                                  int first_of_pair, int produce_per_base_tags, const uint8_t* bases,
                                  const uint8_t* quals, const uint16_t* errors, uint32_t len,
                                  const fgb_strand_columns* ab, const fgb_strand_columns* ba,
                                  const char cell_tag[2], const char* cell, const char* const* rx,
                                  const uint8_t* rx_first, uint32_t n_rx, uint8_t* out, size_t cap, size_t* out_len);

/* MI grouping of an input record stream (src/lib/mi_group.rs:386-470 MiGroupIterator): consecutive records
 * with the same key form a group; the key is the value of `tag` (a Z tag), with a trailing "/A" or "/B"
 * removed when strip_strand_suffix is set (duplex: fgumi-umi lib.rs:355-363 extract_mi_base), followed --
 * when cell_tag is given -- by a tab and the value of that tag (empty if absent).  Records without `tag`
 * are skipped: keep[i] = 0.  group_begin[g] .. group_begin[g+1] delimit group g IN THE SEQUENCE OF KEPT
 * RECORDS (group_begin has room for n_records + 1 entries); when nothing is skipped the table can be handed
 * to fgb_caller_add_groups as group_rec directly. */
fgb_status fgb_host_group_by_mi(const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                const char tag[2], int strip_strand_suffix, const char* cell_tag,
                                uint8_t* keep, uint64_t* group_begin, uint64_t* n_groups);

/* ---- raw-record helpers of the host prep (pure host code, no device needed) ------------------ */
/* The reference exposes these from fgumi-raw-bam; the callers use them for every source read, and
 * they are exported so a host integration -- and the CPU test-suite -- can call the same code.
 *   fgb_host_is_fr_pair                     overlap.rs:15-62   is_fr_pair_raw
 *   fgb_host_num_bases_extending_past_mate  overlap.rs:65-136  num_bases_extending_past_mate_raw
 *   fgb_host_clip_cigar_ops                 cigar.rs:355-397   clip_cigar_ops_raw; out_ops holds n_ops + 2
 *   fgb_host_read_pos_at_ref_pos            cigar.rs:412-457   read_pos_at_ref_pos_raw; returns 0 = None
 *   fgb_host_simplify_cigar                 noodles_compat.rs:10-55; out_kinds / out_lens hold n_ops   */
/*   fgb_host_source_reads   the simplex sub-group prep: for each record (the rec_off convention of
 *                           fgb_caller_add_group) the mate-overlap clip and create_source_read
 *                           (vanilla_caller.rs:863-955), then filter_source_reads_by_alignment
 *                           (:961-1013).  Writes the surviving rows back to back into out_bases /
 *                           out_quals (capacity: the sum of the records' l_seq), row r at
 *                           [row_off[r], row_off[r+1]), its record index in orig_idx[r]; *n_rows rows,
 *                           *n_minority reads dropped by the CIGAR filter.
 *   fgb_host_consensus_umis simple_umi.rs:65-122, 236-245; umis = n NUL-terminated strings; returns
 *                           FGB_ERR_INVALID_ARG where the reference panics (unequal lengths, DNA mixed
 *                           with other characters) or when `cap` is too small                          */
fgb_status fgb_host_source_reads(const uint8_t* records, const uint64_t* rec_off, uint32_t n_records,
                                 uint8_t min_input_base_quality, int trim, uint8_t* out_bases,
                                 uint8_t* out_quals, uint64_t* row_off, uint32_t* orig_idx,
                                 uint32_t* n_rows, uint32_t* n_minority);
fgb_status fgb_host_consensus_umis(const char* const* umis, uint32_t n, char* out, size_t cap);
/*   fgb_host_simplex_record  build_consensus_record_into (vanilla_caller.rs:1365-1473): the BAM record
 *                           (block_size word included) of one simplex consensus read from its four
 *                           columns.  read_type 0 fragment, 1 R1, 2 R2; cell_tag / cell may be NULL; rx =
 *                           n_rx NUL-terminated RX values of the source reads.  The record assembly of
 *                           fgb_caller_flush calls the same code.                                       */
fgb_status fgb_host_simplex_record(const char* read_name_prefix, const char* read_group_id, const char* umi,
                                   uint8_t read_type, int produce_per_base_tags, const uint8_t* bases,
                                   const uint8_t* quals, const uint16_t* depths, const uint16_t* errors,
                                   uint32_t len, const char cell_tag[2], const char* cell,
                                   const char* const* rx, uint32_t n_rx, uint8_t* out, size_t cap,
                                   size_t* out_len);
int fgb_host_is_fr_pair(const uint8_t* record, size_t len);
uint32_t fgb_host_num_bases_extending_past_mate(const uint8_t* record, size_t len);
fgb_status fgb_host_clip_cigar_ops(const uint32_t* ops, uint32_t n_ops, uint32_t clip_amount, int from_start,
                                   uint32_t* out_ops, uint32_t* out_n, uint32_t* ref_consumed);
int fgb_host_read_pos_at_ref_pos(const uint32_t* ops, uint32_t n_ops, uint64_t alignment_start,
                                 uint64_t ref_pos, int return_last_base_if_deleted, uint64_t* read_pos);
fgb_status fgb_host_simplify_cigar(const uint32_t* ops, uint32_t n_ops, uint8_t* out_kinds, uint32_t* out_lens,
                                   uint32_t* out_n);

/* One assembled consensus record (BAM bytes without the block_size word) through the filter, on the
 * host: masks bases in place (sequence nibble -> N, quality -> 2), then applies the read-level gates
 * (filter_duplex_read filter.rs:477-557 when the record has aD / bD, else filter_read :453-471; then
 * commands/filter.rs:909-929).  *status = FGB_FILTER_*, *masked = bases newly masked.  Pure host
 * code: no device needed. */
fgb_status fgb_filter_record(uint8_t* record, size_t len, const fgb_duplex_filter_params* p,
                             uint32_t* masked, uint8_t* status);

/* Device-resident form: masks `cols` in place for the units of `in`, writes one status byte (and
 * optionally the newly-masked count) per unit.  All pointers are device pointers. */
fgb_status fgb_filter_simplex_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* cols,
                                     const fgb_filter_params* fp, uint8_t* unit_status,
                                     uint32_t* unit_masked, void* stream);

/* Device-resident variant of the unpack step alone (multi-kernel flows, tests): all pointers of
 * `in`, `raw` and the row columns are device pointers; enqueues one kernel on `stream`.  Columns that start on a
 * 4-byte boundary and whose sizes ((n_raw + 1) / 2 and n_raw bytes) are multiples of 4 take the word kernel (aligned
 * 32-bit window loads, nothing outside the columns is read); any other shape takes a byte-load kernel. */
fgb_status fgb_unpack_bam4_device(fgb_handle* h, const fgb_batch* in, const fgb_raw_columns* raw,
                                  uint8_t* bases, uint8_t* quals, void* stream);
fgb_status fgb_wait(fgb_handle* h);

/* Pinned host allocation helpers (cudaHostAlloc / cudaFreeHost); fgb_host_is_pinned: 1 when `p` lies in
 * page-locked host memory known to the CUDA runtime. */
fgb_status fgb_host_alloc(void** p, size_t bytes);
void fgb_host_free(void* p);
int fgb_host_is_pinned(const void* p);

/* ---- strand combine, K2 (duplex) and K3 (CODEC) --------------------------------------- */
/* One duplex combine job: AB single-strand unit ⊕ BA single-strand unit → one duplex read.
 * len = min(cons_len[unit_a], cons_len[unit_b]) (duplex_caller.rs:846-849).  Errors are
 * recounted against the pooled source reads of both units (duplex_caller.rs:943-951). */
typedef struct fgb_duplex_job {
  uint32_t unit_a;      /* index into the voted batch's units[]                               */
  uint32_t unit_b;
  uint64_t out_off;     /* first output element (FGB_OUT_ALIGN-aligned)                       */
} fgb_duplex_job;

enum {   /* per-job status: which arm of duplex_consensus (duplex_caller.rs:855-1013) was taken */
  FGB_DUPLEX_BOTH = 0,     /* combined; output length = min(cons_len a, cons_len b)            */
  FGB_DUPLEX_A_ONLY = 1,   /* B had no coverage in the truncated region; output = A, full len  */
  FGB_DUPLEX_B_ONLY = 2,   /* A had no coverage; output = B, full len (is_ba_only)             */
  FGB_DUPLEX_NONE = 3,     /* neither strand has coverage: no duplex read                       */
  FGB_DUPLEX_PENDING = 255 /* internal to fgb_vote_duplex_device: not combined yet; never returned */
};

typedef struct fgb_duplex_out {
  uint8_t* base;           /* [n_out]; a job's row must hold max(cons_len a, cons_len b)       */
  uint8_t* qual;           /* [n_out] */
  uint16_t* errors;        /* [n_out] */
  uint8_t* status;         /* [n_jobs] FGB_DUPLEX_* (may be NULL)                              */
} fgb_duplex_out;

/* ---- since ABI 3: the duplex combine in the vote kernels' epilogue ------------------------------------
 * A duplex molecule's single-strand units are voted in one tile and combined while the tile's source rows are
 * still in shared memory and the single-strand words it just wrote are in L2: K2 neither reads the SS columns
 * back from HBM nor re-reads the source rows for the exact error recount (duplex_caller.rs:943-951).
 *
 * fgb_plan_tiles_jobs plans like fgb_plan_tiles but keeps the two units of a job (and every unit between
 * them) in one tile where they fit a stage, sorts the tiles by class (fills class_tiles like
 * fgb_sort_tiles_by_class) and attaches to every tile the jobs both of whose units it holds:
 * job_index[tile_jobs[t].begin .. +count) are indices into jobs[].  Jobs that cannot be attached (units in
 * different tiles, an oversize unit) are simply not listed; *n_attached counts the listed ones.  Call with
 * tiles == NULL to size the tile arrays (*n_tiles), job_index holds n_jobs entries. */
typedef struct fgb_tile_jobs {
  uint32_t begin;       /* first entry of job_index[] for this tile                              */
  uint16_t count;       /* attached jobs                                                         */
  uint16_t max_items;   /* 8-position words of the longest attached job                          */
} fgb_tile_jobs;

fgb_status fgb_plan_tiles_jobs(const fgb_unit* units, uint64_t n_units, const fgb_read_desc* reads,
                               uint64_t n_reads, const fgb_duplex_job* jobs, uint64_t n_jobs,
                               fgb_tile* tiles, uint64_t cap, uint64_t* n_tiles, uint64_t class_tiles[3],
                               fgb_tile_jobs* tile_jobs, uint32_t* job_index, uint64_t* n_attached);

/* Vote `in` (tiles from fgb_plan_tiles_jobs, class_tiles set) into `ss` and combine `jobs` into `out`: attached
 * both-strand jobs in the vote's epilogue, every other job (single-strand arms, unattached jobs, rows that are
 * not 8-aligned) by the standalone kernels afterwards.  Results are those of fgb_vote_device followed by
 * fgb_duplex_combine_device, bit for bit.  All pointers are device pointers; tile_jobs has in->n_tiles entries.
 * `in` and `ss` follow fgb_vote_device's alignment rule (FGB_ERR_LAYOUT otherwise, nothing enqueued).  The
 * combine runs in the epilogue only when out->base, out->qual and tile_jobs are 8-byte aligned and out->errors and
 * jobs 16-byte aligned; otherwise the call is fgb_vote_device followed by fgb_duplex_combine_device. */
fgb_status fgb_vote_duplex_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* ss,
                                  const fgb_duplex_job* jobs, uint64_t n_jobs,
                                  const fgb_tile_jobs* tile_jobs, const uint32_t* job_index,
                                  const fgb_duplex_out* out, void* stream);

/* `ss` are the four single-strand columns the vote wrote for `in` (device pointers).  Any column alignment: when
 * in->bases, ss->base, ss->qual, out->base and out->qual are 8-byte aligned and ss->depth and out->errors 16-byte
 * aligned a word kernel runs, otherwise a kernel with one warp per job and byte / u16 accesses. */
fgb_status fgb_duplex_combine_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* ss,
                                     const fgb_duplex_job* jobs, uint64_t n_jobs,
                                     const fgb_duplex_out* out, void* stream);

/* One CODEC combine job (codec_caller.rs:721-781): the two single-strand consensuses are
 * oriented (reverse-complemented when flagged, :507-520), padded with lowercase 'n'/Q0/0/0 to
 * `len` (:980), combined (:1029-1152), quality-masked (:1183-1212) and, when `rc_out`, the
 * result is reverse-complemented back (:783-784). */
typedef struct fgb_codec_job {
  uint32_t unit_a;      /* R1 single-strand unit                                              */
  uint32_t unit_b;      /* R2 single-strand unit                                              */
  uint64_t out_off;
  uint32_t len;         /* consensus_length                                                   */
  uint32_t pad_a_left;  /* 'n' columns to the left of A after orientation                     */
  uint32_t pad_b_left;
  uint8_t rc_a, rc_b;   /* reverse-complement the single-strand consensus before padding      */
  uint8_t rc_out;       /* reverse-complement the combined consensus                          */
  uint8_t reserved0;
} fgb_codec_job;

typedef struct fgb_codec_params {   /* CodecConsensusOptions, codec_caller.rs:99-166          */
  int32_t single_strand_qual;       /* -1 = None                                              */
  int32_t outer_bases_qual;         /* -1 = None                                              */
  uint32_t outer_bases_length;
  uint32_t max_duplex_disagreements;
  double max_duplex_disagreement_rate;
} fgb_codec_params;

enum {   /* per-job status byte (the reference raises anyhow::bail! and the command downgrades
            it to a per-group rejection by substring match, commands/codec.rs:391,617-624)    */
  FGB_CODEC_OK = 0,
  FGB_CODEC_HIGH_DISAGREEMENT_COUNT = 1,   /* codec_caller.rs:1160-1162 */
  FGB_CODEC_HIGH_DISAGREEMENT_RATE = 2     /* codec_caller.rs:1163-1165 */
};

typedef struct fgb_codec_out {
  fgb_columns cols;        /* [n_out] combined consensus columns                               */
  uint8_t* status;         /* [n_jobs] FGB_CODEC_*                                             */
  uint32_t* disagreements; /* [n_jobs] duplex_disagreements (may be NULL)                      */
  uint32_t* duplex_bases;  /* [n_jobs] duplex_bases_count   (may be NULL)                      */
} fgb_codec_out;

fgb_status fgb_codec_combine_device(fgb_handle* h, const fgb_batch* in, const fgb_columns* ss,
                                    const fgb_codec_job* jobs, uint64_t n_jobs,
                                    const fgb_codec_params* cp, const fgb_codec_out* out,
                                    void* stream);

/* ---- simplex record assembly on the device (K5) ------------------------------------------------------
 * build_consensus_record_into (vanilla_caller.rs:1365-1473) for the units of a batch, written by the device at
 * their final place in the ConsensusOutput stream.  The host supplies what only it knows: per unit the read type,
 * the UMI, the cell barcode and the RX consensus (in a string blob that starts with the read-name prefix and the
 * read group id), the record's size and offset.  Only for units of at most 255 reads (cD / cM then fit one byte
 * and the size is known before the vote). */
typedef struct fgb_record_job {
  uint64_t out_off;                /* byte offset of the record (its block_size word first) in the stream           */
  uint32_t str_off;                /* offset of [umi][cell][rx] in the string blob                                   */
  uint32_t size;                   /* bytes of the record incl. the block_size word                                  */
  uint16_t umi_len, cell_len, rx_len;
  uint8_t read_type;               /* 0 fragment, 1 R1, 2 R2                                                         */
  uint8_t flags;                   /* FGB_RECJOB_*                                                                   */
} fgb_record_job;
enum { FGB_RECJOB_HAS_CELL = 1, FGB_RECJOB_HAS_RX = 2, FGB_RECJOB_SKIP = 4 /* no record for this unit */ };

/* ---- the general host-buffer call --------------------------------------------------------------------
 * Any input format, optionally narrow outputs, the filter epilogue, and -- for the duplex / CODEC callers
 * -- the strand combine of the voted units in the same call.  With combine jobs the batch is processed as
 * ONE piece (a molecule's units must be voted before its job runs) and `out` receives the single-strand
 * columns (they become the ac/ad/ae/aq, bc/bd/be/bq tags). */
enum { FGB_IN_BYTES = 0, FGB_IN_PACK8 = 1, FGB_IN_BAM4 = 2, FGB_IN_RECORDS = 3 };
enum { FGB_OUT_U16 = 0, FGB_OUT_U8 = 1 };
typedef struct fgb_submit_options {
  uint32_t input_format;           /* FGB_IN_*  */
  uint32_t output_format;          /* FGB_OUT_* */
  const fgb_raw_columns* raw;      /* FGB_IN_BAM4 only */
  const fgb_filter_params* filter; /* non-NULL: run the filter epilogue before the copy back      */
  uint8_t* unit_status;            /* host, n_units bytes (required with `filter`)                */
  uint32_t* unit_masked;           /* host, n_units words, may be NULL                            */
  /* ---- since ABI 2 ---- */
  const fgb_record_columns* records;   /* FGB_IN_RECORDS only                                     */
  const fgb_duplex_job* duplex_jobs;   /* host; K2 after the vote                                 */
  uint64_t n_duplex_jobs;
  uint64_t n_duplex_out;               /* elements in each column of duplex_out                   */
  const fgb_duplex_out* duplex_out;    /* host columns                                            */
  const fgb_codec_job* codec_jobs;     /* host; K3 after the vote                                 */
  uint64_t n_codec_jobs;
  uint64_t n_codec_out;
  const fgb_codec_params* codec_params;
  const fgb_codec_out* codec_out;      /* host columns                                            */
  /* FGB_IN_RECORDS only: the overlapping-bases pre-pass on the device (the batch is then processed as one piece) */
  const fgb_overlap_run* overlap_runs;
  uint64_t n_overlap_runs;
  uint64_t* overlap_stats;             /* host u64[4], ADDED to at fgb_wait: overlapping bases, agreeing,
                                          disagreeing, corrected (CorrectionStats, overlapping.rs:42-77)  */
  uint8_t overlap_agreement;           /* FGB_OVERLAP_AGREE_*    */
  uint8_t overlap_disagreement;        /* FGB_OVERLAP_DISAGREE_* */
  /* simplex record assembly on the device: n_units jobs; the finished stream lands in rec_out (host, page-locked
   * for an asynchronous copy) and `out` may then hold NULL columns (nothing else is copied back).  Not with
   * FGB_OUT_U8, the filter or combine jobs. */
  uint8_t rec_cell_tag[2];
  uint8_t rec_per_base_tags;
  uint8_t reserved[3];
  const fgb_record_job* rec_jobs;
  const uint8_t* rec_strings;          /* [read-name prefix][read group id] then the units' strings              */
  uint64_t n_rec_string_bytes;
  uint32_t rec_prefix_len, rec_rg_len;
  uint8_t* rec_out;
  uint64_t n_rec_out_bytes;
} fgb_submit_options;
fgb_status fgb_submit_ex(fgb_handle* h, const fgb_batch* in, const fgb_columns* out,
                         const fgb_submit_options* opt);
/* Device-resident variant of the RECORDS unpack step alone (tests, multi-kernel flows): every pointer of
 * `in`, `rec` and the row columns is a device pointer; enqueues one kernel on `stream`. */
fgb_status fgb_unpack_records_device(fgb_handle* h, const fgb_batch* in, const fgb_record_columns* rec,
                                     uint8_t* bases, uint8_t* quals, void* stream);

/* ---- statistics, K4 -------------------------------------------------------------------- */
/* Synchronises the handle's streams and copies the device counters (cumulative). */
fgb_status fgb_stats(fgb_handle* h, uint64_t counters[FGB_NCOUNTERS]);
/* Device pointer to the live counter block (u64[FGB_NCOUNTERS]) so a multi-GPU driver can
 * ncclAllReduce it in place without a host round trip. */
fgb_status fgb_stats_device_ptr(fgb_handle* h, uint64_t** dev_counters);
fgb_status fgb_stats_reset(fgb_handle* h);
/* Number of kernel launches this handle has enqueued (for bench.py's gpu_launches). */
uint64_t fgb_launch_count(const fgb_handle* h);
/* Capability bits of the engine behind this ABI (a test stand-in may offer fewer). */
enum { FGB_CAP_RECORD_ASSEMBLY = 1 };
uint32_t fgb_engine_caps(void);

/* ---- record-level caller: the ConsensusCaller boundary itself --------------------------- */
/* Mirrors `trait ConsensusCaller` (caller.rs:205-234) for batches of MI groups: raw BAM records in,
 * a ConsensusOutput byte stream (`[u32 LE block_size][BAM record]...`, caller.rs:173-178) out.
 * The host side does what the reference's caller does around the vote (filtering, sub-grouping,
 * mate-overlap clip, source-read preparation, CIGAR filter, min-reads / orphan rules, record and
 * tag assembly, RX consensus, statistics); the vote itself runs on the GPU through fgb_submit. */
enum { FGB_MODE_SIMPLEX = 0, FGB_MODE_DUPLEX = 1, FGB_MODE_CODEC = 2 };

typedef struct fgb_caller_options {        /* VanillaUmiConsensusOptions, vanilla_caller.rs:284-341 */
  uint8_t mode;                            /* FGB_MODE_*                                           */
  uint8_t error_rate_pre_umi;              /* 45 */
  uint8_t error_rate_post_umi;             /* 40 */
  uint8_t min_input_base_quality;          /* 10 */
  uint8_t min_consensus_base_quality;      /* 40 (library) / 2 (CLI)                               */
  uint8_t produce_per_base_tags;           /* 1  */
  uint8_t trim;                            /* 0  */
  uint8_t consensus_call_overlapping_bases;/* 1 in the CLI (--consensus-call-overlapping-bases,
                                              commands/common.rs:347-356): run the R1/R2 overlap
                                              pre-pass on each group first; simplex/duplex only   */
  uint32_t min_reads;                      /* simplex: -M (per-position depth gate too); duplex:
                                              min total reads (duplex_caller.rs:358-395)           */
  uint32_t min_xy_reads;                   /* duplex only: min reads of the better-covered strand  */
  uint32_t min_yx_reads;                   /* duplex only: min reads of the other strand; 0 allows
                                              single-strand molecules                              */
  char tag[2];                             /* UMI tag, "MI"                                        */
  char cell_tag[2];                        /* {0,0} = none                                         */
  const char* read_name_prefix;            /* consensus read name = "<prefix>:<MI>"                */
  const char* read_group_id;               /* RG tag value                                         */
  /* CODEC only (CodecConsensusOptions, codec_caller.rs:99-166): min_reads = min_reads_per_strand */
  uint32_t min_duplex_length;              /* 1 */
  uint32_t reserved1;
  fgb_codec_params codec;                  /* single_strand_qual / outer_bases_* / disagreement gates */
  /* `fgumi simplex | fgumi filter` or `fgumi duplex | fgumi filter` in one pass (template mode,
   * commands/filter.rs:614-697): a template -- the fragment / R1 / R2 reads of one MI -- is emitted only
   * if all of its reads pass.  Simplex reads are masked on the device (`filter`), duplex reads on the
   * assembled records (`duplex_filter`); CODEC mode rejects filter_enabled. */
  uint8_t filter_enabled;
  uint8_t zero_copy_records;               /* 1: the caller promises that the records passed to add_group(s) stay valid
                                              and unchanged until the next flush returns.  A simplex caller with a device
                                              then ships them from where they are when they lie in page-locked memory
                                              (fgb_host_alloc / cudaHostAlloc / cudaHostRegister) instead of staging a copy;
                                              every add call of a batch must pass the same `records` pointer.  Ignored
                                              (a copy is staged) for pageable memory and by the other callers. */
  uint8_t track_rejects;                   /* simplex: keep the raw bytes of every rejected read (vanilla_caller.rs:371-374,
                                              the --rejects output of `fgumi simplex`) for fgb_caller_take_rejects.  With
                                              consensus_call_overlapping_bases the pre-pass then runs on the host, in the
                                              caller's staged copy (rejected reads are kept as the pre-pass leaves them). */
  uint8_t reserved2;
  uint32_t n_threads;                      /* host threads for fgb_caller_add_groups and the record
                                              assembly of flush; 0 or 1 = the calling thread only  */
  fgb_filter_params filter;                /* filter.per_base_tags is set from produce_per_base_tags */
  fgb_duplex_filter_params duplex_filter;  /* duplex mode with filter_enabled: `fgumi duplex | fgumi
                                              filter`, template mode, on the assembled records     */
} fgb_caller_options;

enum {   /* ConsensusCallingStats (caller.rs:238-286) as a flat counter array                      */
  FGB_STAT_TOTAL_READS = 0,
  FGB_STAT_CONSENSUS_READS = 1,
  FGB_STAT_FILTERED_READS = 2,
  FGB_STAT_REJ_INSUFFICIENT_READS = 3,        /* RejectionReason::InsufficientReads              */
  FGB_STAT_REJ_SECONDARY_SUPPLEMENTARY = 4,   /* ::SecondaryOrSupplementary                      */
  FGB_STAT_REJ_ZERO_LENGTH = 5,               /* ::ZeroLengthAfterTrimming                       */
  FGB_STAT_REJ_MINORITY_ALIGNMENT = 6,        /* ::MinorityAlignment                             */
  FGB_STAT_REJ_ORPHAN_CONSENSUS = 7,          /* ::OrphanConsensus                               */
  FGB_STAT_REJ_POTENTIAL_COLLISION = 8,       /* ::PotentialCollision (duplex_caller.rs:1799-1823) */
  FGB_STAT_REJ_FRAGMENT_READ = 9,             /* ::FragmentRead (codec_caller.rs:564-566)        */
  FGB_STAT_REJ_INSUFFICIENT_OVERLAP = 10,     /* ::InsufficientOverlap (codec_caller.rs:688-694) */
  FGB_STAT_REJ_INDEL_ERROR = 11,              /* ::IndelErrorBetweenStrands (:697-737)           */
  FGB_STAT_DUPLEX_BASES = 12,                 /* consensus_duplex_bases_emitted (:1157)          */
  FGB_STAT_DUPLEX_DISAGREEMENTS = 13,         /* duplex_disagreement_base_count (:1158)          */
  FGB_STAT_OVERLAP_BASES = 14,                /* CorrectionStats (overlapping.rs:42-77)          */
  FGB_STAT_OVERLAP_AGREEING = 15,
  FGB_STAT_OVERLAP_DISAGREEING = 16,
  FGB_STAT_OVERLAP_CORRECTED = 17,
  FGB_STAT_FILTER_RECORDS = 18,               /* consensus reads seen by the filter               */
  FGB_STAT_FILTER_PASSED = 19,                /* reads emitted (whole templates that passed)      */
  FGB_STAT_FILTER_BASES_MASKED = 20,
  FGB_NSTATS = 24
};

/* ---- overlapping-bases pre-pass (OverlappingBasesConsensusCaller, overlapping.rs:79-337) ---- */
/* apply_overlapping_consensus (overlapping.rs:625-667) on one MI group, IN PLACE: primary R1/R2
 * records with the same name are paired and the bases they align to the same reference position
 * are co-called (sequence nibbles and qualities rewritten).  stats[4] += {overlapping_bases,
 * bases_agreeing, bases_disagreeing, bases_corrected}.  Host-only; needs no handle. */
fgb_status fgb_overlap_apply_group(uint8_t* records, const uint64_t* rec_off, uint32_t n_records,
                                   uint8_t agreement, uint8_t disagreement, uint64_t stats[4]);

typedef struct fgb_caller fgb_caller;
/* device >= 0: a caller with its own engine handle on that GPU.
 * device == FGB_DEVICE_NONE: a PLANNING-ONLY caller -- fgb_caller_add_group(s) run the whole host prep
 * and queue the batch, fgb_caller_pending exposes it, and fgb_caller_flush fails with FGB_ERR_NO_DEVICE.
 * It makes no CUDA call and computes no consensus (there is no CPU fallback); it exists so the host side of
 * the three callers can be inspected and tested on a machine without a GPU.  A simplex caller plans on
 * record headers as a caller with a device does (the overlapping-bases pre-pass runs on the host, in its
 * copy of the records); fgb_caller_pending lays the plans out as a flush would and decodes the rows from
 * that copy. */
#define FGB_DEVICE_NONE (-1)
fgb_status fgb_caller_create(int device, const fgb_caller_options* opt, fgb_caller** out);
/* What is queued for the next flush: the packed batch (tiles not planned yet: tiles = NULL, n_tiles = 0;
 * units[] holds n_units entries WITHOUT the sentinel, so the reads of the last unit end at n_reads), the
 * duplex jobs and the CODEC jobs.  Host pointers, valid until the next add / flush / destroy.  A simplex
 * caller with a device builds its rows on the device and reports an empty batch here. */
fgb_status fgb_caller_pending(const fgb_caller* c, fgb_batch* batch, const fgb_duplex_job** duplex_jobs,
                              uint64_t* n_duplex_jobs, const fgb_codec_job** codec_jobs,
                              uint64_t* n_codec_jobs);
void fgb_caller_destroy(fgb_caller* c);
size_t fgb_caller_last_error(const fgb_caller* c, char* buf, size_t buf_len);
/* consensus_reads() for one MI group: `records` holds n_records raw BAM records (no block_size
 * prefix) back to back, record i spanning [rec_off[i], rec_off[i+1]).  Groups are queued. */
fgb_status fgb_caller_add_group(fgb_caller* c, const uint8_t* records, const uint64_t* rec_off,
                                uint32_t n_records);
/* The same for many groups at once: group g holds records [group_rec[g], group_rec[g+1]) of the
 * rec_off table (n_groups + 1 entries in group_rec, group_rec[n_groups] + 1 entries in rec_off).
 * With options.n_threads > 1 the per-group host work (filtering, source-read preparation, CIGAR
 * grouping, ...) runs on that many threads over contiguous ranges of groups and the results are
 * merged in input order, so the output is identical to calling fgb_caller_add_group in a loop.  This
 * is the reference's "one caller per worker" (simplex.rs:574) folded behind one call.
 * Errors: a group whose first record lacks the UMI tag (FGB_ERR_MISSING_TAG), a malformed record
 * (FGB_ERR_INVALID_ARG / FGB_ERR_LAYOUT: offsets must ascend), a read longer than FGB_MAX_READ_LEN or a group of
 * more than 65535 reads (FGB_ERR_UNIT_TOO_LARGE) fail the CALL: nothing of a failing call stays queued, whatever the
 * caller's mode and n_threads (counters included), and work queued by earlier calls is never touched.
 * (fgb_caller_add_group, the one-group form, has nothing to roll back: a failing group is simply not queued.) */
fgb_status fgb_caller_add_groups(fgb_caller* c, const uint8_t* records, const uint64_t* rec_off,
                                 const uint64_t* group_rec, uint64_t n_groups);
/* Rejected reads (options.track_rejects, simplex callers): the records rejected by every add call since the last
 * take, each with its block_size word in front (a BAM record stream like ConsensusOutput), in the order the
 * reference's reject sites run -- secondary / supplementary reads, a group or sub-group below min_reads, reads of
 * zero length after trimming, the minority of the alignment filter (ascending input order; the reference iterates
 * a HashSet there, vanilla_caller.rs:964, 1193-1196), what is left below min_reads after it, and the surviving reads
 * of an orphan R1 / R2 consensus (:1095-1105).  *data stays valid until the next add / take / destroy. */
fgb_status fgb_caller_take_rejects(fgb_caller* c, const uint8_t** data, uint64_t* len, uint64_t* count);
/* Votes everything queued (one fgb_submit) and returns the concatenated ConsensusOutput of all
 * groups in input order.  *out_data stays valid until the next flush / destroy. */
fgb_status fgb_caller_flush(fgb_caller* c, const uint8_t** out_data, uint64_t* out_len,
                            uint64_t* out_count);
fgb_status fgb_caller_stats(const fgb_caller* c, uint64_t stats[FGB_NSTATS]);

/* ---- UMI assignment: the four `fgumi group` strategies (crates/fgumi-umi/src/assigner.rs for mapped data,
 * src/lib/umi/parallel_assigner.rs for `group --allow-unmapped`) ---------------------------------------------
 * A batch of position groups; group g is calls [group_off[g], group_off[g+1]), call c is UMIs
 * [call_off[c], call_off[c+1]), UMI u is bytes [umi_off[u], umi_off[u+1]) of `umis` (what umi_for_read made of
 * the read's tag: fgb_host_umi_for_read).  A call is one UmiAssigner::assign (the orientation sub-groups of a
 * position group are separate calls, group.rs:382-407).  Per UMI the result is a kind (FGB_MOL_*) and an id
 * LOCAL to its group: mapped rules keep one counter across a group's calls, unmapped rules restart at 0 on
 * every call.  group_mi_count[g] = max(id) + 1 over the group (0 if nothing is assigned), so the MI of a UMI is
 * "N", "N/A" or "N/B" with N = id + the sum of the earlier groups' counts + the run's base.
 * The device finds the UMI graph's edges (umi_kernels.cuh); unique / count / sort and the order-dependent rules
 * (BFS from roots in sorted order, union-find, numbering) run on n_threads host threads. */
enum { FGB_UMI_IDENTITY = 0, FGB_UMI_EDIT = 1, FGB_UMI_ADJACENCY = 2, FGB_UMI_PAIRED = 3 };
enum { FGB_UMI_RULES_MAPPED = 0, FGB_UMI_RULES_UNMAPPED = 1 };
enum { FGB_MOL_NONE = 0, FGB_MOL_SINGLE = 1, FGB_MOL_A = 2, FGB_MOL_B = 3 };
typedef struct fgb_umi_options {
  uint32_t strategy;        /* FGB_UMI_*                                                                 */
  uint32_t edits;           /* max mismatches; must be 0 for identity                                    */
  uint32_t rules;           /* FGB_UMI_RULES_*                                                           */
  uint32_t min_umi_length;  /* 0 = none; else every UMI of a call is truncated to it, a shorter one fails */
  uint32_t n_threads;       /* host threads; 0 or 1 = the calling thread only                           */
  uint32_t reserved;
} fgb_umi_options;
/* Errors fail the whole batch with FGB_ERR_INVALID_ARG and fgb_last_error names the call: valid UMIs of different
 * base lengths in one mapped adjacency call, a paired UMI without exactly one '-', a UMI shorter than
 * min_umi_length, edits != 0 with identity, malformed offsets.  ids / kinds hold n_umis entries. */
fgb_status fgb_umi_assign(fgb_handle* h, const fgb_umi_options* opt, const uint8_t* umis, const uint64_t* umi_off,
                          uint64_t n_umis, const uint64_t* call_off, uint64_t n_calls, const uint64_t* group_off,
                          uint64_t n_groups, uint64_t* ids, uint8_t* kinds, uint64_t* group_mi_count);
/* umi_for_read (group.rs:300-350): the upper-cased UMI, or for mapped paired rules the prefixed form
 * "a..a:<first>-b..b:<second>" (prefixes of edits + 1 characters; swapped when R2 is earlier).  Host code. */
fgb_status fgb_host_umi_for_read(const fgb_umi_options* opt, const uint8_t* umi, size_t len, int is_r1_earlier,
                                 uint8_t* out, size_t cap, size_t* out_len);
/* The unique-key table of one call as fgb_umi_assign sends it to the device, in the order the rules sort it:
 * identity and mapped edit by string, unmapped edit by first appearance, adjacency and paired by count
 * descending then string.  Exposed with fgb_host_umi_resolve so the host half can be tested without a device. */
typedef struct fgb_umi_key {
  uint64_t bits;            /* BitEnc (bitenc.rs:32-90): base i in bits 2i..2i+1, A=0 C=1 G=2 T=3         */
  uint64_t str_off;         /* the key's string in key_bytes                                             */
  uint32_t str_len;
  uint32_t count;           /* UMIs of the call with this key                                            */
  uint32_t first;           /* index within the call of its first UMI                                    */
  uint32_t dash;            /* position of the '-' (paired keys)                                         */
  uint8_t len;              /* bases in bits                                                             */
  uint8_t flags;            /* FGB_UMI_KEY_LAST: the last key of its BitEnc (unmapped rules look BitEncs
                               up in a map where the last index wins, parallel_assigner.rs:184-185)      */
  uint8_t reserved[6];
} fgb_umi_key;
enum { FGB_UMI_KEY_LAST = 1 };
/* keys has room for n_umis entries, key_bytes for umi_off[n_umis] - umi_off[0] bytes, key_of for n_umis
 * (UINT32_MAX: the UMI has no key). */
fgb_status fgb_host_umi_prepare(const fgb_umi_options* opt, const uint8_t* umis, const uint64_t* umi_off,
                                uint64_t n_umis, fgb_umi_key* keys, uint64_t* n_keys, uint8_t* key_bytes,
                                uint32_t* key_of);
/* The rules of one call given its key table and capture lists (key i's neighbours edges[edge_off[i] ..
 * edge_off[i+1]), ascending): ids from 0 as a fresh assigner would give them. */
fgb_status fgb_host_umi_resolve(const fgb_umi_options* opt, const uint8_t* umis, const uint64_t* umi_off,
                                uint64_t n_umis, const fgb_umi_key* keys, uint64_t n_keys, const uint8_t* key_bytes,
                                const uint32_t* key_of, const uint64_t* edge_off, const uint32_t* edges,
                                uint64_t* ids, uint8_t* kinds);

/* The capture lists the device finds for ONE call, as fgb_umi_assign computes them (the CSR fgb_host_umi_resolve
 * takes): *n_keys keys (the order of fgb_host_umi_prepare), edge_off[0 .. *n_keys] (room for n_umis + 1 entries),
 * *n_edges entries, written to `edges` only when cap >= *n_edges (call with cap 0 to size).  For tests and for
 * integrations that apply their own rules to the graph. */
fgb_status fgb_umi_edges(fgb_handle* h, const fgb_umi_options* opt, const uint8_t* umis, const uint64_t* umi_off,
                         uint64_t n_umis, uint64_t* n_keys, uint64_t* edge_off, uint32_t* edges, uint64_t cap,
                         uint64_t* n_edges);
/* Where the last fgb_umi_assign on this handle spent its time, in ms: [0] key tables on the host, [1] the device
 * phase as the host saw it (staging, copies, kernels), [2] the edge kernels alone (CUDA events around the count
 * pass with its sort / scan and around the fill pass), [3] the rules and numbering on the host. */
fgb_status fgb_umi_last_timing(const fgb_handle* h, double ms[4]);

/* ---- `fgumi group` from raw records (src/lib/commands/group.rs, src/lib/grouper.rs; host code around fgb_umi_assign)
 * Position grouping of an input stream (compute_group_key_from_raw, unified_pipeline/bam.rs:415-499, and
 * RecordPositionGrouper, grouper.rs:406-588): secondary and supplementary records are skipped (keep[i] = 0); the
 * others form groups of consecutive records with the same key -- both unclipped 5' ends (the mate's through MC), lower
 * first, the library of the RG (RGs sharing an LB are one library, an unknown RG is library 0; `header_text` is the
 * SAM header) and, when cell_tag is given, the cell barcode -- and a record at a new key whose QNAME continues the
 * previous kept record's stays in its group (unmapped mates).  group_begin (room for n_records + 1 entries) indexes
 * the KEPT records, the table fgb_grouper_add_groups takes once the skipped records are dropped.  A paired, mapped
 * primary record with a mapped mate and no MC tag fails the call with FGB_ERR_INVALID_ARG and *bad_record = its index;
 * a malformed record gives FGB_ERR_LAYOUT.  Library, cell and QNAME are compared as bytes where the reference
 * compares their hashes (the same answer barring a hash collision). */
fgb_status fgb_host_group_by_position(const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                      const char* header_text, size_t header_len, const char* cell_tag,
                                      uint8_t* keep, uint64_t* group_begin, uint64_t* n_groups, uint64_t* bad_record);

typedef struct fgb_group_options {
  fgb_umi_options umi;      /* strategy / edits / min_umi_length / n_threads; rules = FGB_UMI_RULES_UNMAPPED is
                               --allow-unmapped (the parallel assigners AND the filter's both-unmapped rule)      */
  uint8_t min_map_q;        /* 1 in the CLI                                                                      */
  uint8_t include_non_pf;   /* 0 */
  uint8_t no_umi;           /* group by position only: identity, 0 edits, every UMI "" (group.rs:732-757)        */
  uint8_t reserved0;
  char umi_tag[2];          /* "RX" */
  char assign_tag[2];       /* "MI" */
  uint64_t first_mi;        /* MI number of the first molecule                                                   */
} fgb_group_options;

enum {   /* fgb_grouper_stats: FilterMetrics (group.rs:113-262, per primary READ) and the grouper's own counters */
  FGB_GSTAT_TOTAL = 0, FGB_GSTAT_ACCEPTED = 1, FGB_GSTAT_DISCARDED_NON_PF = 2, FGB_GSTAT_DISCARDED_POOR_ALIGNMENT = 3,
  FGB_GSTAT_DISCARDED_NS_IN_UMI = 4, FGB_GSTAT_DISCARDED_UMI_TOO_SHORT = 5,
  FGB_GSTAT_POSITION_GROUPS = 6,   /* position groups added                                                      */
  FGB_GSTAT_GROUPS_DROPPED = 7,    /* position groups whose assignment the reference rejects (a paired UMI without
                                      exactly one '-', a UMI that is not UTF-8): logged and skipped there          */
  FGB_GSTAT_NEXT_MI = 8,           /* MI number of the next molecule                                             */
  FGB_GSTAT_RECORDS_OUT = 9,
  FGB_GROUP_NSTATS = 12
};
enum { FGB_GROUP_HIST_FAMILY = 0, FGB_GROUP_HIST_POSITION = 1 };

/* The record-level grouper: process_and_write_position_group (group.rs:1460-1592) per position group.
 * add_groups (group g = records [group_rec[g], group_rec[g+1]) of the rec_off table) runs, on n_threads host threads
 * over contiguous ranges of groups: templates from consecutive records with one QNAME, filter_template_raw, the
 * pair-orientation split (non-paired strategies; sub-groups in (r1+, r2+) order, false first), the UMI of R1 (else
 * R2) through umi_for_read.  The records of templates that pass are copied; the caller's buffers are free again on
 * return.  A template with two primary R1s (or R2s) or a malformed record fails the call (FGB_ERR_INVALID_ARG /
 * FGB_ERR_LAYOUT) and leaves nothing of it queued; a group the reference would drop is counted and dropped.
 * flush sends every queued group through fgb_umi_assign in one device phase (a mapped adjacency call with UMIs of
 * different lengths fails it with FGB_ERR_INVALID_ARG and changes nothing), sorts each group's templates stably by
 * (MoleculeId::to_vec_index, QNAME), None first, counts family and position-group sizes, and emits the primary records
 * with the assign tag set (update_string_tag, tags.rs:694-721; a template without an ID unchanged), each with its
 * block_size word, in input order and byte-identical for any n_threads.  *out stays valid until the next flush or
 * destroy.  device == FGB_DEVICE_NONE: planning only -- flush fails with FGB_ERR_NO_DEVICE; pending exposes the UMI
 * batch exactly as it would go to fgb_umi_assign (one entry per queued group with templates) and flush_with_ids
 * completes the flush from ids / kinds / group_mi_count computed elsewhere.  The pointers of pending stay valid until
 * the next add / flush / destroy. */
typedef struct fgb_grouper fgb_grouper;
fgb_status fgb_grouper_create(int device, const fgb_group_options* opt, fgb_grouper** out);
void fgb_grouper_destroy(fgb_grouper* g);
size_t fgb_grouper_last_error(const fgb_grouper* g, char* buf, size_t buf_len);
fgb_status fgb_grouper_add_groups(fgb_grouper* g, const uint8_t* records, const uint64_t* rec_off,
                                  const uint64_t* group_rec, uint64_t n_groups);
fgb_status fgb_grouper_pending(fgb_grouper* g, const uint8_t** umis, const uint64_t** umi_off, uint64_t* n_umis,
                               const uint64_t** call_off, uint64_t* n_calls, const uint64_t** group_off,
                               uint64_t* n_groups);
fgb_status fgb_grouper_flush(fgb_grouper* g, const uint8_t** out, uint64_t* out_len, uint64_t* n_records);
fgb_status fgb_grouper_flush_with_ids(fgb_grouper* g, const uint64_t* ids, const uint8_t* kinds,
                                      const uint64_t* group_mi_count, const uint8_t** out, uint64_t* out_len,
                                      uint64_t* n_records);
fgb_status fgb_grouper_stats(const fgb_grouper* g, uint64_t stats[FGB_GROUP_NSTATS]);
/* Family sizes (templates per molecule) or position-group sizes (molecules per group) accumulated over every flush,
 * ascending: *n entries, written only when cap >= *n (call with cap 0 to size). */
fgb_status fgb_grouper_histogram(const fgb_grouper* g, int which, uint64_t* sizes, uint64_t* counts, uint64_t cap,
                                 uint64_t* n);
/* Where the last fgb_grouper_flush spent its time, in ms: [0..3] fgb_umi_last_timing of its assignment, [4] the
 * sort, tags and output stream on the host. */
fgb_status fgb_grouper_last_timing(const fgb_grouper* g, double ms[5]);

/* ---- `fgumi dedup` from raw records (src/lib/commands/dedup.rs; host code around fgb_umi_assign and the template
 * score kernel, dedup_kernels.cuh)
 * Position grouping for dedup (RecordPositionGrouper::with_secondary_supplementary, grouper.rs:437-444, 488-547):
 * fgb_host_group_by_position with every record kept.  A secondary or supplementary record has the default key
 * (unified_pipeline/bam.rs:431-435), so it joins the previous record's group when it continues that record's QNAME and
 * otherwise opens a group of its own, which later such records join; MC is not checked on it.  Same arguments and
 * errors as fgb_host_group_by_position. */
fgb_status fgb_host_dedup_group_by_position(const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                            const char* header_text, size_t header_len, const char* cell_tag,
                                            uint8_t* keep, uint64_t* group_begin, uint64_t* n_groups,
                                            uint64_t* bad_record);

typedef struct fgb_dedup_options {
  fgb_umi_options umi;      /* strategy / edits / min_umi_length / n_threads; rules must be FGB_UMI_RULES_MAPPED    */
  uint8_t min_map_q;        /* 0 in the CLI; MQ tags are compared signed                                         */
  uint8_t include_non_pf;   /* 0 */
  uint8_t no_umi;           /* dedup by position only: identity, 0 edits, every UMI "" (dedup.rs:918-947)         */
  uint8_t remove_duplicates;/* skip records flagged 0x400 in the output instead of emitting them                 */
  char umi_tag[2];          /* "RX" */
  char assign_tag[2];       /* "MI" */
  uint64_t first_mi;        /* MI number of the first molecule                                                   */
} fgb_dedup_options;

enum {   /* fgb_deduper_stats: DedupMetrics (dedup.rs:71-92), FilterMetrics per TEMPLATE, and the deduper's counters */
  FGB_DSTAT_TOTAL_TEMPLATES = 0, FGB_DSTAT_UNIQUE_TEMPLATES = 1, FGB_DSTAT_DUPLICATE_TEMPLATES = 2,
  FGB_DSTAT_TOTAL_READS = 3, FGB_DSTAT_UNIQUE_READS = 4, FGB_DSTAT_DUPLICATE_READS = 5,
  FGB_DSTAT_SECONDARY_READS = 6, FGB_DSTAT_SUPPLEMENTARY_READS = 7,
  FGB_DSTAT_MISSING_TC_TAG = 8,    /* secondary / supplementary records of kept templates without a tc tag        */
  FGB_DSTAT_FILTER_TOTAL = 9, FGB_DSTAT_FILTER_ACCEPTED = 10, FGB_DSTAT_FILTER_NON_PF = 11,
  FGB_DSTAT_FILTER_POOR_ALIGNMENT = 12, FGB_DSTAT_FILTER_NS_IN_UMI = 13, FGB_DSTAT_FILTER_UMI_TOO_SHORT = 14,
  FGB_DSTAT_POSITION_GROUPS = 15,  /* position groups added                                                      */
  FGB_DSTAT_NEXT_MI = 16,          /* MI number of the next molecule                                             */
  FGB_DSTAT_RECORDS_OUT = 17,
  FGB_DEDUP_NSTATS = 20
};

/* The record-level deduper: process_position_group (dedup.rs:673-806) and its output (:1057-1138) per position group.
 * add_groups (group g = records [group_rec[g], group_rec[g+1]), every record of the stream as
 * fgb_host_dedup_group_by_position keeps it) runs on n_threads host threads: templates from consecutive records with
 * one QNAME, records in Template::from_records order (R1, R2, R1 supplementaries reversed, R2 supplementaries reversed,
 * R1 secondaries reversed, R2 secondaries reversed; template.rs:159-330), filter_template (dedup.rs:257-402; counts
 * per template, both-unmapped always rejected, MQ compared signed), 0x400 cleared on every record of a passing
 * template, the pair-orientation split (non-paired strategies), the UMI of R1 (else R2) through umi_for_read.  A
 * template with two primary R1s (or R2s), a malformed record or an assignment error (a paired UMI without exactly one
 * '-', a UMI that is not UTF-8; dedup.rs:717-719) fails the call and leaves nothing of it queued.
 * flush scores the primary records of every queued template on the device (fgb_record_quality_scores, started before
 * the assignment and waited for after it), sends every queued group through fgb_umi_assign, sorts each group's
 * templates stably by (MoleculeId::to_vec_index, QNAME), None first, keeps in each family the first template of that
 * order with the highest score (R1 score + R2 score) and flags every record of the others 0x400, and emits every record
 * of every template in that order with the assign tag set (update_string_tag; a template without an ID unchanged),
 * each with its block_size word; remove_duplicates skips records carrying 0x400.  Byte-identical for any n_threads.
 * device == FGB_DEVICE_NONE: planning only -- flush fails with FGB_ERR_NO_DEVICE; pending exposes the UMI batch as it
 * would go to fgb_umi_assign and flush_with_ids completes the flush from ids / kinds / group_mi_count and per-entry
 * template scores (indexed like the pending batch) computed elsewhere.  Pointers stay valid as for fgb_grouper_*. */
typedef struct fgb_deduper fgb_deduper;
fgb_status fgb_deduper_create(int device, const fgb_dedup_options* opt, fgb_deduper** out);
void fgb_deduper_destroy(fgb_deduper* d);
size_t fgb_deduper_last_error(const fgb_deduper* d, char* buf, size_t buf_len);
fgb_status fgb_deduper_add_groups(fgb_deduper* d, const uint8_t* records, const uint64_t* rec_off,
                                  const uint64_t* group_rec, uint64_t n_groups);
fgb_status fgb_deduper_pending(fgb_deduper* d, const uint8_t** umis, const uint64_t** umi_off, uint64_t* n_umis,
                               const uint64_t** call_off, uint64_t* n_calls, const uint64_t** group_off,
                               uint64_t* n_groups);
fgb_status fgb_deduper_flush(fgb_deduper* d, const uint8_t** out, uint64_t* out_len, uint64_t* n_records);
fgb_status fgb_deduper_flush_with_ids(fgb_deduper* d, const uint64_t* ids, const uint8_t* kinds,
                                      const uint64_t* group_mi_count, const uint32_t* scores, const uint8_t** out,
                                      uint64_t* out_len, uint64_t* n_records);
fgb_status fgb_deduper_stats(const fgb_deduper* d, uint64_t stats[FGB_DEDUP_NSTATS]);
/* Family sizes (templates per molecule, unassigned templates skipped) over every flush, ascending: *n entries,
 * written only when cap >= *n (call with cap 0 to size). */
fgb_status fgb_deduper_histogram(const fgb_deduper* d, uint64_t* sizes, uint64_t* counts, uint64_t cap, uint64_t* n);
/* Where the last fgb_deduper_flush spent its time, in ms: [0..3] fgb_umi_last_timing of its assignment, [4] the score
 * phase as the host saw it (staging, transfers, kernel, scores back), [5] the score kernel alone (CUDA events), [6]
 * the selection, flags, tags and output stream on the host. */
fgb_status fgb_deduper_last_timing(const fgb_deduper* d, double ms[7]);

/* score_template's per-read term (dedup.rs:230-249) on the device: scores[i] = sum(min(q, 15)) over record i's quality
 * bytes (record i = records[rec_off[i] .. rec_off[i+1]), no block_size prefix), read from qo = 32 + l_read_name +
 * 4 n_cigar + (l_seq + 1) / 2 for min(l_seq, len - qo) bytes (0 when qo >= len): a record whose qualities are cut short
 * by its end is clamped, and 0xFF qualities count 15.  Staged through page-locked chunks; synchronous.  A record
 * shorter than 32 bytes (or a descending rec_off) gives FGB_ERR_LAYOUT, fgb_last_error naming its index. */
fgb_status fgb_record_quality_scores(fgb_handle* h, const uint8_t* records, const uint64_t* rec_off,
                                     uint64_t n_records, uint32_t* scores);

/* ---- `fgumi sort` on raw records (src/lib/sort/, src/lib/commands/sort.rs): coordinate, template-coordinate and
 * queryname.  Keys (fgumi_b200/csrc/sort_keys.h, the same code on the host and the device):
 *   coordinate: one word, (tid << 34) | ((pos + 1) << 1) | reverse, all ones for tid < 0 (the unmapped flag is not
 *     looked at);
 *   template-coordinate: five words compared in order -- primary (tid1, tid2, pos1 of the pair's lower end first),
 *     secondary (pos2, inverted strands), the cell-barcode hash, tertiary (library ordinal, MI, !/A) and
 *     name_hash << 1 | is_upper -- packed bit for bit as TemplateKey::new (inline_buffer.rs:478-520).  The library
 *     ordinal numbers the distinct LB values of the header's @RG lines in byte order from 1 (0: no RG, an RG the
 *     header lacks, an RG without LB).  The name and cell hashes are 64-bit FNV-1a, not the reference's ahash;
 *   queryname (`--order queryname`, lexicographic) and queryname natural (`--order queryname::natural`): the read name
 *     (empty when l_read_name < 2 or the name runs past the record), then
 *     queryname_flag_order(flag) = ((f & 0xc0) << 8) | ((f & 0x100) << 3) | ((f & 0x800) >> 3) (keys.rs:338-363).
 *     Lexicographic compares the name bytes, embedded NULs included; natural is natural_compare_nul (the name cut at
 *     its first NUL; digit runs compare by value, so "01" and "1" are equal).  Encoded exactly as W big-endian words
 *     of a byte string E plus the word (len(E) << 16) | flag order (fgb_host_sort_name_key); cell_tag is ignored.
 * The order is a stable sort by the key: records with equal keys keep their input order. */
enum {
  FGB_SORT_COORDINATE = 0,
  FGB_SORT_TEMPLATE_COORDINATE = 1,
  FGB_SORT_QUERYNAME = 2,           /* SO:queryname SS:lexicographic */
  FGB_SORT_QUERYNAME_NATURAL = 3    /* SO:queryname SS:natural       */
};
typedef struct fgb_sort_options {
  uint32_t order;           /* FGB_SORT_*                                                                        */
  uint32_t n_threads;       /* host threads (staging copies, host keys); 0 or 1 = the calling thread only        */
  char cell_tag[2];         /* template-coordinate: the cell-barcode tag, "CB" as `fgumi sort` uses; "\0\0" = none */
  uint8_t reserved[6];
  uint64_t device_bytes;    /* device-memory budget of one sorted run; 0 = derived from cudaMemGetInfo per call  */
} fgb_sort_options;
/* Sorts n_records records (record i = records[rec_off[i] .. rec_off[i+1]), no block_size prefix) into `out` as
 * [u32 block_size][record]..., the record section of a BAM: out_len = rec_off[n] - rec_off[0] + 4 n, which `cap` must
 * hold.  Synchronous.  The records are sorted on the device in runs that fit device_bytes (keys, stable radix passes
 * over the key words that vary, record gather); several runs are merged on the host by key, ties by run.
 * `header_text` is the SAM header (its @RG lines give the library ordinals).  A too-small cap or bad options give
 * FGB_ERR_INVALID_ARG; a record shorter than 32 bytes (or a descending rec_off) gives FGB_ERR_LAYOUT with
 * *bad_record = its index.  A failing call frees whatever it allocated. */
fgb_status fgb_sort_records(fgb_handle* h, const fgb_sort_options* opt, const char* header_text, size_t header_len,
                            const uint8_t* records, const uint64_t* rec_off, uint64_t n_records, uint8_t* out,
                            uint64_t cap, uint64_t* out_len, uint64_t* bad_record);
/* The keys of fgb_sort_records on host threads (no device; there is no CPU sort): keys[5 i + w] = word w of record i
 * (coordinate: word 0, the others 0).  Errors as fgb_sort_records; the queryname orders, whose keys do not fit five
 * words, give FGB_ERR_INVALID_ARG (their keys come from fgb_host_sort_name_key). */
fgb_status fgb_host_sort_keys(const fgb_sort_options* opt, const char* header_text, size_t header_len,
                              const uint8_t* records, const uint64_t* rec_off, uint64_t n_records, uint64_t* keys,
                              uint64_t* bad_record);
/* The queryname key words the device's key kernel writes for one record (`len` bytes, no block_size prefix) when it
 * is alone in its run: *n_words = W + 1, W name words (W = ceil(bound / 8), the bound on E from l_read_name:
 * l_read_name - 1 bytes, natural 2 (l_read_name - 1) + 1, so at most 64) and the last word.  Within a run every record
 * gets the run's largest W; the extra name words are 0.  A record shorter than 32 bytes gives FGB_ERR_LAYOUT; a cap
 * below *n_words (which is still set), no words or an order other than the queryname ones give FGB_ERR_INVALID_ARG. */
fgb_status fgb_host_sort_name_key(const fgb_sort_options* opt, const uint8_t* record, uint64_t len, uint64_t* words,
                                  uint32_t cap, uint32_t* n_words);
/* `fgumi sort --verify` (commands/sort.rs:376-408, 692-720): the records whose key is less than the previous record's
 * (template-coordinate: core_cmp, the first four words, inline_buffer.rs:604-618; queryname: the name comparator,
 * then the flag order), and the index of the first of them (UINT64_MAX when there is none). */
fgb_status fgb_host_sort_verify(const fgb_sort_options* opt, const char* header_text, size_t header_len,
                                const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                uint64_t* violations, uint64_t* first_violation, uint64_t* bad_record);
/* Where the last fgb_sort_records on this handle spent its time, in ms, summed over its runs: [0] upload (staging
 * copies and transfers), [1] key kernel, [2] radix passes, [3] offsets scan and record gather (CUDA events for
 * [1]-[3]), [4] download, [5] host merge (0 for one run). */
fgb_status fgb_sort_last_timing(const fgb_handle* h, double ms[6]);

/* ---- `fgumi filter --ref` on raw records (src/lib/commands/filter.rs:550-905): mapped consensus reads masked, their
 * NM / UQ / MD regenerated against the reference (fgumi-sam alignment_tags.rs:254-420) and the reads or templates that
 * fail the read-level gates moved to a rejects stream.  Methylation options and compressed FASTA are not offered. */
typedef struct fgb_reference fgb_reference;
/* Parses an uncompressed FASTA image (`len` bytes) on the host as the reference's sequential reader does -- a contig's
 * name runs from after '>' to the first whitespace, its sequence is every following line up to the next '>' with the
 * line ends (\n, \r\n) removed and the bytes kept as they are -- and uploads the sequence once, as one byte array plus
 * a contig table, to `device`, where it stays until fgb_reference_destroy.  A gzip / BGZF image or text before the
 * first '>' gives FGB_ERR_INVALID_ARG; of two contigs with one name the later one is looked up, as in the reference.
 * device == FGB_DEVICE_NONE parses only: the contig query works, fgb_filter_records refuses it. */
fgb_status fgb_reference_create(int device, const uint8_t* fasta, size_t len, fgb_reference** out);
void fgb_reference_destroy(fgb_reference* r);
/* The contig count; with i < count, contig i's name (NUL-terminated, valid until destroy) and length. */
uint64_t fgb_reference_contigs(const fgb_reference* r);
fgb_status fgb_reference_contig(const fgb_reference* r, uint64_t i, const char** name, uint64_t* length);

typedef struct fgb_record_filter_options {
  fgb_duplex_filter_params filter;   /* the thresholds: cc for simplex reads, cc / ab / ba for duplex ones      */
  uint8_t filter_by_template;        /* 1: template mode (the default of `fgumi filter`); 0: each record alone    */
  uint8_t reverse_per_base_tags;     /* --reverse-per-base-tags                                                 */
  uint8_t track_rejects;             /* 1: rejected records go to the rejects stream                           */
  uint8_t reserved[1];
  uint32_t n_threads;                /* host threads (staging copies, templates); 0 or 1 = the calling thread   */
  uint64_t device_bytes;             /* device-memory budget of one run of templates; 0 = from cudaMemGetInfo   */
} fgb_record_filter_options;
enum { FGB_FSTAT_TOTAL = 0, FGB_FSTAT_PASSED = 1, FGB_FSTAT_FAILED = 2, FGB_FSTAT_BASES_MASKED = 3, FGB_FILTER_NSTATS = 4 };
/* Filters n_records records (record i = records[rec_off[i] .. rec_off[i+1]), no block_size prefix; a call holds whole
 * templates, a template being the records that share a QNAME consecutively).  Per record, in the reference's order:
 * the per-base tags of a reverse-strand read reversed (optional), masking (duplex reads, with aD or bD, by the three
 * tiers; others by cc), NM / UQ / MD regenerated when `ref` is given (unmapped: removed; ref_id -1: untouched), then
 * the read gates.  Template mode keeps a template when it has a primary record and every primary record passes; its
 * secondary and supplementary records also need to pass themselves.  Output: *kept and *rejects, library-owned
 * [u32 block_size][record] streams valid until the next call on `h` (records in template order, or input order in
 * single-read mode; rejects only with track_rejects), and stats[FGB_FSTAT_*].  Synchronous.
 * Errors fail the call and emit nothing; *bad_record = the first bad record in input order and fgb_last_error says
 * why: a record shorter than 32 bytes or with truncated fields (FGB_ERR_LAYOUT), a mapped record without `ref`, a
 * ref_id outside the header's @SQ lines, a negative position on a mapped record, a contig missing from the FASTA, an
 * alignment past the contig's end, a CIGAR that consumes more bases than l_seq, a template with two primary R1s or R2s
 * (FGB_ERR_INVALID_ARG). */
fgb_status fgb_filter_records(fgb_handle* h, const fgb_record_filter_options* opt, const fgb_reference* ref,
                              const char* header_text, size_t header_len, const uint8_t* records,
                              const uint64_t* rec_off, uint64_t n_records, const uint8_t** kept, uint64_t* kept_len,
                              const uint8_t** rejects, uint64_t* rejects_len, uint64_t stats[FGB_FILTER_NSTATS],
                              uint64_t* bad_record);
/* Where the last fgb_filter_records on `h` spent its time, in ms, summed over its runs: [0] upload, [1] pass 1 (tags,
 * masking, NM / UQ / MD sizes, gates), [2] template decision and offset scans, [3] pass 2 (edited records written),
 * [4] download (with the growth of the output streams), [5] host work (checks, templates, contig table, and every
 * device and page-locked allocation of the call).  [1]-[3] are CUDA events.  The staging buffers are at most 64 MiB;
 * the environment variable FGB_FILTER_STAGE_BYTES (at least 4096) lowers that, read on every call. */
fgb_status fgb_filter_last_timing(const fgb_handle* h, double ms[6]);

/* ---- `fgumi duplex-metrics` / `fgumi simplex-metrics` on raw records (src/lib/commands/{shared_metrics,
 * duplex_metrics,simplex_metrics}.rs, crates/fgumi-metrics): the QC tables of a UMI-grouped stream (group's output).
 * Per template (consecutive QNAME run of at least two records, Template::from_records order): R1 / R2 = the first
 * record that is paired, mapped with its mate mapped, of that segment, neither secondary nor supplementary (both are
 * required); R1's MI and RX must be Z strings in UTF-8 (else the call fails, before the interval test); the
 * ReadInfoKey (ref, unclipped 5', strand) of both reads, the earlier first, groups consecutive templates into
 * coordinate groups; the insert span (R1's own range when the mates are on different contigs) is tested against the
 * intervals; the read name's htsjdk Murmur3 (seed 42, UTF-16 code units) gives the template's downsampling fraction.
 * The template pass and the family counting (CS / SS / DS sizes, (ab, ba) pairs, per fraction) run on the device; the
 * UMI consensus of the 100 % fraction and the tables run on host threads. */
enum { FGB_METRICS_SIMPLEX = 0, FGB_METRICS_DUPLEX = 1 };
typedef struct fgb_metrics_options {
  uint32_t mode;              /* FGB_METRICS_SIMPLEX / FGB_METRICS_DUPLEX                                         */
  uint32_t n_threads;         /* host threads (templates, UMI consensus); 0 or 1 = the calling thread             */
  uint64_t min_ab_reads;      /* duplex: --min-ab-reads (1); must be >= min_ba_reads                              */
  uint64_t min_ba_reads;      /* duplex: --min-ba-reads (1)                                                       */
  uint64_t min_reads;         /* simplex: --min-reads (1)                                                         */
  uint8_t duplex_umi_counts;  /* duplex: --duplex-umi-counts                                                      */
  uint8_t reserved[7];
  uint64_t device_bytes;      /* device-memory budget of one staged run; 0 = from cudaMemGetInfo                 */
} fgb_metrics_options;
/* The template statuses of fgb_host_metrics_templates. */
enum {
  FGB_MT_SKIP = 0,            /* fewer than 2 records, no R1 or R2, or a read without a CIGAR                     */
  FGB_MT_OUTSIDE = 1,         /* outside every interval                                                           */
  FGB_MT_KEPT = 2,
  FGB_MT_ERR_MI_MISSING = 3, FGB_MT_ERR_MI_UTF8 = 4, FGB_MT_ERR_RX_MISSING = 5, FGB_MT_ERR_RX_UTF8 = 6
};
typedef struct fgb_metrics_template {   /* one template as the device's template pass sees it                     */
  int32_t ref1, start1, ref2, start2;   /* ReadInfoKey: the earlier (ref, unclipped 5', 0-based) read first        */
  uint8_t strand1, strand2;             /* reverse strand                                                          */
  uint8_t status;                       /* FGB_MT_*                                                                */
  uint8_t bucket;                       /* the first fraction index i with hash_fraction <= 0.05 (i + 1)           */
  int32_t contig;                       /* R1's ref_id                                                             */
  int32_t ins_start, ins_end;           /* 1-based insert span                                                     */
  uint8_t mi_kind;                      /* 0: no suffix, 1: "/A", 2: "/B"                                          */
  uint8_t mi_canonical;                 /* the MI's base is a canonical decimal: mi_base is its value              */
  uint8_t name_ascii;                   /* 0: the name has a byte >= 0x80 and its bucket comes from the host       */
  uint8_t reserved;
  uint32_t r1;                          /* R1's record index (in the call)                                         */
  uint64_t mi_base;
  uint32_t mi_off, mi_len, rx_off, rx_len;   /* the MI / RX strings, offsets within R1's record                    */
} fgb_metrics_template;
/* The template pass on host threads, the same code as the device's: templates = the QNAME runs of the records
 * (record i = records[rec_off[i] .. rec_off[i+1]), no block_size prefix), out[t] for run t (cap >= runs), *n_templates.
 * `intervals` (BED or Picard interval list text, NULL = none) are matched by contig name against `header_text`'s @SQ
 * lines.  A malformed record gives FGB_ERR_LAYOUT, a template with two primary R1s or R2s FGB_ERR_INVALID_ARG, each
 * with *bad_record; an unparsable interval line FGB_ERR_INVALID_ARG. */
fgb_status fgb_host_metrics_templates(const char* header_text, size_t header_len, const char* intervals,
                                      size_t intervals_len, const uint8_t* records, const uint64_t* rec_off,
                                      uint64_t n_records, fgb_metrics_template* out, uint64_t cap,
                                      uint64_t* n_templates, uint64_t* bad_record);
/* compute_hash_fraction (shared_metrics.rs:106-184): the name (`len` bytes, lossy UTF-8 to UTF-16) -> the Murmur3 hash,
 * wrapping_abs(hash) / i32::MAX and the bucket (0..19). */
fgb_status fgb_host_metrics_name_fraction(const uint8_t* name, size_t len, int32_t* hash, double* fraction,
                                          uint32_t* bucket);
/* The bucket of a Murmur3 hash, as the device computes it. */
uint32_t fgb_host_metrics_bucket(int32_t hash);
/* BED or Picard interval list text (parse_intervals, shared_metrics.rs:186-253) -> 0-based half-open intervals:
 * *n entries of (name offset, name length, start, end) into `text`, written when cap >= *n. */
fgb_status fgb_host_metrics_intervals(const char* text, size_t len, uint64_t* name_off, uint64_t* name_len,
                                      int64_t* start, int64_t* end, uint64_t cap, uint64_t* n);
/* The TSV float text (csv 1.1 / ryu 1.0 shortest round trip, DESIGN.md section 13) of v; returns its length. */
size_t fgb_host_metrics_format_float(double v, char* buf, size_t cap);

typedef struct fgb_metrics fgb_metrics;
/* min_ab_reads < min_ba_reads, an unknown mode or unparsable intervals give FGB_ERR_INVALID_ARG.  device ==
 * FGB_DEVICE_NONE: a planning-only collector -- add_records and finish fail with FGB_ERR_NO_DEVICE. */
fgb_status fgb_metrics_create(int device, const fgb_metrics_options* opt, const char* header_text, size_t header_len,
                              const char* intervals, size_t intervals_len, fgb_metrics** out);
void fgb_metrics_destroy(fgb_metrics* m);
size_t fgb_metrics_last_error(const fgb_metrics* m, char* buf, size_t buf_len);
/* Streams records (a call holds whole QNAME runs; coordinate groups may continue into the next call).  The first
 * paired, primary R1 of the stream with aD and bD, or cD, fails the call (a consensus input).  Errors fail the call
 * with *bad_record = the record index (counted over every call) of the first bad template's first record, or of a
 * failing UMI family's first template, and poison the collector. */
fgb_status fgb_metrics_add_records(fgb_metrics* m, const uint8_t* records, const uint64_t* rec_off, uint64_t n_records,
                                   uint64_t* bad_record);
/* Closes the last coordinate group and builds the tables; no records may follow. */
fgb_status fgb_metrics_finish(fgb_metrics* m, uint64_t* bad_record);
enum {   /* the tables of fgb_metrics_table, each one output file */
  FGB_MTABLE_FAMILY_SIZES = 0,        /* <prefix>.family_sizes.txt                                    */
  FGB_MTABLE_DUPLEX_FAMILY_SIZES = 1, /* <prefix>.duplex_family_sizes.txt (duplex)                    */
  FGB_MTABLE_YIELD = 2,               /* <prefix>.duplex_yield_metrics.txt / .simplex_yield_metrics.txt */
  FGB_MTABLE_UMI_COUNTS = 3,          /* <prefix>.umi_counts.txt                                      */
  FGB_MTABLE_DUPLEX_UMI_COUNTS = 4    /* <prefix>.duplex_umi_counts.txt (duplex with duplex_umi_counts) */
};
/* A finished collector's table `which` as TSV text (valid until destroy); FGB_ERR_INVALID_ARG for a table the mode
 * does not write. */
fgb_status fgb_metrics_table(const fgb_metrics* m, uint32_t which, const char** text, uint64_t* len);
enum {
  FGB_MSTAT_RECORDS = 0, FGB_MSTAT_TEMPLATES = 1, FGB_MSTAT_KEPT = 2, FGB_MSTAT_OUTSIDE = 3, FGB_MSTAT_GROUPS = 4,
  FGB_MSTAT_DS_FAMILIES = 5, FGB_MSTAT_OVERFLOW = 6, FGB_MSTAT_RUNS = 7, FGB_METRICS_NSTATS = 8
};
fgb_status fgb_metrics_stats(const fgb_metrics* m, uint64_t stats[FGB_METRICS_NSTATS]);
/* Where the collector has spent its time so far, in ms: [0] template pass (upload, kernel, download), [1] family pass
 * (upload, group scan, sorts, counting kernels, download), [2] UMI consensus, [3] host assembly (templates, tables).
 * The staging buffers are at most 64 MiB; FGB_METRICS_STAGE_BYTES (at least 4096) lowers that, read on each call. */
fgb_status fgb_metrics_last_timing(const fgb_metrics* m, double ms[4]);

/* ---- `fgumi zipper` on raw records (src/lib/commands/zipper.rs process_raw :826-941, merge_raw :373-521,
 * Template::fix_mate_info in template.rs:411-710): the mapped records of each template get their mate fields, TLEN,
 * MQ / MC / ms, the unmapped read's tags (reversed or reverse-complemented on the reverse strand), its QC flag, AS / XS
 * in the smallest signed type and, on secondary and supplementary records, the tc tag.  BAM records only; SAM text,
 * --restore-unconverted-bases and stdin are not offered. */
typedef struct fgb_zipper_options {
  uint8_t exclude_missing_reads;     /* drop (and count) unmapped templates with no mapped template               */
  uint8_t skip_pa_tags;              /* no tc tag on secondary / supplementary records (--skip-pa-tags)           */
  uint8_t restore_unconverted_bases; /* not offered: non-zero gives FGB_ERR_INVALID_ARG                           */
  uint8_t reserved[1];
  uint32_t n_threads;                /* host threads (staging copies); 0 or 1 = the calling thread                 */
  uint64_t device_bytes;             /* device-memory budget of one run of templates; 0 = from cudaMemGetInfo     */
  uint64_t n_remove, n_reverse, n_revcomp;        /* the expanded tag lists (a named set like Consensus expanded   */
  const char (*tags_to_remove)[2];                /* by the caller): two bytes per name, no NUL                     */
  const char (*tags_to_reverse)[2];
  const char (*tags_to_revcomp)[2];
} fgb_zipper_options;
enum { FGB_ZSTAT_MERGED = 0, FGB_ZSTAT_UNMAPPED_ONLY = 1, FGB_ZSTAT_EXCLUDED = 2, FGB_ZSTAT_RECORDS_OUT = 3,
       FGB_ZIPPER_NSTATS = 4 };
/* Zips n_unmapped unmapped records (whole QNAME runs) with the mapped records not yet consumed (whole QNAME runs, in
 * the same name order; record i of a stream = records[off[i] .. off[i+1]), no block_size prefix).  Stateless.  Each
 * unmapped template (Template::from_records order) is merged with the next mapped template when their names are
 * equal as bytes -- the mapped records come out in template order -- else emitted unchanged (or, with
 * exclude_missing_reads, dropped).  *mapped_consumed = the mapped records the join used; without last_call the
 * rest are the caller's to pass again, with last_call a mapped template left over fails the call.  Output: *out, a
 * library-owned [u32 block_size][record] stream valid until the next call on `h`, and stats[FGB_ZSTAT_*].
 * Synchronous.  Errors fail the call and emit nothing; *bad_record names the first bad record met in join order,
 * counting the unmapped records as 0 .. n_unmapped - 1 and mapped record j as n_unmapped + j: a record shorter than
 * 32 bytes, with truncated fields or an aux area that does not parse to its end (FGB_ERR_LAYOUT), a record carrying
 * one tag twice, a mapped record with a CIGAR op code past 8, a template with two primary R1s or R2s, a mapped template
 * left over with last_call (FGB_ERR_INVALID_ARG).  A tag list entry with a NUL byte or restore_unconverted_bases
 * give FGB_ERR_INVALID_ARG.  One call runs on the handle's one GPU. */
fgb_status fgb_zipper_records(fgb_handle* h, const fgb_zipper_options* opt, const uint8_t* unmapped,
                              const uint64_t* u_off, uint64_t n_unmapped, const uint8_t* mapped, const uint64_t* m_off,
                              uint64_t n_mapped, int last_call, const uint8_t** out, uint64_t* out_len,
                              uint64_t* mapped_consumed, uint64_t stats[FGB_ZIPPER_NSTATS], uint64_t* bad_record);
/* The same on host threads, with the same per-record rules (no device; for tests, there is no CPU zipper): *out is a
 * malloc'ed stream the caller frees with fgb_host_free_buffer. */
fgb_status fgb_host_zipper_records(const fgb_zipper_options* opt, const uint8_t* unmapped, const uint64_t* u_off,
                                   uint64_t n_unmapped, const uint8_t* mapped, const uint64_t* m_off, uint64_t n_mapped,
                                   int last_call, uint8_t** out, uint64_t* out_len, uint64_t* mapped_consumed,
                                   uint64_t stats[FGB_ZIPPER_NSTATS], uint64_t* bad_record);
void fgb_host_free_buffer(void* p);
/* Where the last fgb_zipper_records on `h` spent its time, in ms, summed over its runs: [0] upload, [1] size pass,
 * [2] offset scan, [3] write pass, [4] download (with the output's growth), [5] host work (checks, join, template
 * table, allocations).  [1]-[3] are CUDA events.  The staging buffers are at most 64 MiB; FGB_ZIPPER_STAGE_BYTES (at
 * least 4096) lowers that, read on every call. */
fgb_status fgb_zipper_last_timing(const fgb_handle* h, double ms[6]);

/* sizeof() of the ABI structs as this library was compiled, so a binding can check its own layout:
 * 0 fgb_caller_options, 1 fgb_filter_params, 2 fgb_submit_options, 3 fgb_raw_columns,
 * 4 fgb_raw_read, 5 fgb_batch, 6 fgb_codec_params, 7 fgb_params, 8 fgb_duplex_filter_params,
 * 9 fgb_record_columns, 10 fgb_umi_options, 11 fgb_group_options, 12 fgb_sort_options, 13 fgb_dedup_options,
 * 14 fgb_record_filter_options, 15 fgb_metrics_options, 16 fgb_metrics_template, 17 fgb_zipper_options; 0 for an
 * unknown id. */
uint32_t fgb_struct_size(uint32_t id);

#ifdef __cplusplus
}
#endif
#endif /* FGUMI_B200_H */
