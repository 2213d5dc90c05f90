"""ctypes binding of the C-ABI in include/fgumi_b200.h (libfgumi_b200.so, built in-tree).

The library is the product; this file only declares its symbols.  Loading fails loudly when the
shared object is missing — there is no Python/CPU fallback for any compute entry point.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FGUMI_B200_LIB") or os.path.join(_HERE, "libfgumi_b200.so")   # override: kernel A/B runs

FGB_OK = 0
FGB_ERR_INVALID_ARG = 1
FGB_ERR_CUDA = 2
FGB_ERR_NO_DEVICE = 3
FGB_ERR_LAYOUT = 4
FGB_ERR_UNIT_TOO_LARGE = 5
FGB_ERR_NOMEM = 6
FGB_ERR_BUSY = 7
FGB_ERR_MISSING_TAG = 8
FGB_ERR_NOT_ENCODABLE = 9

FGB_READ_ALIGN = 8
FGB_OUT_ALIGN = 8
FGB_MAX_READ_LEN = 65535     # a row descriptor holds 16 bits of length
FGB_NCOUNTERS = 12
COUNTER_NAMES = (
    "units", "positions", "exact_positions", "nocall_positions", "input_reads",
    "duplex_bases", "duplex_disagreements", "combined_jobs",
    "filter_records", "filter_passed", "filter_bases_masked",
)

FGB_DUPLEX_BOTH, FGB_DUPLEX_A_ONLY, FGB_DUPLEX_B_ONLY, FGB_DUPLEX_NONE = 0, 1, 2, 3
FGB_CODEC_OK, FGB_CODEC_HIGH_DISAGREEMENT_COUNT, FGB_CODEC_HIGH_DISAGREEMENT_RATE = 0, 1, 2


class FgbParams(C.Structure):
    _fields_ = [
        ("error_rate_pre_umi", C.c_uint8),
        ("error_rate_post_umi", C.c_uint8),
        ("min_consensus_base_quality", C.c_uint8),
        ("reserved0", C.c_uint8),
        ("min_reads", C.c_uint32),
    ]


class FgbUnit(C.Structure):
    _fields_ = [("out_off", C.c_uint64), ("read_begin", C.c_uint32), ("cons_len", C.c_uint32)]


class FgbTile(C.Structure):
    _fields_ = [
        ("byte_begin", C.c_uint64),
        ("byte_len", C.c_uint32),
        ("unit_begin", C.c_uint32),
        ("n_units", C.c_uint32),
        ("read_begin", C.c_uint32),
        ("n_reads", C.c_uint32),
        ("flags", C.c_uint32),
    ]


class FgbBatch(C.Structure):
    _fields_ = [
        ("n_units", C.c_uint64),
        ("n_reads", C.c_uint64),
        ("n_bytes", C.c_uint64),
        ("n_out", C.c_uint64),
        ("n_tiles", C.c_uint64),
        ("bases", C.c_void_p),
        ("quals", C.c_void_p),
        ("reads", C.c_void_p),
        ("units", C.c_void_p),
        ("tiles", C.c_void_p),
        ("class_tiles", C.c_uint64 * 3),   # since ABI 2: run lengths of a class-sorted tile array (0,0,0 = unsorted)
    ]


class FgbColumns(C.Structure):
    _fields_ = [("base", C.c_void_p), ("qual", C.c_void_p), ("depth", C.c_void_p),
                ("errors", C.c_void_p)]


class FgbDuplexJob(C.Structure):
    _fields_ = [("unit_a", C.c_uint32), ("unit_b", C.c_uint32), ("out_off", C.c_uint64)]


class FgbDuplexOut(C.Structure):
    _fields_ = [("base", C.c_void_p), ("qual", C.c_void_p), ("errors", C.c_void_p),
                ("status", C.c_void_p)]


class FgbCodecJob(C.Structure):
    _fields_ = [
        ("unit_a", C.c_uint32),
        ("unit_b", C.c_uint32),
        ("out_off", C.c_uint64),
        ("len", C.c_uint32),
        ("pad_a_left", C.c_uint32),
        ("pad_b_left", C.c_uint32),
        ("rc_a", C.c_uint8),
        ("rc_b", C.c_uint8),
        ("rc_out", C.c_uint8),
        ("reserved0", C.c_uint8),
    ]


class FgbRawColumns(C.Structure):
    _fields_ = [("n_raw", C.c_uint64), ("seq4", C.c_void_p), ("quals_raw", C.c_void_p),
                ("raw_reads", C.c_void_p), ("min_input_base_quality", C.c_uint8),
                ("reserved", C.c_uint8 * 7)]


class FgbFilterParams(C.Structure):
    _fields_ = [("min_reads", C.c_uint32), ("min_base_quality", C.c_int32),
                ("max_read_error_rate", C.c_double), ("max_base_error_rate", C.c_double),
                ("min_mean_base_quality", C.c_double), ("max_no_call_fraction", C.c_double),
                ("per_base_tags", C.c_uint8), ("reserved", C.c_uint8 * 7)]


class FgbDuplexFilterParams(C.Structure):
    _fields_ = [("cc", FgbFilterParams), ("ab_min_reads", C.c_uint32), ("ba_min_reads", C.c_uint32),
                ("ab_max_read_error_rate", C.c_double), ("ba_max_read_error_rate", C.c_double),
                ("ab_max_base_error_rate", C.c_double), ("ba_max_base_error_rate", C.c_double),
                ("require_ss_agreement", C.c_uint8), ("reserved", C.c_uint8 * 7)]


class FgbStrandColumns(C.Structure):
    _fields_ = [("bases", C.c_void_p), ("quals", C.c_void_p), ("depths", C.c_void_p), ("errors", C.c_void_p),
                ("len", C.c_uint32), ("present", C.c_uint32)]


class FgbRecordColumns(C.Structure):
    _fields_ = [("n_bytes", C.c_uint64), ("records", C.c_void_p), ("raw_reads", C.c_void_p),
                ("min_input_base_quality", C.c_uint8), ("reserved", C.c_uint8 * 7)]


class FgbSubmitOptions(C.Structure):
    _fields_ = [("input_format", C.c_uint32), ("output_format", C.c_uint32), ("raw", C.c_void_p),
                ("filter", C.c_void_p), ("unit_status", C.c_void_p), ("unit_masked", C.c_void_p),
                # since ABI 2
                ("records", C.c_void_p),
                ("duplex_jobs", C.c_void_p), ("n_duplex_jobs", C.c_uint64), ("n_duplex_out", C.c_uint64),
                ("duplex_out", C.c_void_p),
                ("codec_jobs", C.c_void_p), ("n_codec_jobs", C.c_uint64), ("n_codec_out", C.c_uint64),
                ("codec_params", C.c_void_p), ("codec_out", C.c_void_p),
                ("overlap_runs", C.c_void_p), ("n_overlap_runs", C.c_uint64), ("overlap_stats", C.c_void_p),
                ("overlap_agreement", C.c_uint8), ("overlap_disagreement", C.c_uint8),
                ("rec_cell_tag", C.c_uint8 * 2), ("rec_per_base_tags", C.c_uint8), ("reserved", C.c_uint8 * 3),
                ("rec_jobs", C.c_void_p), ("rec_strings", C.c_void_p), ("n_rec_string_bytes", C.c_uint64),
                ("rec_prefix_len", C.c_uint32), ("rec_rg_len", C.c_uint32), ("rec_out", C.c_void_p),
                ("n_rec_out_bytes", C.c_uint64)]


FGB_DEVICE_NONE = -1      # fgb_caller_create: planning-only caller (no engine, flush refuses)
FGB_FILTER_PASS, FGB_FILTER_INSUFFICIENT_READS, FGB_FILTER_EXCESSIVE_ERROR_RATE = 0, 1, 2
FGB_FILTER_LOW_MEAN_QUALITY, FGB_FILTER_TOO_MANY_NO_CALLS, FGB_FILTER_NO_RECORD = 3, 4, 255


FGB_IN_BYTES, FGB_IN_PACK8, FGB_IN_BAM4, FGB_IN_RECORDS = 0, 1, 2, 3
FGB_OUT_U16, FGB_OUT_U8 = 0, 1


class FgbCodecParams(C.Structure):
    _fields_ = [
        ("single_strand_qual", C.c_int32),
        ("outer_bases_qual", C.c_int32),
        ("outer_bases_length", C.c_uint32),
        ("max_duplex_disagreements", C.c_uint32),
        ("max_duplex_disagreement_rate", C.c_double),
    ]


class FgbCallerOptions(C.Structure):
    _fields_ = [
        ("mode", C.c_uint8), ("error_rate_pre_umi", C.c_uint8), ("error_rate_post_umi", C.c_uint8),
        ("min_input_base_quality", C.c_uint8), ("min_consensus_base_quality", C.c_uint8),
        ("produce_per_base_tags", C.c_uint8), ("trim", C.c_uint8),
        ("consensus_call_overlapping_bases", C.c_uint8),
        ("min_reads", C.c_uint32), ("min_xy_reads", C.c_uint32), ("min_yx_reads", C.c_uint32),
        ("tag", C.c_char * 2), ("cell_tag", C.c_char * 2),
        ("read_name_prefix", C.c_char_p), ("read_group_id", C.c_char_p),
        ("min_duplex_length", C.c_uint32), ("reserved1", C.c_uint32), ("codec", FgbCodecParams),
        ("filter_enabled", C.c_uint8), ("zero_copy_records", C.c_uint8), ("track_rejects", C.c_uint8), ("reserved2", C.c_uint8), ("n_threads", C.c_uint32),
        ("filter", FgbFilterParams), ("duplex_filter", FgbDuplexFilterParams),
    ]


FGB_UMI_IDENTITY, FGB_UMI_EDIT, FGB_UMI_ADJACENCY, FGB_UMI_PAIRED = 0, 1, 2, 3
FGB_UMI_RULES_MAPPED, FGB_UMI_RULES_UNMAPPED = 0, 1
FGB_MOL_NONE, FGB_MOL_SINGLE, FGB_MOL_A, FGB_MOL_B = 0, 1, 2, 3


class FgbUmiOptions(C.Structure):
    _fields_ = [("strategy", C.c_uint32), ("edits", C.c_uint32), ("rules", C.c_uint32),
                ("min_umi_length", C.c_uint32), ("n_threads", C.c_uint32), ("reserved", C.c_uint32)]


class FgbGroupOptions(C.Structure):
    _fields_ = [("umi", FgbUmiOptions), ("min_map_q", C.c_uint8), ("include_non_pf", C.c_uint8),
                ("no_umi", C.c_uint8), ("reserved0", C.c_uint8), ("umi_tag", C.c_char * 2),
                ("assign_tag", C.c_char * 2), ("first_mi", C.c_uint64)]


FGB_GROUP_NSTATS = 12
GROUP_STAT_NAMES = ("total_records", "accepted_records", "discarded_non_pf", "discarded_poor_alignment",
                    "discarded_ns_in_umi", "discarded_umi_too_short", "position_groups", "groups_dropped", "next_mi",
                    "records_out")
FGB_GROUP_HIST_FAMILY, FGB_GROUP_HIST_POSITION = 0, 1


class FgbDedupOptions(C.Structure):
    _fields_ = [("umi", FgbUmiOptions), ("min_map_q", C.c_uint8), ("include_non_pf", C.c_uint8),
                ("no_umi", C.c_uint8), ("remove_duplicates", C.c_uint8), ("umi_tag", C.c_char * 2),
                ("assign_tag", C.c_char * 2), ("first_mi", C.c_uint64)]


FGB_DEDUP_NSTATS = 20
DEDUP_STAT_NAMES = ("total_templates", "unique_templates", "duplicate_templates", "total_reads", "unique_reads",
                    "duplicate_reads", "secondary_reads", "supplementary_reads", "missing_tc_tag", "total_records",
                    "accepted_records", "discarded_non_pf", "discarded_poor_alignment", "discarded_ns_in_umi",
                    "discarded_umi_too_short", "position_groups", "next_mi", "records_out")


FGB_SORT_COORDINATE, FGB_SORT_TEMPLATE_COORDINATE, FGB_SORT_QUERYNAME, FGB_SORT_QUERYNAME_NATURAL = 0, 1, 2, 3


class FgbSortOptions(C.Structure):
    _fields_ = [("order", C.c_uint32), ("n_threads", C.c_uint32), ("cell_tag", C.c_char * 2),
                ("reserved", C.c_uint8 * 6), ("device_bytes", C.c_uint64)]


class FgbRecordFilterOptions(C.Structure):
    _fields_ = [("filter", FgbDuplexFilterParams), ("filter_by_template", C.c_uint8),
                ("reverse_per_base_tags", C.c_uint8), ("track_rejects", C.c_uint8), ("reserved", C.c_uint8 * 1),
                ("n_threads", C.c_uint32), ("device_bytes", C.c_uint64)]


FILTER_STAT_NAMES = ("total", "passed", "failed", "bases_masked")


class FgbZipperOptions(C.Structure):
    _fields_ = [("exclude_missing_reads", C.c_uint8), ("skip_pa_tags", C.c_uint8),
                ("restore_unconverted_bases", C.c_uint8), ("reserved", C.c_uint8 * 1), ("n_threads", C.c_uint32),
                ("device_bytes", C.c_uint64), ("n_remove", C.c_uint64), ("n_reverse", C.c_uint64),
                ("n_revcomp", C.c_uint64), ("tags_to_remove", C.c_void_p), ("tags_to_reverse", C.c_void_p),
                ("tags_to_revcomp", C.c_void_p)]


ZIPPER_STAT_NAMES = ("merged", "unmapped_only", "excluded", "records_out")


class FgbMetricsOptions(C.Structure):
    _fields_ = [("mode", C.c_uint32), ("n_threads", C.c_uint32), ("min_ab_reads", C.c_uint64),
                ("min_ba_reads", C.c_uint64), ("min_reads", C.c_uint64), ("duplex_umi_counts", C.c_uint8),
                ("reserved", C.c_uint8 * 7), ("device_bytes", C.c_uint64)]


class FgbMetricsTemplate(C.Structure):
    _fields_ = [("ref1", C.c_int32), ("start1", C.c_int32), ("ref2", C.c_int32), ("start2", C.c_int32),
                ("strand1", C.c_uint8), ("strand2", C.c_uint8), ("status", C.c_uint8), ("bucket", C.c_uint8),
                ("contig", C.c_int32), ("ins_start", C.c_int32), ("ins_end", C.c_int32), ("mi_kind", C.c_uint8),
                ("mi_canonical", C.c_uint8), ("name_ascii", C.c_uint8), ("reserved", C.c_uint8), ("r1", C.c_uint32),
                ("mi_base", C.c_uint64), ("mi_off", C.c_uint32), ("mi_len", C.c_uint32), ("rx_off", C.c_uint32),
                ("rx_len", C.c_uint32)]


METRICS_STAT_NAMES = ("records", "templates", "kept", "outside", "groups", "ds_families", "overflow", "runs")


class FgbUmiKey(C.Structure):
    _fields_ = [("bits", C.c_uint64), ("str_off", C.c_uint64), ("str_len", C.c_uint32), ("count", C.c_uint32),
                ("first", C.c_uint32), ("dash", C.c_uint32), ("len", C.c_uint8), ("flags", C.c_uint8),
                ("reserved", C.c_uint8 * 6)]


FGB_NSTATS = 24
STAT_NAMES = ("total_reads", "consensus_reads", "filtered_reads", "InsufficientReads",
              "SecondaryOrSupplementary", "ZeroLengthAfterTrimming", "MinorityAlignment",
              "OrphanConsensus", "PotentialCollision", "FragmentRead", "InsufficientOverlap",
              "IndelErrorBetweenStrands", "duplex_bases", "duplex_disagreements", "overlapping_bases",
              "overlap_bases_agreeing", "overlap_bases_disagreeing", "overlap_bases_corrected",
              "filter_records", "filter_passed", "filter_bases_masked")


class FgbCodecOut(C.Structure):
    _fields_ = [("cols", FgbColumns), ("status", C.c_void_p), ("disagreements", C.c_void_p),
                ("duplex_bases", C.c_void_p)]


# Every symbol include/fgumi_b200.h declares; tests check the .so exports all of them.
SYMBOLS = (
    "fgb_abi_version", "fgb_create", "fgb_destroy", "fgb_strerror", "fgb_last_error",
    "fgb_get_tables", "fgb_host_tables", "fgb_host_proof_tables", "fgb_host_unanimous_steps", "fgb_tile_capacity_bytes", "fgb_tile_max_units", "fgb_tile_max_reads",
    "fgb_plan_tiles", "fgb_plan_tiles_jobs", "fgb_sort_tiles_by_class", "fgb_vote_device", "fgb_vote_duplex_device", "fgb_submit", "fgb_wait", "fgb_host_alloc",
    "fgb_host_free", "fgb_host_is_pinned", "fgb_duplex_combine_device", "fgb_codec_combine_device", "fgb_stats",
    "fgb_stats_device_ptr", "fgb_stats_reset", "fgb_launch_count", "fgb_engine_caps",
    "fgb_caller_create", "fgb_caller_destroy", "fgb_caller_last_error", "fgb_caller_add_group",
    "fgb_caller_flush", "fgb_caller_take_rejects", "fgb_caller_stats", "fgb_overlap_apply_group", "fgb_pack8_encode",
    "fgb_submit_pack8", "fgb_submit_bam4", "fgb_unpack_bam4_device", "fgb_unpack_records_device", "fgb_submit_ex", "fgb_filter_simplex_device", "fgb_struct_size", "fgb_caller_add_groups", "fgb_filter_record", "fgb_host_is_fr_pair",
    "fgb_host_num_bases_extending_past_mate", "fgb_host_clip_cigar_ops", "fgb_host_read_pos_at_ref_pos", "fgb_host_simplify_cigar", "fgb_host_source_reads", "fgb_host_consensus_umis", "fgb_caller_pending", "fgb_host_simplex_record", "fgb_bgzf_bound", "fgb_bgzf_compress", "fgb_bgzf_scan_members", "fgb_bgzf_inflate_device", "fgb_host_inflate_member", "fgb_bam_header", "fgb_bgzf_uncompressed_size", "fgb_bgzf_decompress", "fgb_bam_read_header", "fgb_bam_split_records", "fgb_host_group_by_mi", "fgb_host_duplex_record",
    "fgb_umi_assign", "fgb_host_umi_for_read", "fgb_host_umi_prepare", "fgb_host_umi_resolve",
    "fgb_umi_edges", "fgb_umi_last_timing",
    "fgb_host_group_by_position", "fgb_grouper_create", "fgb_grouper_destroy", "fgb_grouper_last_error",
    "fgb_grouper_add_groups", "fgb_grouper_pending", "fgb_grouper_flush", "fgb_grouper_flush_with_ids",
    "fgb_grouper_stats", "fgb_grouper_histogram", "fgb_grouper_last_timing",
    "fgb_sort_records", "fgb_host_sort_keys", "fgb_host_sort_verify", "fgb_sort_last_timing", "fgb_host_sort_name_key",
    "fgb_host_dedup_group_by_position", "fgb_deduper_create", "fgb_deduper_destroy", "fgb_deduper_last_error",
    "fgb_deduper_add_groups", "fgb_deduper_pending", "fgb_deduper_flush", "fgb_deduper_flush_with_ids",
    "fgb_deduper_stats", "fgb_deduper_histogram", "fgb_deduper_last_timing", "fgb_record_quality_scores",
    "fgb_reference_create", "fgb_reference_destroy", "fgb_reference_contigs", "fgb_reference_contig",
    "fgb_filter_records", "fgb_filter_last_timing",
    "fgb_host_metrics_templates", "fgb_host_metrics_name_fraction", "fgb_host_metrics_bucket",
    "fgb_host_metrics_intervals", "fgb_host_metrics_format_float", "fgb_metrics_create", "fgb_metrics_destroy",
    "fgb_metrics_last_error", "fgb_metrics_add_records", "fgb_metrics_finish", "fgb_metrics_table",
    "fgb_metrics_stats", "fgb_metrics_last_timing",
    "fgb_zipper_records", "fgb_host_zipper_records", "fgb_host_free_buffer", "fgb_zipper_last_timing",
)

_lib = None


class FgbError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str = ""):
        self.status = status
        msg = f"{where}: fgb_status {status}"
        try:
            msg += f" ({load().fgb_strerror(status).decode()})"
        except Exception:  # pragma: no cover
            pass
        if detail:
            msg += f": {detail}"
        super().__init__(msg)


def load() -> C.CDLL:
    """dlopen libfgumi_b200.so and declare prototypes.  Raises if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  fgumi_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
    lib.fgb_abi_version.restype = u32
    lib.fgb_create.argtypes = [C.c_int, C.POINTER(FgbParams), C.POINTER(vp)]
    lib.fgb_create.restype = C.c_int32
    lib.fgb_destroy.argtypes = [vp]
    lib.fgb_destroy.restype = None
    lib.fgb_strerror.argtypes = [C.c_int32]
    lib.fgb_strerror.restype = C.c_char_p
    lib.fgb_last_error.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.fgb_last_error.restype = C.c_size_t
    lib.fgb_get_tables.argtypes = [vp, vp, vp, vp, vp]
    lib.fgb_get_tables.restype = C.c_int32
    lib.fgb_host_tables.argtypes = [C.c_uint8, C.c_uint8, vp, vp, vp, vp, vp, vp]
    lib.fgb_host_tables.restype = C.c_int32
    lib.fgb_host_proof_tables.argtypes = [C.c_uint8, C.c_uint8, vp, vp, vp]
    lib.fgb_host_proof_tables.restype = C.c_int32
    lib.fgb_host_unanimous_steps.argtypes = [C.c_uint8, C.c_uint8, vp, vp, vp, vp]
    lib.fgb_host_unanimous_steps.restype = C.c_int32
    for f in ("fgb_tile_capacity_bytes", "fgb_tile_max_units", "fgb_tile_max_reads"):
        getattr(lib, f).restype = u32
        getattr(lib, f).argtypes = []
    lib.fgb_plan_tiles.argtypes = [vp, u64, vp, u64, vp, u64, C.POINTER(u64)]
    lib.fgb_plan_tiles.restype = C.c_int32
    lib.fgb_plan_tiles_jobs.argtypes = [vp, u64, vp, u64, vp, u64, vp, u64, C.POINTER(u64), vp, vp, vp, C.POINTER(u64)]
    lib.fgb_plan_tiles_jobs.restype = C.c_int32
    lib.fgb_vote_duplex_device.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbColumns), vp, u64, vp, vp,
                                           C.POINTER(FgbDuplexOut), vp]
    lib.fgb_vote_duplex_device.restype = C.c_int32
    lib.fgb_bgzf_scan_members.argtypes = [vp, C.c_size_t, vp, u64, C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_bgzf_scan_members.restype = C.c_int32
    lib.fgb_bgzf_inflate_device.argtypes = [vp, vp, vp, u64, vp, vp, C.c_int, vp, vp]
    lib.fgb_bgzf_inflate_device.restype = C.c_int32
    lib.fgb_host_inflate_member.argtypes = [vp, u32, vp, u32]
    lib.fgb_host_inflate_member.restype = u32
    lib.fgb_sort_tiles_by_class.argtypes = [vp, u64, vp]
    lib.fgb_sort_tiles_by_class.restype = C.c_int32
    lib.fgb_vote_device.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbColumns), vp]
    lib.fgb_vote_device.restype = C.c_int32
    lib.fgb_submit.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbColumns)]
    lib.fgb_submit.restype = C.c_int32
    lib.fgb_wait.argtypes = [vp]
    lib.fgb_wait.restype = C.c_int32
    lib.fgb_host_alloc.argtypes = [C.POINTER(vp), C.c_size_t]
    lib.fgb_host_alloc.restype = C.c_int32
    lib.fgb_host_free.argtypes = [vp]
    lib.fgb_host_free.restype = None
    lib.fgb_host_is_pinned.argtypes = [vp]
    lib.fgb_host_is_pinned.restype = C.c_int
    lib.fgb_duplex_combine_device.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbColumns), vp,
                                              u64, C.POINTER(FgbDuplexOut), vp]
    lib.fgb_duplex_combine_device.restype = C.c_int32
    lib.fgb_codec_combine_device.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbColumns), vp,
                                             u64, C.POINTER(FgbCodecParams),
                                             C.POINTER(FgbCodecOut), vp]
    lib.fgb_codec_combine_device.restype = C.c_int32
    lib.fgb_stats.argtypes = [vp, C.POINTER(u64)]
    lib.fgb_stats.restype = C.c_int32
    lib.fgb_stats_device_ptr.argtypes = [vp, C.POINTER(vp)]
    lib.fgb_stats_device_ptr.restype = C.c_int32
    lib.fgb_stats_reset.argtypes = [vp]
    lib.fgb_stats_reset.restype = C.c_int32
    lib.fgb_launch_count.argtypes = [vp]
    lib.fgb_launch_count.restype = u64
    lib.fgb_engine_caps.argtypes = []
    lib.fgb_engine_caps.restype = u32
    lib.fgb_caller_create.argtypes = [C.c_int, C.POINTER(FgbCallerOptions), C.POINTER(vp)]
    lib.fgb_caller_create.restype = C.c_int32
    lib.fgb_caller_destroy.argtypes = [vp]
    lib.fgb_caller_destroy.restype = None
    lib.fgb_caller_last_error.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.fgb_caller_last_error.restype = C.c_size_t
    lib.fgb_caller_add_group.argtypes = [vp, vp, vp, u32]
    lib.fgb_caller_add_group.restype = C.c_int32
    lib.fgb_caller_flush.argtypes = [vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_caller_flush.restype = C.c_int32
    lib.fgb_caller_take_rejects.argtypes = [vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_caller_take_rejects.restype = C.c_int32
    lib.fgb_caller_stats.argtypes = [vp, C.POINTER(u64)]
    lib.fgb_caller_stats.restype = C.c_int32
    lib.fgb_overlap_apply_group.argtypes = [vp, vp, C.c_uint32, C.c_uint8, C.c_uint8, vp]
    lib.fgb_overlap_apply_group.restype = C.c_int32
    lib.fgb_pack8_encode.argtypes = [vp, vp, u64, vp]
    lib.fgb_pack8_encode.restype = C.c_int32
    lib.fgb_submit_pack8.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbColumns)]
    lib.fgb_submit_pack8.restype = C.c_int32
    lib.fgb_submit_bam4.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbRawColumns), C.POINTER(FgbColumns)]
    lib.fgb_submit_bam4.restype = C.c_int32
    lib.fgb_unpack_bam4_device.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbRawColumns), vp, vp, vp]
    lib.fgb_unpack_bam4_device.restype = C.c_int32
    lib.fgb_unpack_records_device.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbRecordColumns), vp, vp, vp]
    lib.fgb_unpack_records_device.restype = C.c_int32
    lib.fgb_submit_ex.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbColumns), C.POINTER(FgbSubmitOptions)]
    lib.fgb_submit_ex.restype = C.c_int32
    lib.fgb_filter_simplex_device.argtypes = [vp, C.POINTER(FgbBatch), C.POINTER(FgbColumns),
                                              C.POINTER(FgbFilterParams), vp, vp, vp]
    lib.fgb_filter_simplex_device.restype = C.c_int32
    lib.fgb_filter_record.argtypes = [vp, C.c_size_t, C.POINTER(FgbDuplexFilterParams), vp, vp]
    lib.fgb_filter_record.restype = C.c_int32
    lib.fgb_host_is_fr_pair.argtypes = [vp, C.c_size_t]
    lib.fgb_host_is_fr_pair.restype = C.c_int
    lib.fgb_host_num_bases_extending_past_mate.argtypes = [vp, C.c_size_t]
    lib.fgb_host_num_bases_extending_past_mate.restype = u32
    lib.fgb_host_clip_cigar_ops.argtypes = [vp, u32, u32, C.c_int, vp, vp, vp]
    lib.fgb_host_clip_cigar_ops.restype = C.c_int32
    lib.fgb_host_read_pos_at_ref_pos.argtypes = [vp, u32, u64, u64, C.c_int, vp]
    lib.fgb_host_read_pos_at_ref_pos.restype = C.c_int
    lib.fgb_host_simplify_cigar.argtypes = [vp, u32, vp, vp, vp]
    lib.fgb_host_simplify_cigar.restype = C.c_int32
    lib.fgb_host_source_reads.argtypes = [vp, vp, u32, C.c_uint8, C.c_int, vp, vp, vp, vp, vp, vp]
    lib.fgb_host_source_reads.restype = C.c_int32
    lib.fgb_host_consensus_umis.argtypes = [vp, u32, vp, C.c_size_t]
    lib.fgb_host_consensus_umis.restype = C.c_int32
    lib.fgb_host_simplex_record.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint8, C.c_int, vp, vp, vp, vp, u32,
                                            C.c_char_p, C.c_char_p, vp, u32, vp, C.c_size_t, vp]
    lib.fgb_host_simplex_record.restype = C.c_int32
    lib.fgb_host_duplex_record.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, C.c_int, vp, vp, vp, u32,
                                           C.POINTER(FgbStrandColumns), C.POINTER(FgbStrandColumns), C.c_char_p,
                                           C.c_char_p, vp, vp, u32, vp, C.c_size_t, vp]
    lib.fgb_host_duplex_record.restype = C.c_int32
    lib.fgb_host_group_by_mi.argtypes = [vp, vp, u64, C.c_char_p, C.c_int, C.c_char_p, vp, vp, vp]
    lib.fgb_host_group_by_mi.restype = C.c_int32
    lib.fgb_bgzf_bound.argtypes = [C.c_size_t]
    lib.fgb_bgzf_bound.restype = C.c_size_t
    lib.fgb_bgzf_compress.argtypes = [vp, C.c_size_t, C.c_int, u32, C.c_int, vp, C.c_size_t, vp]
    lib.fgb_bgzf_compress.restype = C.c_int32
    lib.fgb_bgzf_uncompressed_size.argtypes = [vp, C.c_size_t, vp]
    lib.fgb_bgzf_uncompressed_size.restype = C.c_int32
    lib.fgb_bgzf_decompress.argtypes = [vp, C.c_size_t, u32, vp, C.c_size_t, vp]
    lib.fgb_bgzf_decompress.restype = C.c_int32
    lib.fgb_bam_read_header.argtypes = [vp, C.c_size_t, vp, vp, vp, vp]
    lib.fgb_bam_read_header.restype = C.c_int32
    lib.fgb_bam_split_records.argtypes = [vp, C.c_size_t, vp, vp, u64, vp, vp]
    lib.fgb_bam_split_records.restype = C.c_int32
    lib.fgb_bam_header.argtypes = [C.c_char_p, C.c_size_t, vp, C.c_size_t, vp]
    lib.fgb_bam_header.restype = C.c_int32
    lib.fgb_caller_pending.argtypes = [vp, C.POINTER(FgbBatch), vp, vp, vp, vp]
    lib.fgb_caller_pending.restype = C.c_int32
    lib.fgb_caller_add_groups.argtypes = [vp, vp, vp, vp, u64]
    lib.fgb_caller_add_groups.restype = C.c_int32
    lib.fgb_umi_assign.argtypes = [vp, C.POINTER(FgbUmiOptions), vp, vp, u64, vp, u64, vp, u64, vp, vp, vp]
    lib.fgb_umi_assign.restype = C.c_int32
    lib.fgb_host_umi_for_read.argtypes = [C.POINTER(FgbUmiOptions), C.c_char_p, C.c_size_t, C.c_int, vp, C.c_size_t,
                                          C.POINTER(C.c_size_t)]
    lib.fgb_host_umi_for_read.restype = C.c_int32
    lib.fgb_host_umi_prepare.argtypes = [C.POINTER(FgbUmiOptions), vp, vp, u64, vp, C.POINTER(u64), vp, vp]
    lib.fgb_host_umi_prepare.restype = C.c_int32
    lib.fgb_host_umi_resolve.argtypes = [C.POINTER(FgbUmiOptions), vp, vp, u64, vp, u64, vp, vp, vp, vp, vp, vp]
    lib.fgb_host_umi_resolve.restype = C.c_int32
    lib.fgb_umi_edges.argtypes = [vp, C.POINTER(FgbUmiOptions), vp, vp, u64, C.POINTER(u64), vp, vp, u64,
                                  C.POINTER(u64)]
    lib.fgb_umi_edges.restype = C.c_int32
    lib.fgb_umi_last_timing.argtypes = [vp, vp]
    lib.fgb_umi_last_timing.restype = C.c_int32
    lib.fgb_host_group_by_position.argtypes = [vp, vp, u64, C.c_char_p, C.c_size_t, C.c_char_p, vp, vp,
                                               C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_host_group_by_position.restype = C.c_int32
    lib.fgb_grouper_create.argtypes = [C.c_int, C.POINTER(FgbGroupOptions), C.POINTER(vp)]
    lib.fgb_grouper_create.restype = C.c_int32
    lib.fgb_grouper_destroy.argtypes = [vp]
    lib.fgb_grouper_destroy.restype = None
    lib.fgb_grouper_last_error.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.fgb_grouper_last_error.restype = C.c_size_t
    lib.fgb_grouper_add_groups.argtypes = [vp, vp, vp, vp, u64]
    lib.fgb_grouper_add_groups.restype = C.c_int32
    lib.fgb_grouper_pending.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(u64), C.POINTER(vp),
                                        C.POINTER(u64), C.POINTER(vp), C.POINTER(u64)]
    lib.fgb_grouper_pending.restype = C.c_int32
    lib.fgb_grouper_flush.argtypes = [vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_grouper_flush.restype = C.c_int32
    lib.fgb_grouper_flush_with_ids.argtypes = [vp, vp, vp, vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_grouper_flush_with_ids.restype = C.c_int32
    lib.fgb_grouper_stats.argtypes = [vp, vp]
    lib.fgb_grouper_stats.restype = C.c_int32
    lib.fgb_grouper_histogram.argtypes = [vp, C.c_int, vp, vp, u64, C.POINTER(u64)]
    lib.fgb_grouper_histogram.restype = C.c_int32
    lib.fgb_grouper_last_timing.argtypes = [vp, vp]
    lib.fgb_grouper_last_timing.restype = C.c_int32
    lib.fgb_host_dedup_group_by_position.argtypes = [vp, vp, u64, C.c_char_p, C.c_size_t, C.c_char_p, vp, vp,
                                                     C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_host_dedup_group_by_position.restype = C.c_int32
    lib.fgb_deduper_create.argtypes = [C.c_int, C.POINTER(FgbDedupOptions), C.POINTER(vp)]
    lib.fgb_deduper_create.restype = C.c_int32
    lib.fgb_deduper_destroy.argtypes = [vp]
    lib.fgb_deduper_destroy.restype = None
    lib.fgb_deduper_last_error.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.fgb_deduper_last_error.restype = C.c_size_t
    lib.fgb_deduper_add_groups.argtypes = [vp, vp, vp, vp, u64]
    lib.fgb_deduper_add_groups.restype = C.c_int32
    lib.fgb_deduper_pending.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(u64), C.POINTER(vp),
                                        C.POINTER(u64), C.POINTER(vp), C.POINTER(u64)]
    lib.fgb_deduper_pending.restype = C.c_int32
    lib.fgb_deduper_flush.argtypes = [vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_deduper_flush.restype = C.c_int32
    lib.fgb_deduper_flush_with_ids.argtypes = [vp, vp, vp, vp, vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_deduper_flush_with_ids.restype = C.c_int32
    lib.fgb_deduper_stats.argtypes = [vp, vp]
    lib.fgb_deduper_stats.restype = C.c_int32
    lib.fgb_deduper_histogram.argtypes = [vp, vp, vp, u64, C.POINTER(u64)]
    lib.fgb_deduper_histogram.restype = C.c_int32
    lib.fgb_deduper_last_timing.argtypes = [vp, vp]
    lib.fgb_deduper_last_timing.restype = C.c_int32
    lib.fgb_record_quality_scores.argtypes = [vp, vp, vp, u64, vp]
    lib.fgb_record_quality_scores.restype = C.c_int32
    lib.fgb_sort_records.argtypes = [vp, C.POINTER(FgbSortOptions), C.c_char_p, C.c_size_t, vp, vp, u64, vp, u64,
                                     C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_sort_records.restype = C.c_int32
    lib.fgb_host_sort_keys.argtypes = [C.POINTER(FgbSortOptions), C.c_char_p, C.c_size_t, vp, vp, u64, vp,
                                       C.POINTER(u64)]
    lib.fgb_host_sort_keys.restype = C.c_int32
    lib.fgb_host_sort_verify.argtypes = [C.POINTER(FgbSortOptions), C.c_char_p, C.c_size_t, vp, vp, u64,
                                         C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_host_sort_verify.restype = C.c_int32
    lib.fgb_host_sort_name_key.argtypes = [C.POINTER(FgbSortOptions), vp, u64, vp, u32, C.POINTER(u32)]
    lib.fgb_host_sort_name_key.restype = C.c_int32
    lib.fgb_sort_last_timing.argtypes = [vp, vp]
    lib.fgb_sort_last_timing.restype = C.c_int32
    lib.fgb_reference_create.argtypes = [C.c_int, vp, C.c_size_t, C.POINTER(vp)]
    lib.fgb_reference_create.restype = C.c_int32
    lib.fgb_reference_destroy.argtypes = [vp]
    lib.fgb_reference_destroy.restype = None
    lib.fgb_reference_contigs.argtypes = [vp]
    lib.fgb_reference_contigs.restype = u64
    lib.fgb_reference_contig.argtypes = [vp, u64, C.POINTER(C.c_char_p), C.POINTER(u64)]
    lib.fgb_reference_contig.restype = C.c_int32
    lib.fgb_filter_records.argtypes = [vp, C.POINTER(FgbRecordFilterOptions), vp, C.c_char_p, C.c_size_t, vp, vp, u64,
                                       C.POINTER(vp), C.POINTER(u64), C.POINTER(vp), C.POINTER(u64), vp,
                                       C.POINTER(u64)]
    lib.fgb_filter_records.restype = C.c_int32
    lib.fgb_filter_last_timing.argtypes = [vp, vp]
    lib.fgb_filter_last_timing.restype = C.c_int32
    lib.fgb_host_metrics_templates.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, vp, vp, u64, vp, u64,
                                               C.POINTER(u64), C.POINTER(u64)]
    lib.fgb_host_metrics_templates.restype = C.c_int32
    lib.fgb_host_metrics_name_fraction.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int32),
                                                   C.POINTER(C.c_double), C.POINTER(u32)]
    lib.fgb_host_metrics_name_fraction.restype = C.c_int32
    lib.fgb_host_metrics_bucket.argtypes = [C.c_int32]
    lib.fgb_host_metrics_bucket.restype = u32
    lib.fgb_host_metrics_intervals.argtypes = [C.c_char_p, C.c_size_t, vp, vp, vp, vp, u64, C.POINTER(u64)]
    lib.fgb_host_metrics_intervals.restype = C.c_int32
    lib.fgb_host_metrics_format_float.argtypes = [C.c_double, C.c_char_p, C.c_size_t]
    lib.fgb_host_metrics_format_float.restype = C.c_size_t
    lib.fgb_metrics_create.argtypes = [C.c_int, C.POINTER(FgbMetricsOptions), C.c_char_p, C.c_size_t, C.c_char_p,
                                       C.c_size_t, C.POINTER(vp)]
    lib.fgb_metrics_create.restype = C.c_int32
    lib.fgb_metrics_destroy.argtypes = [vp]
    lib.fgb_metrics_destroy.restype = None
    lib.fgb_metrics_last_error.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.fgb_metrics_last_error.restype = C.c_size_t
    lib.fgb_metrics_add_records.argtypes = [vp, vp, vp, u64, C.POINTER(u64)]
    lib.fgb_metrics_add_records.restype = C.c_int32
    lib.fgb_metrics_finish.argtypes = [vp, C.POINTER(u64)]
    lib.fgb_metrics_finish.restype = C.c_int32
    lib.fgb_metrics_table.argtypes = [vp, u32, C.POINTER(C.c_char_p), C.POINTER(u64)]
    lib.fgb_metrics_table.restype = C.c_int32
    lib.fgb_metrics_stats.argtypes = [vp, vp]
    lib.fgb_metrics_stats.restype = C.c_int32
    lib.fgb_metrics_last_timing.argtypes = [vp, vp]
    lib.fgb_metrics_last_timing.restype = C.c_int32
    lib.fgb_zipper_records.argtypes = [vp, C.POINTER(FgbZipperOptions), vp, vp, u64, vp, vp, u64, C.c_int,
                                       C.POINTER(vp), C.POINTER(u64), C.POINTER(u64), vp, C.POINTER(u64)]
    lib.fgb_zipper_records.restype = C.c_int32
    lib.fgb_host_zipper_records.argtypes = [C.POINTER(FgbZipperOptions), vp, vp, u64, vp, vp, u64, C.c_int,
                                            C.POINTER(vp), C.POINTER(u64), C.POINTER(u64), vp, C.POINTER(u64)]
    lib.fgb_host_zipper_records.restype = C.c_int32
    lib.fgb_host_free_buffer.argtypes = [vp]
    lib.fgb_host_free_buffer.restype = None
    lib.fgb_zipper_last_timing.argtypes = [vp, vp]
    lib.fgb_zipper_last_timing.restype = C.c_int32
    lib.fgb_struct_size.argtypes = [C.c_uint32]
    lib.fgb_struct_size.restype = C.c_uint32
    _lib = lib
    return lib
