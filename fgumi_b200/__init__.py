"""fgumi_b200 — Hopper-native UMI consensus engine (drop-in for fgumi's consensus hot path).

The product is libfgumi_b200.so (hand-written sm_90a CUDA behind the C-ABI in
include/fgumi_b200.h).  This package is the thin host-side mirror of that boundary.
"""
from .engine import (Engine, PackedBatch, HostColumns, DeviceBatch, DeviceColumns,  # noqa: F401
                     VanillaUmiConsensusOptions, pack_source_reads, pack_uniform, plan_tiles, pack8_encode,
                     pack_raw_reads, RawColumns, RAW_READ_DTYPE,
                     consensus_length, UNIT_DTYPE, TILE_DTYPE, DUPLEX_JOB_DTYPE, CODEC_JOB_DTYPE,
                     TILE_JOBS_DTYPE, plan_tiles_jobs)
from . import lib  # noqa: F401
from .caller import VanillaUmiConsensusCaller, DuplexConsensusCaller, CodecConsensusCaller, ConsensusOutput, ConsensusFilter, DuplexConsensusFilter, apply_overlapping_consensus, bgzf_compress, write_bam  # noqa: F401
from .umi import UmiAssigner, UmiAssignment  # noqa: F401

__version__ = "0.1.0"
