"""The host half of the three record-level callers WITHOUT a GPU: a planning-only caller
(fgb_caller_create(FGB_DEVICE_NONE)) runs the product's group rules and source-read preparation and
queues the packed batch; per MI group its units (source rows in order, consensus length) must equal
what the oracle caller hands to its vote hook, and flushing must fail loudly (no CPU fallback)."""
import os
import sys

import ctypes as C

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import record_oracle as R           # noqa: E402
from tests import oracle_lib as O               # noqa: E402
from tests.test_record_oracle_kat import vote_fn   # noqa: E402
from tests.test_caller_parity import random_groups, random_duplex_groups, random_codec_groups, duplex_job_fn   # noqa: E402
from tests.test_codec_oracle_kat import codec_job_fn   # noqa: E402


class Capture:
    """Wraps the oracle's vote hook and records the row lists it is called with."""

    def __init__(self):
        self.calls = []

    def __call__(self, rows, opt):
        self.calls.append(([(bytes(b), bytes(q)) for b, q in rows], opt.min_reads))
        return vote_fn(rows, opt)


def _cons_len(rows, min_reads):
    return sorted((len(b) for b, _ in rows), reverse=True)[min_reads - 1]


def _compare_groups(fg, product, oracle_call, cap, groups, unordered=False, orphans=None):
    """`orphans`: callable returning the oracle's running OrphanConsensus count.  The simplex oracle
    votes R1 / R2 sub-groups one by one and only then drops a pair whose mate has no consensus; the
    product knows that at planning time and does not queue the lone sub-group -- so its units may be
    a subsequence of the oracle's vote calls, with the difference explained by orphan rejections."""
    n_units = n_skipped = 0
    for g in groups:
        cap.calls.clear()
        o0 = orphans() if orphans else 0
        n_out = oracle_call(g)
        before = len(product.pending()["units"])
        product.add_group(g)
        units = product.pending()["units"][before:]
        want = [(rows, _cons_len(rows, mr)) for rows, mr in cap.calls]
        got = [(u["rows"], u["cons_len"]) for u in units]
        if unordered:
            key = lambda t: (t[1], t[0])
            got, want = sorted(got, key=key), sorted(want, key=key)
        if orphans and len(got) < len(want):
            it = iter(want)
            assert all(any(x == y for y in it) for x in got), "units are not a subsequence of the oracle's calls"
            assert orphans() > o0
            n_skipped += len(want) - len(got)
        elif unordered and len(got) < len(want):
            # duplex / CODEC: the oracle votes strand by strand and may only then find that the molecule
            # cannot be completed; the product sees that while planning and queues nothing for it
            assert got == [] and n_out == 0, (len(got), len(want), n_out)
            n_skipped += len(want)
        else:
            assert got == want
        n_units += len(got)
    return n_units, n_skipped


def test_planning_only_caller_refuses_to_flush():
    import fgumi_b200 as fg
    c = fg.VanillaUmiConsensusCaller("fgumi", "A", device=fg.lib.FGB_DEVICE_NONE)
    c.add_group(random_groups(np.random.default_rng(1), 3)[0])
    with pytest.raises(fg.lib.FgbError) as e:
        c.flush()
    assert e.value.status == fg.lib.FGB_ERR_NO_DEVICE
    c.close()


@pytest.mark.parametrize("min_reads,trim,overlap", [(1, False, False), (2, True, False), (1, False, True)])
def test_simplex_host_prep_matches_oracle(min_reads, trim, overlap):
    import fgumi_b200 as fg
    rng = np.random.default_rng(31 + min_reads)
    groups = random_groups(rng, 200)
    cap = Capture()
    oracle = R.VanillaCallerOracle("fgumi", "A", R.VanillaOptions(min_reads=min_reads, trim=trim), cap, O.builder_call)
    ov = R.OverlappingOracle() if overlap else None

    def call(g):
        if ov is not None:
            recs = [bytearray(r) for r in g]
            ov.apply(recs)
            g = [bytes(r) for r in recs]
        oracle.consensus_reads(g)
    opts = fg.VanillaUmiConsensusOptions(min_reads=min_reads, trim=trim)
    c = fg.VanillaUmiConsensusCaller("fgumi", "A", opts, device=fg.lib.FGB_DEVICE_NONE,
                                     consensus_call_overlapping_bases=overlap)
    n, skipped = _compare_groups(fg, c, call, cap, groups,
                                 orphans=lambda: oracle.stats.rejections.get("OrphanConsensus", 0))
    st = c.statistics()
    c.close()
    assert n > 150 and skipped > 0 and st["total_reads"] == sum(len(g) for g in groups)
    # every simplex decision is taken while planning: all counters already equal the oracle's
    o = oracle.stats
    assert st["total_reads"] == o.total_reads and st["consensus_reads"] == o.consensus_reads
    assert st["filtered_reads"] == o.filtered_reads
    for name in ("InsufficientReads", "SecondaryOrSupplementary", "ZeroLengthAfterTrimming", "MinorityAlignment",
                 "OrphanConsensus"):
        assert st[name] == o.rejections.get(name, 0), name
    assert o.rejections.get("MinorityAlignment", 0) > 0 and o.rejections.get("OrphanConsensus", 0) > 0
    if overlap:
        assert (st["overlapping_bases"], st["overlap_bases_agreeing"], st["overlap_bases_disagreeing"],
                st["overlap_bases_corrected"]) == ov.stats()


@pytest.mark.parametrize("min_reads,overlap,threads", [(1, False, 1), (2, False, 6), (2, True, 1), (3, True, 6)])
def test_simplex_rejected_reads_on_the_device_source_read_path(min_reads, overlap, threads):
    """The same stream from the path device callers take (records staged and shipped whole, rows built on the device:
    direct_add / plan_subgroup), run here over the CPU mock engine (oracle/libfgb_cpu_caller.so): rejected reads equal
    the record oracle's -- with the overlapping-bases pre-pass on, the reads as the pre-pass leaves them -- a failing
    call rolls its rejects back, and the consensus output is the one a caller without the option produces."""
    import fgumi_b200 as fg
    from tests.bam_builder import make_record
    L = fg.lib
    O.build()
    os.environ["FGB_CPU_THREADS"] = "4"
    cpu = C.CDLL(O.SO_CPU_CALLER)
    vp, u64 = C.c_void_p, C.c_uint64
    cpu.fgb_caller_create.argtypes = [C.c_int, C.POINTER(L.FgbCallerOptions), C.POINTER(vp)]
    cpu.fgb_caller_add_groups.argtypes = [vp, vp, vp, vp, u64]
    cpu.fgb_caller_flush.argtypes = [vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    cpu.fgb_caller_take_rejects.argtypes = [vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    cpu.fgb_caller_destroy.argtypes = [vp]
    rng = np.random.default_rng(81 + min_reads)
    groups = random_groups(rng, 240)

    def table(gs):
        recs = [r for g in gs for r in g]
        blob = np.frombuffer(b"".join(recs), np.uint8).copy()
        off = np.zeros(len(recs) + 1, dtype=np.uint64); off[1:] = np.cumsum([len(r) for r in recs])
        grp = np.zeros(len(gs) + 1, dtype=np.uint64); grp[1:] = np.cumsum([len(g) for g in gs])
        return blob, off, grp

    def make(track):
        o = L.FgbCallerOptions()
        o.mode = 0; o.error_rate_pre_umi = 45; o.error_rate_post_umi = 40; o.min_input_base_quality = 10
        o.min_consensus_base_quality = 2; o.produce_per_base_tags = 1; o.min_reads = min_reads
        o.consensus_call_overlapping_bases = int(overlap); o.n_threads = threads; o.track_rejects = int(track)
        o.tag = b"MI"; o.cell_tag = b"\0\0"; o.read_name_prefix = b"fgumi"; o.read_group_id = b"A"
        h = vp()
        assert cpu.fgb_caller_create(0, C.byref(o), C.byref(h)) == 0
        return h

    def take(h):
        d, n, cnt = vp(), u64(), u64()
        assert cpu.fgb_caller_take_rejects(h, C.byref(d), C.byref(n), C.byref(cnt)) == 0
        raw = C.string_at(d.value, n.value) if n.value else b""
        out, p = [], 0
        while p < len(raw):
            k = int.from_bytes(raw[p:p + 4], "little")
            out.append(raw[p + 4:p + 4 + k]); p += 4 + k
        assert len(out) == cnt.value
        return out

    def flush(h):
        d, n, cnt = vp(), u64(), u64()
        assert cpu.fgb_caller_flush(h, C.byref(d), C.byref(n), C.byref(cnt)) == 0
        return C.string_at(d.value, n.value) if n.value else b""

    oracle = R.VanillaCallerOracle("fgumi", "A", R.VanillaOptions(min_reads=min_reads), Capture(), O.builder_call, track_rejects=True)
    ov = R.OverlappingOracle() if overlap else None
    for g in groups:
        if ov is not None:
            recs = [bytearray(r) for r in g]
            ov.apply(recs)
            g = [bytes(r) for r in recs]
        oracle.consensus_reads(g)
    h = make(True)
    blob, off, grp = table(groups[:90])
    assert cpu.fgb_caller_add_groups(h, blob.ctypes.data, off.ctypes.data, grp.ctypes.data, 90) == 0
    got = take(h)
    # a failing call in between: nothing of it stays, rejects included
    bad = [make_record(name=b"x", flags=0, pos=5, seq=b"ACGTACGTAC", quals=bytes([30] * 10), tags=[(b"MI", "Z", b"9")])[:20]]
    bblob, boff, bgrp = table(groups[90:150] + [bad] + groups[150:160])
    assert cpu.fgb_caller_add_groups(h, bblob.ctypes.data, boff.ctypes.data, bgrp.ctypes.data, len(bgrp) - 1) != 0
    assert take(h) == []
    blob2, off2, grp2 = table(groups[90:])
    assert cpu.fgb_caller_add_groups(h, blob2.ctypes.data, off2.ctypes.data, grp2.ctypes.data, len(groups) - 90) == 0
    got += take(h)
    assert len(oracle.rejected_reads) > 40 and got == oracle.rejected_reads
    out_tracked = flush(h)
    cpu.fgb_caller_destroy(h)
    h2 = make(False)
    ball, oall, gall = table(groups)
    assert cpu.fgb_caller_add_groups(h2, ball.ctypes.data, oall.ctypes.data, gall.ctypes.data, len(groups)) == 0
    assert take(h2) == []
    assert flush(h2) == out_tracked and len(out_tracked) > 10000
    cpu.fgb_caller_destroy(h2)


@pytest.mark.parametrize("min_reads,trim,threads", [(1, False, 1), (2, True, 1), (3, False, 5), (2, False, 5)])
def test_simplex_rejected_reads_match_oracle(min_reads, trim, threads):
    """options.track_rejects: the raw bytes of every rejected read, in the order the reference's reject sites run
    (vanilla_caller.rs:752-754, 1061-1063, 1095-1105, 1137-1142, 1170-1209), against the record oracle's restatement
    -- every site is hit by these groups (the statistics say so), with one thread and with the groups spread over
    five; a take in the middle splits the stream without losing or repeating a record."""
    import fgumi_b200 as fg
    rng = np.random.default_rng(71 + min_reads)
    groups = random_groups(rng, 260)
    oracle = R.VanillaCallerOracle("fgumi", "A", R.VanillaOptions(min_reads=min_reads, trim=trim), Capture(), O.builder_call,
                                   track_rejects=True)
    for g in groups:
        oracle.consensus_reads(g)
    want = oracle.rejected_reads
    c = fg.VanillaUmiConsensusCaller("fgumi", "A", fg.VanillaUmiConsensusOptions(min_reads=min_reads, trim=trim),
                                     device=fg.lib.FGB_DEVICE_NONE, n_threads=threads, track_rejects=True)
    c.add_groups(groups[:100])
    got = c.take_rejects()
    assert c.take_rejects() == []                                   # taken means gone
    c.add_groups(groups[100:])
    got += c.take_rejects()
    st = c.statistics()
    c.close()
    assert len(want) > 50 and st["filtered_reads"] == len(want) == oracle.stats.filtered_reads
    assert got == want
    rej = oracle.stats.rejections
    assert rej.get("SecondaryOrSupplementary", 0) > 0 and rej.get("MinorityAlignment", 0) > 0 and rej.get("OrphanConsensus", 0) > 0
    assert min_reads == 1 or rej.get("InsufficientReads", 0) > 0
    # callers without the option keep nothing; the other modes refuse it
    plain = fg.VanillaUmiConsensusCaller("fgumi", "A", device=fg.lib.FGB_DEVICE_NONE)
    plain.add_groups(groups[:50])
    assert plain.take_rejects() == []
    plain.close()
    with pytest.raises(fg.lib.FgbError):
        o = fg.lib.FgbCallerOptions()
        o.mode, o.track_rejects, o.min_reads, o.min_xy_reads, o.tag, o.cell_tag = 1, 1, 1, 1, b"MI", b"\0\0"
        o.error_rate_pre_umi, o.error_rate_post_umi, o.min_input_base_quality, o.min_consensus_base_quality = 45, 40, 10, 2
        h = C.c_void_p()
        st = fg.lib.load().fgb_caller_create(fg.lib.FGB_DEVICE_NONE, C.byref(o), C.byref(h))
        if st != 0:
            raise fg.lib.FgbError(st, "fgb_caller_create")


@pytest.mark.parametrize("min_reads", [(1, 1, 1), (2, 1, 0), (3, 2, 1)])
def test_duplex_host_prep_matches_oracle(min_reads):
    import fgumi_b200 as fg
    rng = np.random.default_rng(77 + sum(min_reads))
    groups = random_duplex_groups(rng, 150)
    cap = Capture()
    oracle = R.DuplexCallerOracle("fgumi", "A", min_reads=min_reads, per_base=True, vote_fn=cap,
                                  builder_fn=O.builder_call, duplex_job_fn=duplex_job_fn)
    c = fg.DuplexConsensusCaller("fgumi", "A", min_reads=min_reads, device=fg.lib.FGB_DEVICE_NONE)
    n, _ = _compare_groups(fg, c, lambda g: oracle.consensus_reads(g)[1], cap, groups, unordered=True)
    pend = c.pending()
    st = c.statistics()
    c.close()
    assert n > 200 and len(pend["duplex_jobs"]) > 50
    assert st["total_reads"] == oracle.stats.total_reads
    assert st["PotentialCollision"] == oracle.stats.rejections.get("PotentialCollision", 0) > 0


def test_codec_host_prep_matches_oracle():
    import fgumi_b200 as fg
    rng = np.random.default_rng(5)
    groups = random_codec_groups(rng, 150)
    cap = Capture()
    oracle = R.CodecCallerOracle("fgumi", "A", vote_fn=cap, builder_fn=O.builder_call, codec_job_fn=codec_job_fn)
    c = fg.CodecConsensusCaller("fgumi", "A", device=fg.lib.FGB_DEVICE_NONE)
    n, _ = _compare_groups(fg, c, lambda g: oracle.consensus_reads(g)[1], cap, groups, unordered=True)
    pend = c.pending()
    st = c.statistics()
    c.close()
    assert n > 100 and len(pend["codec_jobs"]) * 2 == n
    # the CODEC rejections are all decided while planning (only the disagreement gate waits for the GPU)
    assert st["total_reads"] == oracle.total_input_reads and st["filtered_reads"] == oracle.reads_filtered
    for name in ("FragmentRead", "InsufficientReads", "MinorityAlignment", "InsufficientOverlap", "IndelErrorBetweenStrands"):
        assert st[name] == oracle.rejections.get(name, 0), name
    assert oracle.rejections.get("InsufficientOverlap", 0) > 0 and oracle.rejections.get("IndelErrorBetweenStrands", 0) > 0


@pytest.mark.parametrize("mode", ["simplex", "duplex", "codec"])
def test_threaded_add_groups_queues_the_same_batch(mode):
    """fgb_caller_add_groups on several host threads (worker sub-callers merged in input order) must
    queue exactly what group-by-group calls on one thread queue: units, rows, jobs and counters."""
    import fgumi_b200 as fg
    rng = np.random.default_rng(12)
    if mode == "simplex":
        groups = random_groups(rng, 300)
        mk = lambda t: fg.VanillaUmiConsensusCaller("fgumi", "A", device=fg.lib.FGB_DEVICE_NONE, n_threads=t,
                                                    consensus_call_overlapping_bases=True)
    elif mode == "duplex":
        groups = random_duplex_groups(rng, 200)
        mk = lambda t: fg.DuplexConsensusCaller("fgumi", "A", min_reads=(1, 1, 0), device=fg.lib.FGB_DEVICE_NONE, n_threads=t)
    else:
        groups = random_codec_groups(rng, 200)
        mk = lambda t: fg.CodecConsensusCaller("fgumi", "A", device=fg.lib.FGB_DEVICE_NONE, n_threads=t)
    one = mk(1)
    for g in groups:
        one.add_group(g)
    many = mk(5)
    many.add_groups(groups)
    a, b = one.pending(), many.pending()
    sa, sb = one.statistics(), many.statistics()
    one.close(); many.close()
    assert a["units"] == b["units"] and a["n_out"] == b["n_out"] and len(a["units"]) > 100
    assert np.array_equal(a["duplex_jobs"], b["duplex_jobs"]) and np.array_equal(a["codec_jobs"], b["codec_jobs"])
    assert sa == sb


@pytest.mark.parametrize("mode", ["simplex", "duplex", "codec"])
@pytest.mark.parametrize("threads", [1, 5])
def test_failing_add_groups_call_leaves_nothing_queued(mode, threads):
    """A call that fails (here: a truncated record in a group in the middle of the call) queues nothing
    of itself and counts nothing, whatever the thread count; what earlier calls queued stays, and the caller goes on
    to queue later calls exactly as if the failing one had never been made."""
    import fgumi_b200 as fg
    from tests.bam_builder import make_record
    rng = np.random.default_rng(21)
    if mode == "simplex":
        gen, mk = random_groups, lambda t: fg.VanillaUmiConsensusCaller("fgumi", "A", device=fg.lib.FGB_DEVICE_NONE, n_threads=t)
    elif mode == "duplex":
        gen, mk = random_duplex_groups, lambda t: fg.DuplexConsensusCaller("fgumi", "A", min_reads=(1, 1, 0), device=fg.lib.FGB_DEVICE_NONE, n_threads=t)
    else:
        gen, mk = random_codec_groups, lambda t: fg.CodecConsensusCaller("fgumi", "A", device=fg.lib.FGB_DEVICE_NONE, n_threads=t)
    first, second, third = gen(rng, 150), gen(rng, 400), gen(rng, 150)
    bad = [make_record(name=b"x", flags=0, pos=5, seq=b"ACGTACGTAC", quals=bytes([30] * 10), tags=[(b"MI", "Z", b"9")])[:20]]
    broken = second[:250] + [bad] + second[250:]
    c = mk(threads)
    c.add_groups(first)
    before, stats_before = c.pending(), c.statistics()
    with pytest.raises(fg.lib.FgbError) as e:
        c.add_groups(broken)
    assert e.value.status in (fg.lib.FGB_ERR_INVALID_ARG, fg.lib.FGB_ERR_LAYOUT)
    after, stats_after = c.pending(), c.statistics()
    assert after["units"] == before["units"] and after["n_out"] == before["n_out"] and stats_after == stats_before
    c.add_groups(third)
    got, got_stats = c.pending(), c.statistics()
    c.close()
    ref = mk(threads)
    ref.add_groups(first); ref.add_groups(third)
    want, want_stats = ref.pending(), ref.statistics()
    ref.close()
    assert got["units"] == want["units"] and got["n_out"] == want["n_out"] and got_stats == want_stats
    assert np.array_equal(got["duplex_jobs"], want["duplex_jobs"]) and np.array_equal(got["codec_jobs"], want["codec_jobs"])


@pytest.mark.parametrize("sanitizer", ["address,undefined", "thread"])
def test_host_caller_under_sanitizers(tmp_path, sanitizer):
    """caller_host.cpp itself compiled with ASan+UBSan, and with TSan, into tests/native/caller_plan.cpp:
    planning-only callers of the three modes over random MI groups, one thread against six, two rounds
    (pooled buffers reused), with the serial and with the threaded merge of the worker batches; the harness
    also compares the two queued batches byte for byte."""
    import shutil
    import struct
    import subprocess
    import fgumi_b200 as fg
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "fgumi_b200")
    fg.lib.load()                                   # the engine symbols come from the built library
    exe = tmp_path / "caller_plan"
    r = subprocess.run([gxx, "-std=c++17", "-O1", "-g", "-fsanitize=" + sanitizer, "-fno-sanitize-recover=all",
                        "-o", str(exe), os.path.join(root, "tests", "native", "caller_plan.cpp"),
                        os.path.join(libdir, "csrc", "host", "caller_host.cpp"),
                        os.path.join(libdir, "csrc", "host_tables.cpp"),
                        "-L" + libdir, "-lfgumi_b200", "-Wl,-rpath," + libdir, "-lpthread"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    rng = np.random.default_rng(2)
    for mode, groups in ((0, random_groups(rng, 150)), (1, random_duplex_groups(rng, 80)), (2, random_codec_groups(rng, 80))):
        path = tmp_path / ("groups%d.bin" % mode)
        with open(path, "wb") as f:
            f.write(struct.pack("<II", mode, len(groups)))
            for g in groups:
                f.write(struct.pack("<I", len(g)))
                for rec in g:
                    f.write(struct.pack("<I", len(rec)) + bytes(rec))
        for merge_bytes in ("0", str(1 << 40)):     # threaded merge of the worker batches / serial merge
            env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", TSAN_OPTIONS="halt_on_error=1",
                       FGB_PARALLEL_MERGE_BYTES=merge_bytes)
            r = subprocess.run([str(exe), str(path), "6"], capture_output=True, text=True, timeout=600, env=env)
            assert r.returncode == 0 and "ok units" in r.stdout and "fuzz:" in r.stdout, (mode, merge_bytes, r.returncode,
                                                                          r.stdout[-300:], r.stderr[-3000:])


def _oracle_stream(mode, variant, groups):
    """What the reference pipeline would write for these groups (oracle callers, then the oracle filter)."""
    from tests.test_codec_oracle_kat import codec_job_fn as cjf
    if mode == 0:
        oracle = R.VanillaCallerOracle("fgumi", "A", R.VanillaOptions(min_reads=1, min_consensus_base_quality=2,
                                                                    cell_tag=b"CB"), vote_fn, O.builder_call)
        ov = R.OverlappingOracle()
        stream = bytearray()
        for g in groups:
            recs = [bytearray(r) for r in g]
            ov.apply(recs)
            stream += oracle.consensus_reads([bytes(r) for r in recs])[0]
        if variant == 1:
            flt = R.SimplexFilterOracle(R.FilterThresholds(1, 0.2, 0.3), 10, None, 0.5)
            return flt.filter_stream(bytes(stream))[0]
        return bytes(stream)
    if mode == 1:
        mr = (1, 1, 1) if variant == 1 else (1, 1, 0)
        oracle = R.DuplexCallerOracle("fgumi", "A", min_reads=mr, per_base=True, cell_tag=b"CB", vote_fn=vote_fn,
                                      builder_fn=O.builder_call, duplex_job_fn=duplex_job_fn)
        stream = b"".join(oracle.consensus_reads(g)[0] for g in groups)
        if variant == 1:
            T = R.FilterThresholds
            flt = R.DuplexFilterOracle(T(3, 0.05, 0.2), T(2, 0.05, 0.1), T(1, 0.1, 0.3), 20, None, 0.3, False)
            return flt.filter_stream(stream)[0]
        return stream
    oracle = R.CodecCallerOracle("codec", "RG1", per_base=True, cell_tag=b"CB", vote_fn=vote_fn, builder_fn=O.builder_call,
                                 codec_job_fn=cjf)
    return b"".join(oracle.consensus_reads(g)[0] for g in groups)


@pytest.mark.parametrize("sanitizer", ["address,undefined", "thread"])
def test_callers_end_to_end_on_a_mock_engine(tmp_path, sanitizer):
    """The WHOLE record-level path of the product's host code -- add_groups, tile planning, submit, record
    assembly on threads, the simplex and duplex filter stages, two flushes on one caller -- run on the CPU
    with tests/native/mock_engine.cpp (the oracle's vote / combine behind the engine's entry points) in
    place of the GPU, under ASan+UBSan and under TSan; the bytes must equal the oracle callers' output."""
    import shutil
    import struct
    import subprocess
    import fgumi_b200 as fg
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "fgumi_b200")
    fg.lib.load()
    exe = tmp_path / "caller_e2e"
    nat = os.path.join(root, "tests", "native")
    r = subprocess.run([gxx, "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-fsanitize=" + sanitizer,
                        "-fno-sanitize-recover=all", "-o", str(exe), os.path.join(nat, "caller_e2e.cpp"),
                        os.path.join(nat, "mock_engine.cpp"), os.path.join(libdir, "csrc", "host", "caller_host.cpp"),
                        os.path.join(libdir, "csrc", "host_tables.cpp"), os.path.join(root, "oracle", "fgumi_oracle.cpp"),
                        os.path.join(root, "oracle", "oracle_capi.cpp"),
                        "-L" + libdir, "-lfgumi_b200", "-Wl,-rpath," + libdir, "-lpthread"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    rng = np.random.default_rng(4)
    cases = [(0, random_groups(rng, 120)), (1, random_duplex_groups(rng, 90)), (2, random_codec_groups(rng, 90))]
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", TSAN_OPTIONS="halt_on_error=1")
    for mode, groups in cases:
        path = tmp_path / ("groups%d.bin" % mode)
        with open(path, "wb") as f:
            f.write(struct.pack("<II", mode, len(groups)))
            for g in groups:
                f.write(struct.pack("<I", len(g)))
                for rec in g:
                    f.write(struct.pack("<I", len(rec)) + bytes(rec))
        for variant in ((0, 1) if mode < 2 else (0,)):
            want = _oracle_stream(mode, variant, groups)
            assert len(want) > 1000
            for threads in (1, 4):
                outp = tmp_path / ("out_%d_%d_%d.bin" % (mode, variant, threads))
                r = subprocess.run([str(exe), str(path), str(threads), str(variant), str(outp)], capture_output=True,
                                   text=True, timeout=900, env=env)
                assert r.returncode == 0 and r.stdout.startswith("ok count"), (mode, variant, threads, r.stdout[-300:], r.stderr[-3000:])
                got = open(outp, "rb").read()
                if got != want:
                    from tests.bam_builder import parse_records
                    a, b = parse_records(got), parse_records(want)
                    assert len(a) == len(b), (mode, variant, threads, len(a), len(b))
                    for i, (x, y) in enumerate(zip(a, b)):
                        assert x == y, (mode, variant, threads, i, x, y)
                assert got == want, (mode, variant, threads)
            if mode == 0 and variant == 0:
                # the zero-copy path: the mock engine reports the harness' blob as page-locked, no staging copy is made
                outp = tmp_path / "out_zero_copy.bin"
                r = subprocess.run([str(exe), str(path), "4", "0", str(outp)], capture_output=True, text=True, timeout=900,
                                   env=dict(env, FGB_MOCK_PINNED="1"))
                assert r.returncode == 0 and r.stdout.startswith("ok count"), (r.stdout[-300:], r.stderr[-3000:])
                assert open(outp, "rb").read() == want
    # a batch the group rules reject whole (min_reads = 2, every group one overlapping pair): nothing is voted, yet
    # the pre-pass counters must match the reference, which co-calls every pair of every group; two flushes
    from tests.test_overlap_device import group, oracle_run, stat_view
    groups = [group(rng, "single", g, 2) for g in range(40)]
    path = tmp_path / "groups_rejected.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<II", 0, len(groups)))
        for g in groups:
            f.write(struct.pack("<I", len(g)))
            for rec in g:
                f.write(struct.pack("<I", len(rec)) + bytes(rec))
    want, count, s, ov = oracle_run(groups, 2)
    assert count == 0 and ov[0] > 1000
    for threads, extra in ((1, {}), (4, {}), (4, {"FGB_MOCK_PINNED": "1"})):
        outp = tmp_path / "out_rejected.bin"
        r = subprocess.run([str(exe), str(path), str(threads), "2", str(outp)], capture_output=True, text=True,
                           timeout=900, env=dict(env, **extra))
        assert r.returncode == 0 and r.stdout.startswith("ok count 0 "), (threads, extra, r.stdout[-300:], r.stderr[-3000:])
        assert open(outp, "rb").read() == b""
        st = dict(zip(fg.lib.STAT_NAMES, (int(x) for x in r.stdout.split()[3:])))
        assert {k: st[k] for k in stat_view(s, ov)} == stat_view(s, ov, 2), (threads, extra)
