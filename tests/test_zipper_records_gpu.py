"""fgb_zipper_records on the GPU against the literal replay of tests/zipper_oracle.py, output streams and stats byte
for byte: synthetic aligned streams, consensus tags with the Consensus sets, both options, 4 KiB staging, carried
mapped records, long reads and kilobyte MC values, a call of over a million records, every error, and the file-level
run through sort and group."""
import os
import struct

import numpy as np
import pytest

from tests import zipper_oracle as O
from tests.bam_builder import make_record
from tests.test_zipper_records import arrays, pair, unmapped_pair
from tests.zipper_streams import streams

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def Z():
    from fgumi_b200 import zipper
    return zipper


def zip_dev(Z, um, mp, last_call=True, **kw):
    z = Z.Zipper(0, **kw)
    try:
        ub, uo = arrays(um)
        mb, mo = arrays(mp)
        return z.zip(ub, uo, mb, mo, last_call), z
    finally:
        z.close()


OK = {"tags_to_remove": "remove", "tags_to_reverse": "reverse", "tags_to_revcomp": "revcomp",
      "exclude_missing_reads": "exclude_missing", "skip_pa_tags": "skip_tc"}


def check(Z, um, mp, last_call=True, **kw):
    (data, used, stats), _ = zip_dev(Z, um, mp, last_call, **kw)
    out, consumed, ostats = O.zipper(um, mp, last_call=last_call,
                                     **{OK[k]: v for k, v in kw.items() if k in OK})
    assert data == O.stream(out)
    assert used == consumed
    assert list(stats.values()) == ostats
    return data


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("exclude", [False, True])
@pytest.mark.parametrize("skip", [False, True])
def test_random_streams(Z, seed, exclude, skip):
    um, mp = streams(100 + seed, n_templates=400, consensus=seed % 2 == 1)
    check(Z, um, mp, tags_to_remove=["NM"], tags_to_reverse=["Consensus"], tags_to_revcomp=["Consensus", "RX"],
          exclude_missing_reads=exclude, skip_pa_tags=skip, n_threads=4)


def test_small_staging_and_carry(Z, monkeypatch):
    monkeypatch.setenv("FGB_ZIPPER_STAGE_BYTES", "4096")
    um, mp = streams(7, n_templates=3000, consensus=True, missing=0.05)
    names = [O.name(r) for r in um]
    cuts = [0]
    for c in (len(um) // 7, len(um) // 3, len(um) // 3, len(um) // 2, len(um)):   # includes an empty call
        while 0 < c < len(um) and names[c] == names[c - 1]:
            c += 1
        cuts.append(c)
    got, m0 = b"", 0
    for k in range(len(cuts) - 1):
        (data, used, _), _ = zip_dev(Z, um[cuts[k]:cuts[k + 1]], mp[m0:], last_call=k == len(cuts) - 2,
                                     tags_to_revcomp=["Consensus"], tags_to_reverse=["Consensus"], device_bytes=1 << 20)
        got += data
        m0 += used
    assert m0 == len(mp)
    assert got == O.stream(O.zipper(um, mp, reverse=["Consensus"], revcomp=["Consensus"])[0])


def test_long_reads_and_long_mc(Z):
    L = 65535
    cig = "".join("1M1I" for _ in range(L // 4)) + "%dM" % (L - 2 * (L // 4))
    um = unmapped_pair(t1=[(b"cD", "Z", b"ACGT" * (L // 4)), (b"cd", "Bs", list(range(1000)))])
    seq = b"A" * L
    a = make_record(name=b"q", flags=0x41 | 0x10, ref_id=0, pos=5, cigar=cig, seq=seq, tags=[(b"MC", "Z", b"1M")])
    b = make_record(name=b"q", flags=0x81, ref_id=0, pos=9, cigar=cig, seq=seq)
    data = check(Z, um, [a, b], tags_to_revcomp=["Consensus"], tags_to_reverse=["Consensus"])
    assert len(data) > 2 * L + 2 * len(cig)


def test_million_records(Z):
    um, mp = [], []
    base_u = unmapped_pair(name=b"q0000000")
    base_m = pair(name=b"q0000000", t1=[(b"AS", "i", 77)], t2=[(b"MQ", "C", 3)])
    for t in range(260_000):
        nm = b"q%07d" % t
        um += [r.replace(b"q0000000", nm, 1) for r in base_u]
        mp += [r.replace(b"q0000000", nm, 1) for r in base_m]
    (data, used, stats), z = zip_dev(Z, um, mp, n_threads=8)
    assert stats["records_out"] == 520_000 and used == len(mp) and len(um) + len(mp) >= 1_000_000
    exp = O.stream(O.zipper(um[:2000], mp[:2000])[0])
    assert data[:len(exp)] == exp
    # every template is the same edit of the first one, so the whole stream is the first template's bytes, renamed
    first = O.stream(O.zipper(um[:2], mp[:2])[0])
    assert len(data) == 260_000 * len(first)
    assert data[-len(first):] == first.replace(b"q0000000", b"q%07d" % 259_999)


def test_errors(Z):
    um, mp = unmapped_pair(), pair()
    cases = [
        (um, [mp[0], mp[1][:40]], 4, len(um) + 1),                                   # truncated
        (um, [mp[0], mp[1] + b"xxZab"], 4, len(um) + 1),                             # aux does not parse
        (um, pair(t1=[(b"RX", "Z", b"A"), (b"RX", "Z", b"B")]), 1, len(um)),         # a tag twice
        (um, [mp[0], mp[0]], 1, len(um) + 1),                                        # two primary R1s
        (um, mp + pair(name=b"z"), 1, len(um) + 2),                                  # leftover
        ([um[0], um[0]], mp, 1, 1),                                                  # two R1s in the unmapped stream
        ([um[0][:20]] + um[1:], mp + [mp[0][:8]], 4, 0),                             # first of two layout errors
        ([um[0], um[0]], [mp[0][:20], mp[1]], 1, 1),                                 # INVALID_ARG before LAYOUT
        (um + [r.replace(b"q\0", b"r\0") for r in (um[0], um[0])], [mp[0][:20], mp[1]], 4, 4),  # LAYOUT first
    ]
    from fgumi_b200 import lib as L
    for u, m, status, bad in cases:
        z = Z.Zipper(0)
        ub, uo = arrays(u)
        mb, mo = arrays(m)
        with pytest.raises(L.FgbError) as e:
            z.zip(ub, uo, mb, mo, True)
        assert e.value.status == status and z.bad_record == bad, (e.value, z.bad_record, bad)
        z.close()
    z = Z.Zipper(0, tags_to_remove=["A\x00"])   # a tag-list entry with a NUL byte
    ub, uo = arrays(um)
    mb, mo = arrays(mp)
    with pytest.raises(L.FgbError) as e:
        z.zip(ub, uo, mb, mo, True)
    assert e.value.status == 1
    z.close()
    z = Z.Zipper(0)
    z.opt.restore_unconverted_bases = 1   # not offered
    with pytest.raises(L.FgbError) as e:
        z.zip(ub, uo, mb, mo, True)
    assert e.value.status == 1
    z.close()


def _write_bam(path, text, recs):
    from fgumi_b200 import bamio
    with open(path, "wb") as f:
        bamio._write_bgzf(f, bamio.mapped_bam_header(text) + O.stream(recs), 1, 2)


def test_zipper_file_and_chain(Z, tmp_path):
    from fgumi_b200 import bamio
    from fgumi_b200.group import ReadGrouper
    from fgumi_b200.sort import RecordSorter
    um, mp = streams(31, n_templates=3000, missing=0.02, odd_mc=False)
    sq = b"@SQ\tSN:chr0\tLN:100000\n@SQ\tSN:chr1\tLN:100000\n@SQ\tSN:chr2\tLN:100000\n"
    u_text = b"@HD\tVN:1.6\tSO:queryname\n@RG\tID:A\tSM:s\n@CO\tunmapped\n"
    m_text = b"@HD\tVN:1.6\tSO:queryname\n" + sq + b"@PG\tID:bwa\tPN:bwa\n@CO\tmapped\n"
    _write_bam(tmp_path / "u.bam", u_text, um)
    _write_bam(tmp_path / "m.bam", m_text, mp)
    (tmp_path / "ref.fa").write_bytes(b">chr0\nA\n")
    (tmp_path / "ref.dict").write_bytes(b"@HD\tVN:1.6\n" + sq)
    z = Z.Zipper(0, n_threads=4)
    bamio.zipper_file(str(tmp_path / "u.bam"), str(tmp_path / "m.bam"), str(tmp_path / "ref.fa"),
                      str(tmp_path / "z.bam"), z, batch_records=1000)
    z.close()
    text, bodies, off, _ = bamio.read_bam(str(tmp_path / "z.bam"))
    exp = O.zipper(um, mp)[0]
    got = bytes(bodies)
    assert got == b"".join(exp)
    assert text == O.output_header(u_text, m_text, b"@HD\tVN:1.6\n" + sq, "fgumi_b200 zipper")
    # the chain: sort template-coordinate then group, on the device's output and on the oracle's
    outs = []
    for recs in ([bytes(bodies[int(off[i]):int(off[i + 1])]) for i in range(len(off) - 1)], exp):
        b, o = arrays(recs)
        s = RecordSorter(0, "template-coordinate")
        sorted_stream = s.sort(text, b, o)
        s.close()
        sb, so = bamio.split_stream(sorted_stream)
        g = ReadGrouper(0, strategy="adjacency", edits=1)
        outs.append(bamio.group_records(text, sb, so, g))
        g.close()
    assert outs[0] == outs[1] and len(outs[0]) > 0
