"""fgb_host_zipper_records (the device zipper's per-record rules on host threads) against the literal replay of
tests/zipper_oracle.py, byte for byte: the edit-placement cases, random streams at 1 and 6 threads, the join's carry
and its errors, the header builder and the options struct."""
import ctypes as C
import struct

import numpy as np
import pytest

from tests import zipper_oracle as O
from tests.bam_builder import make_record
from tests.zipper_streams import streams


@pytest.fixture(scope="module")
def Z():
    from fgumi_b200 import lib as L
    L.load()
    from fgumi_b200 import zipper
    return zipper


def arrays(recs):
    off = np.zeros(len(recs) + 1, np.uint64)
    for i, r in enumerate(recs):
        off[i + 1] = off[i] + len(r)
    return np.frombuffer(b"".join(recs) or b"\0", np.uint8), off


def run(Z, um, mp, last_call=True, **kw):
    ub, uo = arrays(um)
    mb, mo = arrays(mp)
    return Z.host_zip(Z.options(**kw), ub, uo, mb, mo, last_call)


def check(Z, um, mp, last_call=True, **kw):
    st, data, used, stats, bad = run(Z, um, mp, last_call, **kw)
    assert st == 0, (st, bad)
    okw = {k: v for k, v in kw.items() if k != "n_threads"}
    ok = {"tags_to_remove": "remove", "tags_to_reverse": "reverse", "tags_to_revcomp": "revcomp",
          "exclude_missing_reads": "exclude_missing", "skip_pa_tags": "skip_tc"}
    out, consumed, ostats = O.zipper(um, mp, last_call=last_call, **{ok[k]: v for k, v in okw.items()})
    exp = O.stream(out)
    if data != exp:
        got = [r for r in _split(data)]
        for i, (a, b) in enumerate(zip(got, out)):
            assert a == b, (i, a.hex(), b.hex())
    assert data == exp
    assert used == consumed and stats == ostats
    return out


def _split(data):
    p = 0
    while p < len(data):
        (n,) = struct.unpack_from("<I", data, p)
        yield data[p + 4:p + 4 + n]
        p += 4 + n


def pair(name=b"q", f1=0, f2=0, t1=(), t2=(), pos1=100, pos2=200, c1="10M", c2="10M", ref=0):
    a = make_record(name=name, flags=0x41 | f1, ref_id=-1 if f1 & 4 else ref, pos=-1 if f1 & 4 else pos1,
                    cigar=[] if f1 & 4 else c1, seq=b"ACGTACGTAC", tags=t1)
    b = make_record(name=name, flags=0x81 | f2, ref_id=-1 if f2 & 4 else ref, pos=-1 if f2 & 4 else pos2,
                    cigar=[] if f2 & 4 else c2, seq=b"ACGTACGTAC", tags=t2)
    return [a, b]


def unmapped_pair(name=b"q", t1=((b"RX", "Z", b"ACGT"),), t2=((b"RX", "Z", b"ACGT"),), qc=0):
    return [make_record(name=name, flags=0x4D | qc, ref_id=-1, pos=-1, cigar=[], seq=b"ACGTACGTAC", tags=t1),
            make_record(name=name, flags=0x8D | qc, ref_id=-1, pos=-1, cigar=[], seq=b"ACGTACGTAC", tags=t2)]


PLACEMENT = {
    "mq_C_moves": dict(t1=[(b"MQ", "C", 200), (b"xx", "Z", b"a")]),
    "mq_i_stays": dict(t1=[(b"MQ", "i", 7), (b"xx", "Z", b"a")]),
    "mc_same_length": dict(t1=[(b"MC", "Z", b"99M"), (b"xx", "Z", b"a")]),
    "mc_other_length": dict(t1=[(b"MC", "Z", b"5M5S"), (b"xx", "Z", b"a")]),
    "mc_non_z_same_length": dict(t1=[(b"MC", "i", 5), (b"xx", "Z", b"a")]),          # 3 value bytes, "10M"
    "mc_non_z_other_length": dict(t1=[(b"MC", "i", 5), (b"xx", "Z", b"a")], c2="1M"),
    "pre_existing_tc": dict(t1=[(b"tc", "Z", b"x"), (b"xx", "Z", b"a")]),
    "mapped_rx_replaced": dict(t1=[(b"RX", "Z", b"OLDOLD"), (b"yy", "i", 3)]),
    "as_and_xs": dict(t1=[(b"AS", "I", 3000000000), (b"XS", "S", 300)], t2=[(b"AS", "C", 200)]),
}


@pytest.mark.parametrize("case", sorted(PLACEMENT))
@pytest.mark.parametrize("remove", [(), ("MQ", "MC", "ms"), ("RX", "PG")])
def test_edit_placement(Z, case, remove):
    kw = dict(PLACEMENT[case])
    mp = pair(**kw)
    mp.append(make_record(name=b"q", flags=0x841 | 0x10, ref_id=1, pos=50, cigar="4S6M", seq=b"ACGTACGTAC",
                          tags=[(b"MQ", "c", 1)]))
    um = unmapped_pair(t1=[(b"RX", "Z", b"ACGT"), (b"AS", "i", 5), (b"PG", "Z", b"p"), (b"cD", "Z", b"acgN")])
    check(Z, um, mp, tags_to_remove=remove, tags_to_revcomp=["Consensus"])


@pytest.mark.parametrize("f1,f2", [(0, 0), (4, 0), (0, 4), (4, 4), (0x10, 0x10), (0x10, 0)])
def test_mate_fix_arms(Z, f1, f2):
    mp = pair(f1=f1, f2=f2, t1=[(b"AS", "c", 9)], t2=[(b"AS", "s", -300), (b"MQ", "i", 1)], c1="3S7M", c2="7M3S")
    mp.append(make_record(name=b"q", flags=0x881, ref_id=0, pos=10, cigar="10M", seq=b"ACGTACGTAC"))
    mp.append(make_record(name=b"q", flags=0x141, ref_id=0, pos=10, cigar="10M", seq=b"ACGTACGTAC"))
    check(Z, unmapped_pair(), mp)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("threads", [1, 6])
def test_random_streams(Z, seed, threads):
    um, mp = streams(seed, consensus=seed % 2 == 1, long_cigar=seed == 4)
    check(Z, um, mp, tags_to_remove=["NM", "XX"] if seed % 3 else [], tags_to_reverse=["Consensus"],
          tags_to_revcomp=["Consensus", "RX"], exclude_missing_reads=seed == 2, skip_pa_tags=seed == 3,
          n_threads=threads)


def test_carry_without_last_call(Z):
    um, mp = streams(11, n_templates=60, missing=0.0)
    names = [O.name(r) for r in um]
    cut = names.index(names[len(um) // 2])
    st, data, used, stats, _ = run(Z, um[:cut], mp, last_call=False)
    assert st == 0
    out, consumed, _ = O.zipper(um[:cut], mp, last_call=False)
    assert data == O.stream(out) and used == consumed
    st2, data2, used2, _, _ = run(Z, um[cut:], mp[used:], last_call=True)
    assert st2 == 0 and used + used2 == len(mp)
    assert data + data2 == O.stream(O.zipper(um, mp)[0])
    st3, data3, used3, _, _ = run(Z, [], mp, last_call=False)   # a call that consumes nothing
    assert st3 == 0 and used3 == 0 and data3 == b""


def test_errors_name_the_record(Z):
    um, mp = unmapped_pair(), pair()
    bad = bytearray(mp[1])
    bad += b"xxZabc"   # no NUL: the aux area does not parse
    st, *_, b = run(Z, um, [mp[0], bytes(bad)])
    assert (st, b) == (4, len(um) + 1)
    dup = pair(t1=[(b"RX", "Z", b"A"), (b"RX", "Z", b"B")])
    st, *_, b = run(Z, um, dup)
    assert (st, b) == (1, len(um))
    st, *_, b = run(Z, um, [mp[0], mp[0]])   # two primary R1s
    assert (st, b) == (1, len(um) + 1)
    st, *_, b = run(Z, um, mp + pair(name=b"z"))   # a mapped template left over
    assert (st, b) == (1, len(um) + 2)
    st, *_, b = run(Z, um, mp + pair(name=b"z"), last_call=False)
    assert (st, b) == (0, None)
    st, *_, b = run(Z, [um[0][:20]] + um[1:], mp)   # short unmapped record first
    assert (st, b) == (4, 0)
    cig = bytearray(mp[0])   # CIGAR op code 9
    cig[32 + cig[8]] = (cig[32 + cig[8]] & 0xF0) | 9
    st, *_, b = run(Z, um, [bytes(cig), mp[1]])
    assert (st, b) == (1, len(um))


def test_first_of_two_errors_of_different_kinds(Z):
    um, mp = unmapped_pair(), pair()
    two_r1 = [um[0], um[0]]   # INVALID_ARG at unmapped record 1, before a cut-short mapped record
    st, *_, b = run(Z, two_r1, [mp[0][:20], mp[1]])
    assert (st, b) == (1, 1)
    # a cut-short mapped record (LAYOUT) met by the join before an unmapped template with two R1s
    st, *_, b = run(Z, um + [r.replace(b"q\0", b"r\0") for r in (um[0], um[0])], [mp[0][:20], mp[1]])
    assert (st, b) == (4, 4)


def test_refused_options(Z):
    um, mp = unmapped_pair(), pair()
    st, *_ = run(Z, um, mp, tags_to_remove=["A\x00"])   # a tag-list entry with a NUL byte
    assert st == 1
    ub, uo = arrays(um)
    mb, mo = arrays(mp)
    o = Z.options()
    o.restore_unconverted_bases = 1
    assert Z.host_zip(o, ub, uo, mb, mo)[0] == 1


def test_positions_wrap_as_i32(Z):
    # an alignment end past i32::MAX: TLEN and the tc position wrap as the reference's release build computes them
    top = 2 ** 31 - 5
    mp = pair(f1=0x10, pos1=top, pos2=top - 3, c1="3S100M5S", c2="100M")
    mp.append(make_record(name=b"q", flags=0x841, ref_id=0, pos=10, cigar="10M", seq=b"ACGTACGTAC"))
    out = check(Z, unmapped_pair(), mp)
    assert struct.unpack_from("<i", out[0], 28)[0] != 0


def test_header_builder():
    from fgumi_b200 import bamio
    u = b"@HD\tVN:1.6\tSO:queryname\n@RG\tID:A\tSM:s\n@RG\tID:B\tSM:u\n@PG\tID:extract\tPN:x\n@CO\tu1\n"
    m = b"@HD\tVN:1.5\n@SQ\tSN:old\tLN:5\n@RG\tID:A\tSM:m\n@PG\tID:bwa\tPN:bwa\n@CO\tm1\n"
    d = b"@HD\tVN:1.6\n@SQ\tSN:chr1\tLN:1000\n@SQ\tSN:chr2\tLN:20\n"
    got = bamio.zipper_header(u, m, d, "zipper -u u.bam")
    exp = O.output_header(u, m, d, "zipper -u u.bam")
    assert got == exp
    lines = got.decode().rstrip("\n").split("\n")
    assert [ln[:3] for ln in lines] == ["@HD", "@SQ", "@SQ", "@RG", "@RG", "@PG", "@PG", "@PG", "@CO", "@CO"]
    assert lines[7] == "@PG\tID:fgumi_b200\tPN:fgumi_b200\tPP:extract\tCL:zipper -u u.bam"
    assert lines[8:] == ["@CO\tu1", "@CO\tm1"]


def test_dict_lookup(tmp_path):
    from fgumi_b200 import bamio
    fa = tmp_path / "ref.fa"
    fa.write_bytes(b">chr1\nACGT\n")
    with pytest.raises(FileNotFoundError):
        bamio.find_dict_path(str(fa))
    (tmp_path / "ref.fa.dict").write_bytes(b"@SQ\tSN:chr1\tLN:4\n")
    assert bamio.find_dict_path(str(fa)) == str(tmp_path / "ref.fa.dict")
    (tmp_path / "ref.dict").write_bytes(b"@SQ\tSN:chr1\tLN:4\n")
    assert bamio.find_dict_path(str(fa)) == str(tmp_path / "ref.dict")


def test_struct_size(Z):
    from fgumi_b200 import lib as L
    assert L.load().fgb_struct_size(17) == C.sizeof(L.FgbZipperOptions) == 64


def test_tag_info_expansion(Z):
    # test_tag_info_expansion / TagInfo tests (zipper.rs:1730-1745, umi lib.rs)
    r, v, c = Z.expand_tags(["AS"], ["Consensus"], ["Consensus"])
    assert r == ["AS"] and v == sorted(O.CONSENSUS_REVERSE) and c == sorted(O.CONSENSUS_REVCOMP)
    assert "ce" not in v
    assert Z.expand_tags([], [], []) == ([], [], [])
