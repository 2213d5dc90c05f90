"""Host side of the record filter without a GPU: the FASTA parser of fgb_reference_create (parse-only references)
against tests/filter_oracle.py -- names with descriptions, \\r\\n, lower case, IUPAC codes, empty contigs, duplicate
names, compressed and headless images refused -- the ABI struct size, and the oracle's own rules on hand-made
records (NM / UQ / MD edits as the reference's editor places them, tag reversal)."""
import ctypes as C
import os
import struct
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import filter_oracle as O      # noqa: E402
from tests import filter_streams as S     # noqa: E402
from tests.bam_builder import make_record   # noqa: E402


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g
    g.build()
    from fgumi_b200 import lib
    return lib


def host_reference(L, data: bytes):
    lib = L.load()
    h = C.c_void_p()
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    st = lib.fgb_reference_create(-1, buf, len(data), C.byref(h))
    if st != 0:
        return st, None
    out = []
    name, ln = C.c_char_p(), C.c_uint64()
    for i in range(lib.fgb_reference_contigs(h)):
        assert lib.fgb_reference_contig(h, i, C.byref(name), C.byref(ln)) == 0
        out.append((name.value, ln.value))
    lib.fgb_reference_destroy(h)
    return 0, out


@pytest.mark.parametrize("crlf", [False, True])
@pytest.mark.parametrize("width", [7, 60, 10_000])
def test_fasta_parser_matches_oracle(L, crlf, width):
    contigs = S.genome(3, n_contigs=4, length=3000)
    data = S.fasta(contigs, width=width, crlf=crlf)
    st, got = host_reference(L, data)
    assert st == 0
    assert got == [(n, len(s)) for n, s in contigs]
    want = O.parse_fasta(data)
    assert {n: len(s) for n, s in want.items()} == dict(got)
    assert any(ch in want[b"chr1"] for ch in b"acgt") and any(ch in want[b"chr1"] for ch in S.IUPAC)


def test_fasta_edge_cases(L):
    data = b">a desc here\nACgt\r\nNNry\n>b\tx\n\n>c\nAC\n>a\nTTT\n"
    st, got = host_reference(L, data)
    assert st == 0 and got == [(b"a", 8), (b"b", 0), (b"c", 2), (b"a", 3)]
    assert O.parse_fasta(data) == {b"a": b"TTT", b"b": b"", b"c": b"AC"}   # the later "a" is the one looked up
    assert host_reference(L, b"\x1f\x8b\x08\x04rest")[0] == L.FGB_ERR_INVALID_ARG
    assert host_reference(L, b"ACGT\n>a\nAC\n")[0] == L.FGB_ERR_INVALID_ARG
    assert host_reference(L, b"")[1] == []


def test_struct_size_of_filter_options(L):
    assert L.load().fgb_struct_size(14) == C.sizeof(L.FgbRecordFilterOptions) == 112


def _tags(r: bytes):
    return r[O.aux_offset(r):]


def test_oracle_tag_edits():
    contig = b"ACGTacgtNNACGTACGTAC"
    g = {b"chr1": contig}
    sq = [b"chr1"]
    # an aligner's NM:C moves to the end in its smallest type; UQ appended; MD of another length spliced in place
    r = bytearray(make_record(name=b"a", ref_id=0, pos=0, cigar="4M1D3M", seq=b"ACGAcgt",
                              tags=[(b"NM", "C", 9), (b"MD", "Z", b"99"), (b"XY", "i", 1)]))
    O.regenerate(r, 0, sq, g)
    assert _tags(bytes(r)) == b"MDZ3T0^a3\0XYi" + struct.pack("<i", 1) + b"NMc\x02UQc\x1e"
    # NM of type i is overwritten in place; MD of the same length too
    r = bytearray(make_record(name=b"b", ref_id=0, pos=10, cigar="5M", seq=b"ACGTA",
                              tags=[(b"NM", "i", 7), (b"MD", "Z", b"1")]))
    O.regenerate(r, 0, sq, g)
    assert _tags(bytes(r)) == b"NMi" + struct.pack("<i", 0) + b"MDZ5\0UQc\x00"
    # read N and '=' are mismatches, reference case kept; the zero runs are written
    r = bytearray(make_record(name=b"c", ref_id=0, pos=4, cigar="4M", seq=b"N=GT"))
    O.regenerate(r, 0, sq, g)
    assert O.find_tag(bytes(r), b"MD") is not None and bytes(r).endswith(b"MDZ0a0c2\0")
    # no reference span: NM 0, UQ 0, MD "0"; unmapped: the tags removed
    r = bytearray(make_record(name=b"d", ref_id=0, pos=4, cigar="4I", seq=b"ACGT"))
    O.regenerate(r, 0, sq, g)
    assert _tags(bytes(r)) == b"NMc\x00UQc\x00MDZ0\0"
    r = bytearray(make_record(name=b"e", flags=4, ref_id=-1, pos=-1, cigar="", seq=b"ACGT",
                              tags=[(b"NM", "i", 1), (b"UQ", "i", 2), (b"MD", "Z", b"4"), (b"RG", "Z", b"x")]))
    O.regenerate(r, 0, sq, g)
    assert _tags(bytes(r)) == b"RGZx\0"


def test_oracle_tag_reversal():
    r = bytearray(make_record(name=b"a", flags=0x10, seq=b"ACGT", cigar="4M",
                              tags=[(b"cd", "Bs", [1, 2, 3, 4]), (b"aq", "Z", b"ABCD"), (b"ac", "Z", b"AacgN"),
                                    (b"xx", "Bs", [1, 2])]))
    O.reverse_per_base_tags(r)
    t = _tags(bytes(r))
    assert t.startswith(b"cdBs" + struct.pack("<I4h", 4, 4, 3, 2, 1) + b"aqZDCBA\0acZNCGTT\0")
    assert t.endswith(b"xxBs" + struct.pack("<I2h", 2, 1, 2))
