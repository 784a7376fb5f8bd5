"""The span decoder and block-start search of the GPU inflate (csrc/inflate.cuh), run on the CPU through
dca_inflate_span_host / dca_inflate_find_host: every stream of tests/gzip_cases.py is split at the candidates the
search finds, each span decoded with window markers, the markers resolved and the spans chained; the bytes must equal
zlib's, every true dynamic and stored block start must be found, and false candidates must be rejected by the chain."""
import gzip
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

from dca_b200 import _lib
from tests.gzip_cases import cases, count_text, member, raw_deflate, stored_with_deflate_inside

CASES = cases()
ST_STOP, ST_END = 0, 1
REGION_BITS = 4096 * 8          # small regions, so that the small test streams have many spans


def header_len(buf, at=0):
    flg = buf[at + 3]
    q = at + 10
    if flg & 4:
        q += 2 + buf[q] + (buf[q + 1] << 8)
    for f in (8, 16):
        if flg & f:
            q = buf.index(b"\x00", q) + 1
    return q + (2 if flg & 2 else 0)


class Stream:
    def __init__(self, gz):
        self.buf = gz
        self.arr = np.frombuffer(gz, dtype=np.uint8)
        self.lib = _lib.load()

    def span(self, start, stop, cap=None):
        info = np.zeros(6, dtype=np.int64)
        out = None if cap is None else np.zeros(max(cap, 1), dtype=np.uint16)
        _lib.check(self.lib.dca_inflate_span_host(self.arr.ctypes.data, len(self.buf), 1, start, stop,
                                                  None if out is None else out.ctypes.data, cap or 0, info.ctypes.data))
        return info, out

    def find(self, a, b):
        f = np.zeros(1, dtype=np.int64)
        _lib.check(self.lib.dca_inflate_find_host(self.arr.ctypes.data, len(self.buf), a, b, f.ctypes.data))
        return int(f[0])

    def btype(self, bit):
        v = int.from_bytes(self.buf[bit >> 3:(bit >> 3) + 2].ljust(2, b"\0"), "little") >> (bit & 7)
        return (v >> 1) & 3


def resolve(out, sym, off):
    """The bytes of one span's symbols, markers from the output before the span at global offset `off`."""
    sym = sym.astype(np.int64)
    m = sym >= 0x8000
    b = sym.copy()
    b[m] = out[off - (sym[m] & 0x7fff) - 1]
    return b.astype(np.uint8)


def serial_blocks(s):
    """Block starts of a serial decode, block by block (each stop one bit past the start), checked against zlib."""
    pos, starts, out = header_len(s.buf) * 8, [], np.zeros(0, np.uint8)
    while True:
        info, _ = s.span(pos, pos + 1)
        assert info[0] in (ST_STOP, ST_END), info
        _, sym = s.span(pos, pos + 1, cap=int(info[2]))
        out = np.concatenate([out, resolve(out, sym[:info[2]], len(out))])
        starts.append(pos)
        pos = int(info[1])
        if info[0] == ST_END:
            return starts, out.tobytes()


@pytest.mark.parametrize("name", sorted(CASES))
def test_serial_decode_and_true_starts_found(name):
    gz, data = CASES[name]
    s = Stream(gz)
    starts, out = serial_blocks(s)
    assert out == data == gzip.decompress(gz)
    for b in starts:
        if s.btype(b) in (0, 2):                   # dynamic or stored: the search must find it
            assert s.find(b, b + 1) == b, (name, b)


@pytest.mark.parametrize("name", sorted(CASES))
def test_span_parallel_decode(name):
    gz, data = CASES[name]
    s = Stream(gz)
    p0, end = header_len(gz) * 8, len(gz) * 8
    true_starts = set(serial_blocks(s)[0])
    cands = [p0] + [c for c in (s.find(r, min(r + REGION_BITS, end)) for r in range(p0 + REGION_BITS, end, REGION_BITS))
                    if c >= 0]
    false = [c for c in cands if c not in true_starts and s.btype(c) in (0, 2)]
    stops = cands[1:] + [1 << 62]
    # pass 1 from the candidates, then the chain: a span counts only from where the one before it stopped
    res = [s.span(a, b)[0] for a, b in zip(cands, stops)]
    starts = list(cands)
    expected, accepted, redone = p0, [], 0
    for k in range(len(cands)):
        if starts[k] != expected:
            assert starts[k] not in true_starts or starts[k] < expected
            starts[k] = expected
            res[k] = s.span(expected, stops[k])[0]
            redone += 1
        assert res[k][0] in (ST_STOP, ST_END), (name, k, res[k])
        accepted.append(k)
        expected = int(res[k][1])
        if res[k][0] == ST_END:
            break
    assert all(starts[k] in true_starts for k in accepted), "a span not starting at a block start was accepted"
    assert all(c not in true_starts for c in false)
    # pass 2 with markers, resolved in span order
    out = np.zeros(0, np.uint8)
    for k in accepted:
        n = int(res[k][2])
        _, sym = s.span(starts[k], stops[k], cap=n)
        info = res[k]
        assert len(out) + info[3] >= 0
        out = np.concatenate([out, resolve(out, sym[:n], len(out))])
    assert out.tobytes() == data


def test_declines_are_statuses():
    gz, data = CASES["level6"]
    s = Stream(gz[:len(gz) // 2])
    info, _ = s.span(header_len(gz) * 8, 1 << 62)
    assert info[0] == 3                              # truncated at the end of the file
    bad = bytearray(gz)
    bad[-9] ^= 0xff                                  # last deflate byte
    info, _ = Stream(bytes(bad)).span(header_len(gz) * 8, 1 << 62)
    assert info[0] in (1, 3)
    s = Stream(gz + b"\x00junk")
    info, _ = s.span(header_len(gz) * 8, 1 << 62)
    assert info[0] == 3                              # trailing garbage


# ------------------------------------------------------------------------------------------------ termination
# Decoding must end in a status whatever the input: a decoder that reads past the bytes it has sees zero bits, which
# decode to symbols for ever unless it stops at the overrun.  These run in a subprocess with a timeout, so a hang fails
# the test instead of stopping the suite.
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 1 << 62
GPU_REGION_BITS = 32768 * 8      # the regions of csrc/inflate.cu


def termination_streams():
    """name -> truncated or crafted gzip bytes whose decoding must end."""
    out = {}
    for name, (gz, _) in CASES.items():
        for frac in (3, 2):
            out["%s_cut_%d" % (name, frac)] = gz[:len(gz) * (frac - 1) // frac] if len(gz) > 20 else gz[:-1]
    out["huffman_only_cut"] = member(count_text(100_000), strategy=zlib.Z_HUFFMAN_ONLY)[:-40_000]
    out["stored_with_deflate_inside"] = stored_with_deflate_inside()[0]
    return out


def decode_all(gz):
    """Every decode the inflate may run on these bytes must return: from the first block, and from the candidate of
    every 32 KB region, to the end of the file (eof) and to the end of the loaded bytes (not eof)."""
    s = Stream(gz)
    if len(gz) < 10 or gz[:2] != b"\x1f\x8b":
        return
    try:
        p0 = header_len(gz) * 8
    except (IndexError, ValueError):
        return
    end = len(gz) * 8
    starts = [p0] + [c for c in (s.find(r, min(r + GPU_REGION_BITS, end)) for r in range(p0 + GPU_REGION_BITS, end,
                                                                                          GPU_REGION_BITS)) if c >= 0]
    info = np.zeros(6, dtype=np.int64)
    for a in starts:
        for eof in (1, 0):
            _lib.check(s.lib.dca_inflate_span_host(s.arr.ctypes.data, len(gz), eof, a, NONE, None, 0, info.ctypes.data))
            assert info[0] in ((1, 3) if eof else (1, 2, 3)) or a != p0, info


def test_truncated_and_crafted_streams_end_in_a_status():
    names = sorted(termination_streams())
    r = subprocess.run([sys.executable, "-m", "tests.test_inflate_host"] + names, cwd=ROOT, timeout=300,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert r.stdout.split().count("ok") == len(names)


def test_crafted_candidate_is_found():
    """The crafted file puts a plausible dynamic block start at the first bit of the second 32 KB region."""
    gz = stored_with_deflate_inside()[0]
    s = Stream(gz)
    r1 = header_len(gz) * 8 + GPU_REGION_BITS
    assert s.find(r1, r1 + GPU_REGION_BITS) == r1


if __name__ == "__main__":
    streams = termination_streams()
    for n in sys.argv[1:]:
        decode_all(streams[n])
        print("ok", n, flush=True)
