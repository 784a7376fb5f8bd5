"""The gzip compressor's block encoder (csrc/deflate.cuh), run on the CPU through dca_gzip_host: every member must
decode with zlib, Python's gzip module and the project's own span decoder (dca_inflate_span_host) to its input, with
CRC-32 and ISIZE checked, and two runs must give the same bytes.  The inputs cover the block size (32 KB) and the
window (32 KB) at their edges, long runs, incompressible bytes and the '%.6f' text the output writer produces."""
import gzip
import zlib

import numpy as np
import pytest

from dca_b200 import _lib

BLOCK = 32768


def gzip_host(data):
    lib = _lib.load()
    n = len(data)
    bound = np.zeros(1, dtype=np.int64)
    _lib.check(lib.dca_gzip_host(None, n, None, 0, bound.ctypes.data_as(lib.dca_gzip_host.argtypes[4])),
               "dca_gzip_host")
    src = np.frombuffer(data, dtype=np.uint8) if n else np.zeros(1, dtype=np.uint8)
    out = np.zeros(int(bound[0]), dtype=np.uint8)
    got = np.zeros(1, dtype=np.int64)
    _lib.check(lib.dca_gzip_host(src.ctypes.data, n, out.ctypes.data, out.size,
                                 got.ctypes.data_as(lib.dca_gzip_host.argtypes[4])), "dca_gzip_host")
    assert got[0] <= bound[0] == 18 + (n + 5 * (-(-n // BLOCK)) if n else 2)
    return out[:int(got[0])].tobytes()


def fixed6_text(values, cols):
    """'%.6f' text of float32 values through the writer's own formatter, as lines of `cols` tab-separated fields."""
    lib = _lib.load()
    bits = np.ascontiguousarray(np.asarray(values, dtype=np.float32)).view(np.uint32)
    out = np.zeros(47 * bits.size + 1, dtype=np.uint8)
    offs = np.zeros(bits.size + 1, dtype=np.int64)
    _lib.check(lib.dca_format_fixed6_host(bits.ctypes.data, bits.size, out.ctypes.data, offs.ctypes.data))
    fields = [out[offs[i]:offs[i + 1]].tobytes() for i in range(bits.size)]
    return b"".join(b"\t".join(fields[r:r + cols]) + b"\n" for r in range(0, len(fields), cols))


def inflate_own(gz):
    """The member decoded by the project's span decoder from its first block to the end of the file."""
    lib = _lib.load()
    arr = np.frombuffer(gz, dtype=np.uint8)
    info = np.zeros(6, dtype=np.int64)
    _lib.check(lib.dca_inflate_span_host(arr.ctypes.data, len(gz), 1, 80, 1 << 62, None, 0, info.ctypes.data))
    assert info[0] == 1 and info[5] == 1, info          # the end of the file, after one member trailer
    out = np.zeros(max(int(info[2]), 1), dtype=np.uint16)
    _lib.check(lib.dca_inflate_span_host(arr.ctypes.data, len(gz), 1, 80, 1 << 62, out.ctypes.data, out.size,
                                         info.ctypes.data))
    sym = out[:int(info[2])]
    assert not (sym & 0x8000).any()
    return sym.astype(np.uint8).tobytes()


def _cases():
    rng = np.random.default_rng(7)
    text = fixed6_text(rng.lognormal(-1.0, 2.0, 40000), 100)
    period = rng.integers(0, 256, BLOCK, dtype=np.uint8).tobytes()
    zeros = np.where(rng.random(30000) < 0.9, 0.0, rng.lognormal(-1.0, 2.0, 30000))
    special = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e30, -1e-30, 0.5e-6, 2.5e-6, 16777217.0] * 500)
    return {
        "empty": b"",
        "one_byte": b"x",
        "block_minus_one": text[:2 * BLOCK - 1],
        "two_blocks": text[:2 * BLOCK],
        "two_blocks_plus_one": text[:2 * BLOCK + 1],
        "run": b"a" * 300001,
        "runs_mixed": b"".join(bytes([65 + k % 7]) * (k * 37 % 1000 + 1) for k in range(600)),
        "repeat_32k_back": period * 4 + period[:1000],
        "repeat_32k_plus_one": (period + b"!") * 3,
        "random": rng.integers(0, 256, 3 * BLOCK + 77, dtype=np.uint8).tobytes(),
        "fixed6_text": text,
        "fixed6_mostly_zero": fixed6_text(zeros, 300),
        "fixed6_special": fixed6_text(special, 25),
    }


CASES = _cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_gzip_host_decodes(name):
    data = CASES[name]
    gz = gzip_host(data)
    assert gz[:10] == bytes([0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 255])
    assert zlib.decompress(gz, wbits=31) == data
    assert gzip.decompress(gz) == data
    assert int.from_bytes(gz[-8:-4], "little") == zlib.crc32(data)
    assert int.from_bytes(gz[-4:], "little") == len(data) % (1 << 32)
    assert inflate_own(gz) == data
    assert gzip_host(data) == gz


def test_gzip_host_random_is_stored():
    data = CASES["random"]
    gz = gzip_host(data)
    blocks = -(-len(data) // BLOCK)
    assert len(gz) == 18 + len(data) + 5 * blocks      # every block stored: 5 bytes of block header each


def test_gzip_host_empty_member():
    assert gzip_host(b"") == bytes([0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 255, 3, 0]) + bytes(8)


@pytest.mark.parametrize("name", ["fixed6_text", "fixed6_mostly_zero"])
def test_gzip_host_ratio_near_zlib_level1(name):
    data = CASES[name]
    assert len(gzip_host(data)) <= 1.10 * len(zlib.compress(data, 1))


def test_gzip_host_rejects_small_output():
    lib = _lib.load()
    src = np.zeros(100, dtype=np.uint8)
    out = np.zeros(50, dtype=np.uint8)
    got = np.zeros(1, dtype=np.int64)
    with pytest.raises(ValueError):
        _lib.check(lib.dca_gzip_host(src.ctypes.data, 100, out.ctypes.data, 50,
                                     got.ctypes.data_as(lib.dca_gzip_host.argtypes[4])), "dca_gzip_host")
