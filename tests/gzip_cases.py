"""gzip streams of count text for the inflate tests, all made with Python's zlib: levels, strategies, memory levels,
window sizes, flush points, concatenated members, hand-built header fields, and edge inputs."""
import struct
import zlib

import numpy as np


def count_text(n_bytes, seed=0):
    """About n_bytes of a tab-separated count table: a header, then gene lines of NB-like counts."""
    rng = np.random.default_rng(seed)
    cols = 200
    lines = ["gene\t" + "\t".join("c%d" % j for j in range(cols))]
    size = len(lines[0])
    g = 0
    while size < n_bytes:
        v = rng.negative_binomial(2, 0.5, cols) * (rng.random(cols) < 0.28)
        line = "g%d\t" % g + "\t".join(map(str, v))
        lines.append(line)
        size += len(line) + 1
        g += 1
    return ("\n".join(lines) + "\n").encode()


def raw_deflate(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, mem=8, wbits=15, flush_every=0,
                flush=zlib.Z_SYNC_FLUSH):
    c = zlib.compressobj(level, zlib.DEFLATED, -wbits, mem, strategy)
    if not flush_every:
        return c.compress(data) + c.flush()
    out = []
    for i in range(0, len(data), flush_every):
        out.append(c.compress(data[i:i + flush_every]))
        out.append(c.flush(flush))
    out.append(c.flush())
    return b"".join(out)


def member(data, flags=0, extra=b"", name=b"", comment=b"", deflated=None, **kw):
    """One gzip member built by hand: FTEXT / FEXTRA / FNAME / FCOMMENT / FHCRC as flagged."""
    h = bytearray(b"\x1f\x8b\x08" + bytes([flags]) + b"\x00\x00\x00\x00\x00\xff")
    if flags & 4:
        h += struct.pack("<H", len(extra)) + extra
    if flags & 8:
        h += name + b"\x00"
    if flags & 16:
        h += comment + b"\x00"
    if flags & 2:
        h += struct.pack("<H", zlib.crc32(bytes(h)) & 0xffff)
    body = raw_deflate(data, **kw) if deflated is None else deflated
    return bytes(h) + body + struct.pack("<II", zlib.crc32(data), len(data) & 0xffffffff)


def stored_with_deflate_inside(size=20_000):
    """A valid member of one stored block whose content, from the first byte of the second 32 KB of the file on, is a
    Huffman-only deflate stream cut short: a plausible dynamic block start that no decoder reaching the end of the
    file may hang on."""
    cut = raw_deflate(count_text(200_000, seed=7), strategy=zlib.Z_HUFFMAN_ONLY)[:size]
    payload = count_text(32768 - 5, seed=8)[:32768 - 5] + cut        # header 10 bytes + block header 5 bytes before
    stored = b"\x01" + struct.pack("<HH", len(payload), len(payload) ^ 0xffff) + payload
    return member(payload, deflated=stored), payload


def cases(size=150_000):
    """name -> (gzip bytes, inflated bytes)."""
    text = count_text(size)
    out = {}
    for lv in range(10):
        out["level%d" % lv] = text, dict(level=lv)
    for name, st in (("filtered", zlib.Z_FILTERED), ("huffman_only", zlib.Z_HUFFMAN_ONLY), ("rle", zlib.Z_RLE),
                     ("fixed", zlib.Z_FIXED)):
        out["strategy_" + name] = text, dict(strategy=st)
    out["mem1"] = text, dict(mem=1)
    out["mem9"] = text, dict(mem=9, level=9)
    for w in range(9, 16):
        out["window%d" % w] = text, dict(wbits=w)
    out["sync_flush"] = text, dict(flush_every=7001, flush=zlib.Z_SYNC_FLUSH)
    out["full_flush"] = text, dict(flush_every=9973, flush=zlib.Z_FULL_FLUSH)
    out["all_zeros"] = bytes(size * 8), dict(level=9)
    out["random"] = np.random.default_rng(1).integers(0, 256, size, dtype=np.uint8).tobytes(), dict()
    res = {k: (member(d, **kw), d) for k, (d, kw) in out.items()}
    parts = [text[:40_000], text[40_000:40_001], b"", text[40_001:]]
    res["members"] = (b"".join([member(parts[0], flags=1, level=1), member(parts[1], flags=4 | 8, extra=b"ab\x00cd",
                                                                          name=b"x.tsv"),
                                member(parts[2], flags=16 | 2, comment=b"empty"),
                                member(parts[3], flags=2 | 8 | 16, name=b"n", comment=b"c", level=9)]), text)
    res["stored_with_deflate_inside"] = stored_with_deflate_inside()
    res["empty"] = member(b""), b""
    res["one_byte"] = member(b"7"), b"7"
    for n in (32 * 1024 - 1, 32 * 1024, 32 * 1024 + 1, 3 * 32 * 1024 + 5):   # compressed sizes around span regions
        d = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes()
        res["stored_%d" % n] = member(d, level=0), d
    return res
