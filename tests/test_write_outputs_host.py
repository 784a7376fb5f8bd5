"""Host-side pieces of the GPU output writer: the gene-block sizing of Autoencoder.write_predictions, the label and
header bytes io.write_text_matrix_device hands to the device (against the host writer's files), and the number
formatter of csrc/write_text.cu run on the CPU (dca_format_fixed6_host) against Python's '%.6f'."""
import numpy as np
import pytest


def test_gene_block_sizing():
    from dca_b200.network import gene_block
    mb = 1 << 20
    assert gene_block(1000, 500, 3, 10 ** 12) == 500                       # everything fits: one block
    assert gene_block(1000, 500, 3, 10 ** 12, max_block_bytes=12000 * 70) == 70
    assert gene_block(1000, 500, 3, 2 * 12000 * 70) == 70                  # half of the free memory
    assert gene_block(10 ** 6, 20000, 3, 80 * 1024 * mb) == (40 * 1024 * mb) // (12 * 10 ** 6)
    assert gene_block(10 ** 6, 20000, 3, 0) == 1                            # never below one gene
    assert gene_block(5000, 512, 0, 10 ** 9) == 512                         # latent only: one pass
    # the block does not depend on the cell count through anything but the device bytes
    for n in (10 ** 3, 10 ** 5, 10 ** 7):
        b = gene_block(n, 30000, 2, 64 << 30, max_block_bytes=1 << 30)
        assert 8 * n * b <= 1 << 30 and (b == 30000 or 8 * n * (b + 1) > 1 << 30)


def test_quote_label():
    from dca_b200.io import quote_label
    assert quote_label("gene1") == b"gene1"
    assert quote_label(7) == b"7"
    assert quote_label("a\tb") == b'"a\tb"'
    assert quote_label('say "hi"') == b'"say ""hi"""'
    assert quote_label("x\ny") == b'"x\ny"'
    assert quote_label("x\ry") == b'"x\ry"'
    assert quote_label("ünï") == "ünï".encode()
    assert quote_label("") == b""


def test_label_bytes():
    from dca_b200.io import label_bytes
    data, off = label_bytes(["a", 'b"', "", "cc"], 4)
    assert data == b'a"b"""cc' and off.tolist() == [0, 1, 6, 6, 8] and off.dtype == np.int64
    with pytest.raises(ValueError, match="labels"):
        label_bytes(["a"], 2)


NAMES = ["plain", "tab\there", 'quo"te', "new\nline", "cr\rx", "", "ünï", "12"]


@pytest.mark.parametrize("rows", [False, True])
def test_header_bytes_match_host_writer(tmp_path, rows):
    from dca_b200.io import header_bytes, write_text_matrix
    m = np.zeros((3, len(NAMES)), np.float32)
    path = str(tmp_path / "m.tsv")
    write_text_matrix(m, path, rownames=["r0", "r1", "r2"] if rows else None, colnames=NAMES)
    head = header_bytes(NAMES, rows)
    assert open(path, "rb").read()[:len(head)] == head
    assert head.endswith(b"\n") and head.startswith(b"\t") == rows


def test_label_lines_match_host_writer(tmp_path):
    """Each line of the host writer starts with label_bytes' label and a tab."""
    from dca_b200.io import label_bytes, write_text_matrix
    m = np.ones((len(NAMES), 2), np.float32)
    path = str(tmp_path / "m.tsv")
    write_text_matrix(m, path, rownames=NAMES)
    data, off = label_bytes(NAMES, len(NAMES))
    expect = b"".join(data[a:b] + b"\t1.000000\t1.000000\n" for a, b in zip(off[:-1], off[1:]))
    assert open(path, "rb").read() == expect


def _format_host(bits):
    from dca_b200 import _lib
    lib = _lib.load()
    bits = np.ascontiguousarray(bits, dtype=np.uint32)
    out = np.zeros(47 * bits.size + 1, np.uint8)
    off = np.zeros(bits.size + 1, np.int64)
    _lib.check(lib.dca_format_fixed6_host(bits.ctypes.data, bits.size, out.ctypes.data, off.ctypes.data),
               "dca_format_fixed6_host")
    b = out[:off[-1]].tobytes()
    return [b[off[i]:off[i + 1]].decode() for i in range(bits.size)]


def test_formatter_host_build_matches_printf():
    rng = np.random.default_rng(1)
    e = np.arange(256, dtype=np.uint32) << 23
    parts = [rng.integers(0, 2 ** 32, 200000, dtype=np.uint64).astype(np.uint32)]
    for m in (0, 1, 2, 2 ** 23 - 1):
        parts += [e | m, e | m | 0x80000000]
    ties = (np.arange(1, 1024)[None, :] / 2.0 ** np.arange(1, 40)[:, None]).astype(np.float32).ravel()
    bnd = ((np.arange(0, 20000) + 0.5) / 1e6).astype(np.float32)
    vals = np.concatenate([ties, bnd, np.nextafter(bnd, np.float32(1)), np.nextafter(bnd, np.float32(-1)),
                           np.array([0.0078125, -0.0, -1e-7, 8e9, 3.4028235e38, 1e-45, np.nan, np.inf, -np.inf],
                                    np.float32)])
    parts.append(vals.view(np.uint32))
    bits = np.concatenate(parts)
    ref = ["" if v != v else "%.6f" % v for v in bits.view(np.float32).astype(np.float64).tolist()]
    assert _format_host(bits) == ref
