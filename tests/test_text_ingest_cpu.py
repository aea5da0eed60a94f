"""Host side shared by the device text parsers (data/text_ingest.py): the block/carry protocol and the cut rule, for
MatrixMarket and Stream.  No GPU needed: the device handle is replaced by a fake."""
import numpy as np
import pytest

from buffalo_b200.data import mm as mmmod
from buffalo_b200.data import stream as smod
from buffalo_b200.data.text_ingest import _Fallback, find_cut


class _FakeIngest(object):
    """Stands in for backend.MMIngest and backend.StreamIngest: records the fed blocks and declines the file at
    finish()."""
    block, blocks = 0, []

    def __init__(self, *args):
        self.bufs = [np.zeros(self.block, np.uint8), np.zeros(self.block, np.uint8)]

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass

    def staging(self, slot):
        return self.bufs[slot]

    def feed(self, slot, n, is_last):
        b = self.bufs[slot][:n].tobytes()
        assert is_last or b.endswith(b"\n")
        _FakeIngest.blocks.append((b, is_last))

    def finish(self):
        return dict(nnz=0, tokmask=0, reject_line=1, range_line=-1, n_slow=0, decline=1, decline_line=-1)


@pytest.mark.parametrize("fmt", ["mm", "stream"])
@pytest.mark.parametrize("block", [16, 64, 100, 4096])
@pytest.mark.parametrize("final_eol", [True, False])
def test_blocks_end_on_line_ends(tmp_path, monkeypatch, fmt, block, final_eol):
    """The caller carries the partial last line of a block into the next one: every block but the last ends with
    '\\n', and the blocks concatenate to the text after the header."""
    from buffalo_b200 import backend
    monkeypatch.setattr(backend, "MMIngest" if fmt == "mm" else "StreamIngest", _FakeIngest)
    monkeypatch.setattr(backend, "device_free_bytes", lambda: 1 << 40)
    body = "".join("%d %d %s\n" % (i % 7 + 1, i % 5 + 1, "1" * (i % 11 + 1)) for i in range(300))
    body = body if final_eol else body[:-1]
    p = tmp_path / "b.txt"
    _FakeIngest.block, _FakeIngest.blocks = block, []
    if fmt == "mm":
        p.write_text("%%MatrixMarket matrix coordinate real general\n7 5 300\n" + body)
        with pytest.raises(_Fallback):
            mmmod._device_ingest(str(p), 7, 5, 300, 2, None, None, block_bytes=block)
    else:
        p.write_text(body)
        with pytest.raises(_Fallback):
            smod._device_ingest(str(p), None, None, None, False, block_bytes=block)
    blocks = _FakeIngest.blocks
    assert b"".join(b for b, _ in blocks) == body.encode()
    assert [last for _, last in blocks] == [False] * (len(blocks) - 1) + [True]
    assert all(len(b) <= block for b, _ in blocks)


# MatrixMarket cuts within its longest accepted line; Stream anywhere in the block (here 3 MiB: several search windows)
@pytest.mark.parametrize("max_line", [mmmod.MAX_LINE, 3 << 20], ids=["mm", "stream"])
def test_find_cut(max_line):
    buf = np.frombuffer(b"ab c\nde f\ngh", np.uint8)
    assert find_cut(buf, len(buf), max_line) == 10
    fits = np.frombuffer(b"a\n" + b"x" * max_line, np.uint8)
    assert find_cut(fits, len(fits), max_line) == 2
    over = np.frombuffer(b"a\n" + b"x" * (max_line + 1), np.uint8)
    with pytest.raises(_Fallback):
        find_cut(over, len(over), max_line)
    with pytest.raises(_Fallback):                       # a block of one unterminated line
        find_cut(np.frombuffer(b"abcdef", np.uint8), 6, 6)
