"""Host side shared by the device text parsers (data/mm.py, data/stream.py): the decline exception, the block feed
through a parser handle's two pinned staging buffers and reads of byte ranges of the input."""
import mmap
import os
import time

import numpy as np


class _Fallback(Exception):
    """The device path declines the file; the host path builds it instead."""


def find_cut(buf, total, max_line):
    """End of the last line in buf[:total], one past its line feed, searched back over at most max_line + 1 bytes in
    1 MiB windows; _Fallback when there is none (a line longer than max_line bytes)."""
    stop, hi = max(0, total - max_line - 1), total
    while hi > stop:
        lo = max(stop, hi - (1 << 20))
        nl = np.flatnonzero(buf[lo:hi] == 10)
        if len(nl):
            return lo + int(nl[-1]) + 1
        hi = lo
    raise _Fallback("a line longer than %d bytes" % min(max_line, total - 1))


def feed_blocks(ing, fin, block, max_line, host_ms):
    """Feeds the rest of the binary file fin to the parser handle ing in blocks of at most `block` bytes, alternating
    its two staging slots.  Every block but the last ends on a line end: the partial last line is carried into the
    next block.  Adds the read time to host_ms["read"].  -> the last fed byte (b"\\n" when nothing was fed)."""
    size = os.fstat(fin.fileno()).st_size
    carry, slot, last_byte = b"", 0, b"\n"
    while True:
        buf = ing.staging(slot)
        k = len(carry)
        buf[:k] = np.frombuffer(carry, np.uint8)
        view, total = memoryview(buf), k
        t0 = time.perf_counter()
        while total < block:
            got = fin.readinto(view[total:])
            if not got:
                break
            total += got
        host_ms["read"] += 1e3 * (time.perf_counter() - t0)
        last = total < block or fin.tell() == size
        cut = total if last else find_cut(buf, total, max_line)
        carry = bytes(buf[cut:total])
        if cut:
            last_byte = bytes(buf[cut - 1:cut])
        ing.feed(slot, cut, last)
        if last:
            return last_byte
        slot ^= 1


def read_ranges(path, offsets, lengths):
    """bytes of the file at [offset, offset + length) for each (offset, length) pair"""
    with open(path, "rb") as f, mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ) as text:
        return [text[o:o + n] for o, n in zip(offsets.tolist(), lengths.tolist())]
