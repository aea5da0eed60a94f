"""Fast writer of large MatrixMarket test files: fixed-width, right-aligned integer columns formatted with NumPy, so
tens of millions of lines take seconds rather than minutes (np.savetxt formats line by line)."""
import numpy as np


def _digits(x, width):
    """uint8 [n, width]: x right-aligned in `width` columns, leading zeros as spaces."""
    x = np.asarray(x, dtype=np.int64)
    p = 10 ** np.arange(width - 1, -1, -1, dtype=np.int64)
    d = (x[:, None] // p) % 10 + ord("0")
    lead = (x[:, None] < p) & (p > 1)
    return np.where(lead, ord(" "), d).astype(np.uint8)


def format_lines(rows, cols, U, I, vals=None, decimal=False):
    """Bytes of the data lines "row col [val]\\n" (1-based rows / cols).  vals: integers; with decimal=True they are
    quarter steps written as "i.ff" (vals = 4 * value)."""
    parts = [_digits(rows, len(str(U))), np.full((len(rows), 1), ord(" "), np.uint8), _digits(cols, len(str(I)))]
    if vals is not None:
        vals = np.asarray(vals, dtype=np.int64)
        parts.append(np.full((len(rows), 1), ord(" "), np.uint8))
        if decimal:
            frac = (vals % 4) * 25
            parts += [_digits(vals // 4, 1), np.full((len(rows), 1), ord("."), np.uint8),
                      (frac[:, None] // np.array([10, 1]) % 10 + ord("0")).astype(np.uint8)]
        else:
            parts.append(_digits(vals, len(str(int(vals.max())))))
    parts.append(np.full((len(rows), 1), ord("\n"), np.uint8))
    return np.concatenate(parts, axis=1).tobytes()


def write_mm(path, U, I, rows, cols, vals=None, decimal=False, chunk=2_000_000):
    kind = "pattern" if vals is None else ("real" if decimal else "integer")
    with open(path, "wb") as f:
        f.write(("%%%%MatrixMarket matrix coordinate %s general\n%d %d %d\n" % (kind, U, I, len(rows))).encode())
        for s in range(0, len(rows), chunk):
            f.write(format_lines(rows[s:s + chunk], cols[s:s + chunk], U, I,
                                 None if vals is None else vals[s:s + chunk], decimal))
