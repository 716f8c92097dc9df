"""numpy restatement of one RigL drop-and-regrow update per layer: what ``ops.rigl_select`` and ``ops.rigl_apply`` must
produce, element for element.

Keys are the fp32 bit patterns of |x| (sign bit cleared) read as unsigned integers, so NaN sorts above +inf.
DROP takes the k smallest |w| keys among mask != 0, GROW the k largest |g| keys among the positions that are 0 after
the drop; ties go to the lower flat index first.  k above the active count drops all of them, and the grow takes as many
as the drop took, so the active count never changes."""
import numpy as np


def keys(x):
    return np.ascontiguousarray(x, dtype=np.float32).reshape(-1).view(np.uint32) & np.uint32(0x7FFFFFFF)


def select(w, g, m, k):
    """(new mask float32, dropped, grown) for one layer."""
    m = np.asarray(m, dtype=np.float32).reshape(-1)
    active = m != 0
    kw, kg = keys(w), keys(g)
    a = np.flatnonzero(active)
    nd = min(int(k), a.size)
    drop = a[np.argsort(kw[a], kind="stable")[:nd]]          # stable: equal keys keep index order
    new = active.copy()
    new[drop] = False
    b = np.flatnonzero(~new)
    ng = min(nd, b.size)
    grow = b[np.argsort(~kg[b], kind="stable")[:ng]]          # complement: largest key first, ties still in index order
    new[grow] = True
    return new.astype(np.float32), nd, ng


def apply(m, new, w, buf=None):
    """(mask, w, buf) after the update: mask <- new; grown positions (new != 0, old == 0) restart at w = 0, buf = 0."""
    m = np.asarray(m, dtype=np.float32).reshape(-1)
    new = np.asarray(new, dtype=np.float32).reshape(-1)
    grown = (new != 0) & (m == 0)
    w = np.array(w, dtype=np.float32).reshape(-1)
    w[grown] = 0.0
    if buf is not None:
        buf = np.array(buf, dtype=np.float32).reshape(-1)
        buf[grown] = 0.0
    return new.copy(), w, buf
