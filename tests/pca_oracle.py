"""numpy fp64 restatement of PCA and Pearson correlation (DESIGN.md §5h): the mean from sequential chunk-order column sums,
the centred Gram matrix in two passes, the covariance, the components from numpy's eigh with the sign rule, the uncentred
transform and Pearson's r.  Written from the formulas, independently of csrc/pca.cu and b200flow/pca.py."""
import numpy as np

CHUNK = 4096


def chunks(n, row_offset=0):
    """the local row ranges [lo, hi) of the 4096-row global chunks that rows [row_offset, row_offset + n) touch."""
    out, g = [], row_offset // CHUNK * CHUNK
    while g < row_offset + n:
        out.append((max(g, row_offset) - row_offset, min(g + CHUNK, row_offset + n) - row_offset))
        g += CHUNK
    return out


def column_sums(x, row_offset=0):
    """per chunk the rows added one by one from +0.0 in row order; the chunks' sums added in chunk order from +0.0."""
    total = np.zeros(x.shape[1])
    for lo, hi in chunks(x.shape[0], row_offset):
        acc = np.zeros(x.shape[1])
        for r in x[lo:hi]:
            acc = acc + r
        total = total + acc
    return total


def mean(x, row_offset=0):
    return column_sums(x, row_offset) * (1.0 / x.shape[0])


def pack(q):
    """the upper triangle of q [D, D], (a, b) with a <= b at a + b(b+1)/2."""
    D = q.shape[0]
    out = np.empty(D * (D + 1) // 2)
    for b in range(D):
        out[b * (b + 1) // 2:b * (b + 1) // 2 + b + 1] = q[:b + 1, b]
    return out


def gram_partials(x, shift=None, row_offset=0):
    """[(sum (x - shift)(x - shift)^T, sum |x - shift| |x - shift|^T)] per chunk: the partial and the scale of its rounding."""
    out = []
    for lo, hi in chunks(x.shape[0], row_offset):
        c = x[lo:hi] - (0.0 if shift is None else shift)
        out.append((c.T @ c, np.abs(c).T @ np.abs(c)))
    return out


def covariance(x, row_offset=0):
    """(mean, C): C = Q (1.0 / (n - 1)), Q the centred Gram matrix with the chunks added in chunk order."""
    n = x.shape[0]
    if n <= 1:
        raise ValueError("Cannot compute the covariance of a RowMatrix with <= 1 row.")
    m = mean(x, row_offset)
    q = np.zeros((x.shape[1], x.shape[1]))
    for p, _ in gram_partials(x, m, row_offset):
        q = q + p
    c = np.triu(q) * (1.0 / (n - 1))
    return m, c + np.triu(c, 1).T


def components(cov, k):
    """(pc [D, k], explainedVariance [k]): eigenvalue magnitudes descending (stable on eigh's output reversed), every
    column's entry of largest magnitude positive (the lowest index among equal magnitudes), s / sum(s)."""
    d, U = np.linalg.eigh(cov)
    s, U = np.abs(d)[::-1], U[:, ::-1]
    order = np.argsort(-s, kind="stable")
    s, U = s[order], U[:, order]
    total = 0.0
    for v in s:
        total = total + v
    pc = U[:, :k].copy()
    for j in range(k):
        col = pc[:, j]
        top = 0
        for i in range(1, col.shape[0]):
            if abs(col[i]) > abs(col[top]):
                top = i
        if col[top] < 0:
            pc[:, j] = -col
    with np.errstate(invalid="ignore", divide="ignore"):
        return pc, s[:k] / np.float64(total)


def fit(x, k):
    """(pc, explainedVariance, mean, cov)."""
    D = x.shape[1]
    if k is None or int(k) != k or not 1 <= k <= D:
        raise ValueError("source vector size %d must be no less than k" % D)
    m, c = covariance(x)
    pc, ev = components(c, int(k))
    return pc, ev, m, c


def transform(x, pc):
    """y = pc^T x per row; the mean is not subtracted."""
    return x @ pc


def pearson(x):
    _, c = covariance(x)
    D = c.shape[0]
    r = np.empty((D, D))
    with np.errstate(invalid="ignore", divide="ignore"):
        for a in range(D):
            for b in range(D):
                r[a, b] = c[a, b] / (np.sqrt(c[a, a]) * np.sqrt(c[b, b]))
                if a == b:
                    r[a, b] = 1.0
                if c[a, a] == 0 or c[b, b] == 0:
                    r[a, b] = np.nan
    return r
