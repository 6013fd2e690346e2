"""LinearSVC on the CPU: the shim's params and refusals, lbfgs as a driver of lbfgs_steps, and the numpy restatement
(tests/svc_oracle.py) against finite differences and against the QP solver; the optimiser on the restatement reaches the
QP optimum within the tolerance the GPU tests use."""
import numpy as np
import pytest
import torch

import svc_oracle as so


class _Frame:
    """the two columns LinearSVC._fit reads, on the host"""

    def __init__(self, x, y, meta=None):
        from pyspark.sql import ColumnData
        self._cols = {"features": ColumnData("vector", torch.as_tensor(x), "f64"),
                      "label": ColumnData("numeric", torch.as_tensor(y, dtype=torch.float64), "f64", meta)}

    def _column_tensor(self, name):
        return self._cols[name].data


def test_defaults_and_param_validation():
    from pyspark.ml.classification import LinearSVC
    from pyspark.ml.feature import IllegalArgumentException
    s = LinearSVC()
    want = {"maxIter": 100, "regParam": 0.0, "tol": 1e-6, "fitIntercept": True, "standardization": True, "threshold": 0.0,
            "aggregationDepth": 2, "maxBlockSizeInMB": 0.0, "weightCol": None, "featuresCol": "features",
            "labelCol": "label", "predictionCol": "prediction", "rawPredictionCol": "rawPrediction"}
    assert {k: s.getOrDefault(k) for k in want} == want
    p = LinearSVC(maxIter=7, regParam=0.5, tol=0.0, fitIntercept=False, standardization=False)._check()
    assert (p.max_iter, p.reg_param, p.tol, p.fit_intercept, p.standardization) == (7, 0.5, 0.0, False, False)
    assert LinearSVC(maxIter=0, aggregationDepth=2, maxBlockSizeInMB=1.5)._check().max_iter == 0
    for bad in ({"maxIter": -1}, {"maxIter": 2.5}, {"regParam": -0.1}, {"tol": -1e-9}, {"aggregationDepth": 1},
                {"aggregationDepth": 2.5}, {"maxBlockSizeInMB": -1.0}, {"weightCol": "w"}):
        with pytest.raises(IllegalArgumentException):
            LinearSVC(**bad)._check()
    with pytest.raises(TypeError):
        LinearSVC(probabilityCol="p")


def test_two_classes_are_required_and_labels_must_be_valid():
    from pyspark.ml.classification import LinearSVC
    from pyspark.ml.feature import IllegalArgumentException
    x = np.zeros((4, 2))
    with pytest.raises(IllegalArgumentException, match="LinearSVC only supports binary classification. 3 classes detected "
                                                       "in label"):
        LinearSVC().fit(_Frame(x, [0, 1, 2, 1]))
    with pytest.raises(IllegalArgumentException, match="1 classes detected"):
        LinearSVC().fit(_Frame(x, [0, 0, 0, 0]))
    meta = {"ml_attr": {"type": "nominal", "vals": ["a", "b", "c"]}}
    with pytest.raises(IllegalArgumentException, match="3 classes detected"):
        LinearSVC().fit(_Frame(x, [0, 1, 1, 0], meta))
    for y in ([0, 1, -1, 1], [0, 1, 0.5, 1]):
        with pytest.raises(IllegalArgumentException, match="invalid label"):
            LinearSVC().fit(_Frame(x, y))
    with pytest.raises(IllegalArgumentException, match="weightCol"):
        LinearSVC(weightCol="w").fit(_Frame(x, [0, 1, 0, 1]))


def _quadratic_problem(seed, D=6):
    rng = np.random.default_rng(seed)
    A = rng.normal(0, 1, (D, D))
    H = torch.from_numpy(A @ A.T + 0.1 * np.eye(D))
    c = torch.from_numpy(rng.normal(0, 1, D))

    def smooth(v):
        return 0.5 * (v @ (H @ v)) - c @ v + torch.log1p((v * v).sum()), H @ v - c + 2 * v / (1 + (v * v).sum())
    return smooth, torch.from_numpy(rng.normal(0, 1, D))


@pytest.mark.parametrize("l1", [None, "zeros", "weights"])
def test_lbfgs_equals_driving_its_steps_by_hand(l1):
    from b200flow.linear import lbfgs, lbfgs_steps
    smooth, v0 = _quadratic_problem(3)
    w = {None: None, "zeros": torch.zeros(6, dtype=torch.float64), "weights": torch.full((6,), 0.3, dtype=torch.float64)}[l1]
    v, hist, it = lbfgs(smooth, v0.clone(), 50, 1e-12, 10, l1=w)
    gen = lbfgs_steps(v0.clone(), 50, 1e-12, 10, l1=w)
    point, calls = next(gen), 1
    while True:
        try:
            point = gen.send(smooth(point))
            calls += 1
        except StopIteration as stop:
            v2, hist2, it2 = stop.value
            break
    assert it > 3 and calls > it
    assert torch.equal(v, v2) and [h.hex() for h in hist] == [h.hex() for h in hist2] and it == it2


def test_restatement_gradient_matches_finite_differences():
    x, y = so.blobs(400, 5, 1.0, 2)
    rng = np.random.default_rng(5)
    for reg, st, fi in ((0.3, True, True), (0.2, False, True), (0.0, True, False)):
        w = rng.normal(0, 0.5, 6)
        if not fi:
            w[-1] = 0.0
        f, g = so.objective(w, x, y, reg, st, fi)
        xs = x * so.inv_std(x)
        margins = 1.0 - (2 * y - 1) * (xs @ w[:-1] + w[-1])
        h = 1e-6
        assert np.min(np.abs(margins)) > 1e-4            # no row sits on a kink within the step
        for j in range(6 if fi else 5):
            e = np.zeros(6)
            e[j] = h
            fd = (so.objective(w + e, x, y, reg, st, fi)[0] - so.objective(w - e, x, y, reg, st, fi)[0]) / (2 * h)
            assert abs(fd - g[j]) <= 1e-7 * max(1.0, abs(g[j])), (reg, st, fi, j)
        if not fi:
            assert g[-1] == 0.0


def test_qp_solution_is_the_restatement_minimum():
    x, y = so.blobs(120, 3, 1.0, 7)
    w, f = so.qp_solve(x, y, 0.05)
    assert f == so.objective(w, x, y, 0.05)[0]
    rng = np.random.default_rng(1)
    for _ in range(200):                                  # no nearby point does better
        assert so.objective(w + rng.normal(0, 1e-3, 4), x, y, 0.05)[0] >= f - 1e-12
    # the subgradient condition: 0 lies in the subdifferential, so the smooth part's gradient is small off the kinks
    assert f > 0.0 and np.isfinite(f)


# the relative objective gap to the QP optimum that LinearSVC is required to reach (tests/test_svc_gpu.py).  The hinge is
# piecewise linear: the quasi-Newton directions and backtracking line search stall on its kinks, so the iterates stop
# short of the optimum by far more than 1e-6.  The restatement run below, the same optimiser on the same objective, ends
# between 1.0e-5 and 1.12e-4 above the SLSQP optimum on these six problems; 2.5e-4 is about twice the largest, room for
# the device sums' different rounding to send the line search down a slightly different path.
FIT_GAP = 2.5e-4
FIT_CASES = [(3.0, 0.01, True, True), (3.0, 0.1, False, True), (3.0, 0.05, True, False), (0.7, 0.01, True, True),
             (0.7, 0.1, False, True), (0.7, 0.05, True, False)]


@pytest.mark.parametrize("gap,reg,st,fi", FIT_CASES)
def test_the_optimiser_on_the_restatement_reaches_the_qp_optimum(gap, reg, st, fi):
    from b200flow.linear import lbfgs
    x, y = so.blobs(200, 5, gap, 4, constant=2)
    _, fq = so.qp_solve(x, y, reg, st, fi)

    def smooth(v):
        f, g = so.objective(v.numpy(), x, y, reg, st, fi)
        return torch.tensor(f, dtype=torch.float64), torch.from_numpy(g)
    z = torch.zeros(6, dtype=torch.float64)
    v, _, _ = lbfgs(smooth, z.clone(), 1000, 1e-12, 10, l1=z)
    f = so.objective(v.numpy(), x, y, reg, st, fi)[0]
    assert -1e-9 <= (f - fq) / fq <= FIT_GAP and v[2] == 0.0, (f - fq) / fq
