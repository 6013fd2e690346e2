"""The preprocessing stages' rules (DESIGN.md §5s) pinned on the numpy restatement (tests/quantile_oracle.py) with
hand-computed answers, and every parameter refusal of Imputer, RobustScaler, MinMaxScaler, MaxAbsScaler, Bucketizer,
QuantileDiscretizer and approxQuantile.  No GPU needed."""
import math

import numpy as np
import pytest

import quantile_oracle as qo

NAN, INF = float("nan"), float("inf")


def test_imputer_hand_answers():
    a, b = [1, 2, NAN, 4, 5], [NAN, NAN, 3, 4, 5]
    assert (qo.mean(a), qo.mean(b)) == (3.0, 4.0)
    assert (qo.quantiles(a, [0.5])[0], qo.quantiles(b, [0.5])[0]) == (2.0, 4.0)
    assert list(qo.fill(np.array(a), 3.0)) == [1, 2, 3, 4, 5]


def test_rank_rule_is_fp64_ceil():
    assert 0.14 * 50 == 7.000000000000001 and qo.target_rank(0.14, 50) == 8
    assert 0.7 * 10 == 7.0 and qo.target_rank(0.7, 10) == 7
    v = np.arange(1.0, 51.0)
    assert qo.quantiles(v, [0.14])[0] == 8.0
    assert qo.target_rank(0.0, 9) == 1 and qo.target_rank(1.0, 9) == 9 and qo.target_rank(1e-300, 9) == 1


def test_signed_zero_infinities_and_all_nan():
    q = qo.quantiles([0.0, -0.0, 0.0, -0.0, 1.0], [0.0, 0.4, 0.41, 1.0])
    assert [math.copysign(1, v) for v in q[:3]] == [-1, -1, 1] and q[3] == 1.0
    assert list(qo.quantiles([INF, -INF, 2.0, NAN], [0.0, 0.5, 1.0])) == [-INF, 2.0, INF]
    assert qo.quantiles([NAN, NAN], [0.5]).shape == (0,)
    assert math.isnan(qo.mean([NAN])) and math.isnan(qo.mode([NAN]))
    assert qo.mean([1.0, INF]) == INF and math.isnan(qo.mean([INF, -INF]))


def test_mode_ties_take_the_smallest_and_fold_signed_zero():
    assert qo.mode([3, 3, 1, 1, 2]) == 1.0
    assert qo.mode([-0.0, 0.0, 5, 5]) == 0.0
    assert qo.mode([7, 9, 9, 7, 4], missing=9) == 7.0


def test_missing_value_and_casts():
    assert qo.mean([1, 2, -1, 6], missing=-1) == 3.0
    assert qo.cast(2.7, "i32") == 2 and qo.cast(-2.7, "i32") == -2 and qo.cast(NAN, "i32") == 0
    assert qo.cast(1e12, "i32") == 2 ** 31 - 1 and qo.cast(0.1, "f32") == float(np.float32(0.1))


def test_bucketizer_edges():
    s = [-0.5, 0.0, 0.5, 1.0]
    assert [qo.bucket(x, s) for x in (-0.5, -0.1, 0.0, 0.2, 0.5, 0.9, 1.0)] == [0, 0, 1, 1, 2, 2, 2]
    assert qo.bucket(NAN, s) == 3.0
    assert qo.bucket(-0.0, s) == 0.0                        # Arrays.binarySearch: -0.0 sorts below the split 0.0
    for x in (-0.6, 1.1, INF):
        with pytest.raises(qo.OutOfBounds):
            qo.bucket(x, s)
    with pytest.raises(ValueError):
        qo.bucket(NAN, s, keep=False)
    inf_s = [-INF, 0.0, INF]
    assert qo.bucket(INF, inf_s) == 1.0 and qo.bucket(-INF, inf_s) == 0.0


def test_discretizer_distinct_splits_and_doctest():
    assert qo.distinct_splits([5.0, -0.0, 0.0, 0.0, 2.0, 2.0, 9.0]) == [-INF, 0.0, 2.0, INF]
    v = [0.1, 0.4, 1.2, 1.5, NAN, NAN]
    s = qo.discretizer_splits(v, 2)
    assert s == [-INF, 0.4, INF]
    assert [qo.bucket(x, s) for x in v] == [0, 1, 1, 1, 2, 2]
    assert qo.discretizer_splits([3.0] * 10, 4) == [-INF, 3.0, INF]


def test_min_max_constant_column_and_nan():
    x = np.array([[1.0, 5.0], [3.0, 5.0], [NAN, 5.0]])
    out = qo.min_max(x, [1.0, 5.0], [3.0, 5.0], lo=-1.0, hi=1.0)
    assert out[0, 0] == -1.0 and out[1, 0] == 1.0 and math.isnan(out[2, 0]) and list(out[:, 1]) == [0.0] * 3


def _refuses(stage, action="fit"):
    from pyspark.ml.feature import IllegalArgumentException
    with pytest.raises(IllegalArgumentException):
        stage.fit(None) if action == "fit" else stage.transform(None)


def test_parameter_refusals():
    from pyspark.ml.feature import (Bucketizer, Imputer, MinMaxScaler, QuantileDiscretizer, RobustScaler)
    _refuses(Imputer(inputCols=["a"], outputCols=["b"], strategy="median_ish"))
    _refuses(Imputer(inputCols=["a"], outputCols=["b"], relativeError=1.5))
    _refuses(Imputer(inputCols=["a", "b"], outputCols=["c"]))
    _refuses(Imputer(inputCol="a", inputCols=["a"], outputCols=["b"]))
    _refuses(RobustScaler(inputCol="f", outputCol="o", lower=0.8, upper=0.2))
    _refuses(RobustScaler(inputCol="f", outputCol="o", upper=1.5))
    _refuses(RobustScaler(inputCol="f", outputCol="o", relativeError=-0.1))
    _refuses(MinMaxScaler(inputCol="f", outputCol="o", min=1.0, max=1.0))
    _refuses(QuantileDiscretizer(inputCol="a", outputCol="b", numBuckets=1))
    _refuses(QuantileDiscretizer(inputCol="a", outputCol="b", handleInvalid="drop"))
    _refuses(QuantileDiscretizer(inputCol="a", outputCol="b", relativeError=2.0))
    _refuses(QuantileDiscretizer(inputCols=["a", "b"], outputCols=["c", "d"], numBucketsArray=[3]))
    _refuses(Bucketizer(splits=[0.0, 1.0], inputCol="a", outputCol="b"), "transform")
    _refuses(Bucketizer(splits=[0.0, 2.0, 1.0], inputCol="a", outputCol="b"), "transform")
    _refuses(Bucketizer(splits=[0.0, 0.0, 1.0], inputCol="a", outputCol="b"), "transform")
    _refuses(Bucketizer(splits=[0.0, NAN, 1.0], inputCol="a", outputCol="b"), "transform")
    _refuses(Bucketizer(splitsArray=[[0.0, 1.0, 2.0]], inputCols=["a", "b"], outputCols=["c", "d"]), "transform")


def test_quantile_probability_and_splits_helpers():
    from b200flow import quantile as q
    from pyspark.ml.feature import distinct_splits
    with pytest.raises(ValueError):
        q.check_probabilities([0.5, 1.01])
    with pytest.raises(ValueError):
        q.check_probabilities([-0.1])
    assert q.target_rank(0.14, 50) == 8 and q.target_rank(0.0, 3) == 1
    assert distinct_splits([1.0, -0.0, 0.0, 3.0, 3.0, 4.0]) == qo.distinct_splits([1.0, -0.0, 0.0, 3.0, 3.0, 4.0])
    for code, kind in ((q.F32, "f32"), (q.F64, "f64"), (q.I32, "i32")):
        for v in (2.7, -2.7, NAN, 1e12, -1e12, 0.1):
            a, b = q.cast_surrogate(v, code), qo.cast(v, kind)
            assert a == b or (a != a and b != b)
