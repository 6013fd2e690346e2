"""OneVsRest without a GPU: param validation and its messages, the number of classes from the label metadata or the largest
label, copy() forwarding a param map to the classifier, and Spark's Vector.argmax rule (ties, NaN, -0.0) on CPU tensors."""
import math

import pytest
import torch

from pyspark.ml.classification import (GBTClassifier, LogisticRegression, OneVsRest, RandomForestClassifier, _first_argmax,
                                       _ovr_num_classes)
from pyspark.ml.feature import IllegalArgumentException
from pyspark.sql import ColumnData, DataFrame


def _frame(labels, meta=None):
    y = torch.tensor(labels, dtype=torch.float64)
    cols = {"features": ColumnData("vector", torch.zeros((len(labels), 2), dtype=torch.float64), "f64"),
            "label": ColumnData("numeric", y, "f64", meta)}
    return DataFrame(len(labels), None, None, {}, cols)


def test_params_and_their_validation():
    ovr = OneVsRest()
    assert ovr.getFeaturesCol() == "features" and ovr.getLabelCol() == "label" and ovr.getPredictionCol() == "prediction"
    assert ovr.getRawPredictionCol() == "rawPrediction" and ovr.getParallelism() == 1 and ovr.getClassifier() is None
    with pytest.raises(IllegalArgumentException, match="needs the classifier"):
        ovr.fit(_frame([0, 1, 2]))
    with pytest.raises(IllegalArgumentException, match="must be a classifier"):
        OneVsRest(classifier="gbt").fit(_frame([0, 1, 2]))
    with pytest.raises(IllegalArgumentException, match="must be a classifier"):
        OneVsRest(classifier=OneVsRest(classifier=GBTClassifier())).fit(_frame([0, 1]))
    with pytest.raises(IllegalArgumentException, match="weightCol"):
        OneVsRest(classifier=GBTClassifier(), weightCol="w").fit(_frame([0, 1, 2]))
    for bad in (0, -1, 1.5, True):
        with pytest.raises(IllegalArgumentException, match="parallelism"):
            OneVsRest(classifier=GBTClassifier(), parallelism=bad).fit(_frame([0, 1, 2]))
    gbt = GBTClassifier()
    assert OneVsRest(classifier=gbt, parallelism=4)._check() is gbt
    with pytest.raises(TypeError):
        OneVsRest(probabilityCol="p")                                # no probability column in Spark's OneVsRest
    with pytest.raises(IllegalArgumentException, match="does not exist"):
        OneVsRest(classifier=gbt, labelCol="nope").fit(_frame([0, 1]))


def test_number_of_classes():
    assert _ovr_num_classes(_frame([0, 1, 4, 2]), "label") == 5
    # nominal metadata wins over the values: a class absent from the rows still counts
    assert _ovr_num_classes(_frame([0, 1], {"ml_attr": {"type": "nominal", "vals": ["a", "b", "c"]}}), "label") == 3
    assert _ovr_num_classes(_frame([]), "label") == 0
    for bad in ([0, 1.5], [0, -1]):
        with pytest.raises(IllegalArgumentException, match="invalid label"):
            _ovr_num_classes(_frame(bad), "label")


def test_copy_forwards_the_param_map_to_the_classifier():
    gbt = GBTClassifier(maxDepth=5)
    ovr = OneVsRest(classifier=gbt)
    c = ovr.copy({gbt.maxDepth: 3, ovr.predictionCol: "p"})
    assert c.getClassifier().getMaxDepth() == 3 and c.getPredictionCol() == "p"
    assert c.getClassifier().uid == gbt.uid and c.getClassifier() is not gbt
    assert gbt.getMaxDepth() == 5 and ovr.getPredictionCol() == "prediction"      # the originals are untouched
    rf = RandomForestClassifier()
    c2 = ovr.copy({rf.numTrees: 7})                                   # a param of another estimator reaches nobody
    assert c2.getClassifier().getMaxDepth() == 5 and not c2.getClassifier().hasParam("numTrees")
    assert ovr.copy().getClassifier() is gbt
    lr = LogisticRegression()
    assert OneVsRest(classifier=lr).copy({lr.regParam: 0.5}).getClassifier().getRegParam() == 0.5


def test_argmax_is_sparks_first_strict_maximum():
    nan, inf = math.nan, math.inf
    raw = torch.tensor([[1.0, 3.0, 3.0],            # tie: the first
                        [2.0, 2.0, 2.0],
                        [0.0, -0.0, 0.0],           # -0.0 == +0.0: index 0
                        [-0.0, 0.0, -1.0],
                        [nan, 5.0, 7.0],            # NaN at 0: nothing is > NaN
                        [1.0, nan, 0.5],            # NaN later is never chosen
                        [1.0, nan, 2.0],
                        [-inf, -inf, -5.0],
                        [-1.0, -2.0, -0.5]], dtype=torch.float64)
    assert _first_argmax(raw).tolist() == [1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 2.0, 2.0, 2.0]
    assert torch.argmax(raw[4:5], 1).item() == 0 and torch.argmax(raw[5:6], 1).item() == 1   # why torch.argmax is not used
    assert _first_argmax(torch.zeros((3, 1), dtype=torch.float64)).tolist() == [0.0, 0.0, 0.0]
    assert _first_argmax(torch.zeros((2, 0), dtype=torch.float64)).tolist() == [0.0, 0.0]
