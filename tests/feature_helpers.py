"""Helpers for the preprocessing tests (tests/test_feature_scaling_gpu.py)."""


def kdd_frame(n, C, seed):
    """a KDD-shaped DataFrame over synthetic raw records, its code columns indexed (`<name>_num`), and its feature names"""
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.feature import StringIndexer
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, C, seed=seed, device="cuda")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    df = Pipeline(stages=[StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]).fit(df).transform(df)
    return df, [c for c in df.columns if c not in cats + ["label", "label_num"]]
