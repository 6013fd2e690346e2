"""Minimal pyspark.ml.stat: MultivariateGaussian, the components of a GaussianMixtureModel, Correlation (Pearson) on
the PCA kernels' centred Gram matrix (b200flow/pca.py, DESIGN.md §5h), and ChiSquareTest, ANOVATest and FValueTest on the
feature-selection kernels (b200flow/selection.py, DESIGN.md §5i)."""


class MultivariateGaussian:
    """mean (DenseVector) and cov (DenseMatrix) of one Gaussian distribution."""

    def __init__(self, mean, cov):
        self.mean, self.cov = mean, cov

    def __repr__(self):
        return "MultivariateGaussian(mean=%r, cov=%r)" % (self.mean, self.cov)


class Correlation:
    @staticmethod
    def corr(dataset, column, method="pearson"):
        """a one-row host-side frame whose field `pearson(<column>)` is the D x D correlation DenseMatrix of a vector
        column; NaN wherever either variance is 0.  The same bits for any number of ranks."""
        from b200flow import dist as bdist
        from b200flow import pca as _pca
        import pandas as pd
        from ..sql import LocalFrame
        from .feature import IllegalArgumentException, _materialize
        from .linalg import DenseMatrix
        if method != "pearson":
            raise IllegalArgumentException("only 'pearson' is built" if method == "spearman" else
                                           "method must be 'pearson', got %r" % (method,))
        if column not in dataset._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % column)
        try:
            r = _pca.pearson(_materialize(dataset, column), group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        return LocalFrame(pd.DataFrame({"%s(%s)" % (method, column): [DenseMatrix(r.shape[0], r.shape[1], r.T.ravel())]}))


def _run_test(fn, dataset, featuresCol, labelCol):
    """(TestResult, D) of one of b200flow.selection's tests on a vector column and a numeric label column."""
    from b200flow import dist as bdist
    from b200flow import selection as _sel
    from .feature import IllegalArgumentException, SparkException, _peek
    for c in (featuresCol, labelCol):
        if c not in dataset._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % c)
    try:
        return fn(_peek(dataset, featuresCol), _peek(dataset, labelCol)[:, 0].contiguous(), group=bdist.group())
    except _sel.TooManyValuesError as e:
        raise SparkException(str(e))
    except ValueError as e:        # includes b200flow's UnsupportedParamError
        raise IllegalArgumentException(str(e))


def _test_frame(res, stat_name, flatten):
    import pandas as pd
    from ..sql import LocalFrame
    from .linalg import DenseVector
    dof = [int(v) for v in res.dof]
    if flatten:
        return LocalFrame(pd.DataFrame({"featureIndex": list(range(len(dof))), "pValue": [float(v) for v in res.p_values],
                                        "degreesOfFreedom": dof, stat_name: [float(v) for v in res.statistics]}))
    return LocalFrame(pd.DataFrame({"pValues": [DenseVector(res.p_values.copy())], "degreesOfFreedom": [dof],
                                    stat_name + "s": [DenseVector(res.statistics.copy())]}))


class ChiSquareTest:
    @staticmethod
    def test(dataset, featuresCol, labelCol, flatten=False):
        """Pearson's independence test of every (categorical) feature against the (categorical) label: one row with
        pValues, degreesOfFreedom and statistics, or one row per feature with flatten=True.  The same bits for any number
        of ranks."""
        from b200flow import selection as _sel
        return _test_frame(_run_test(_sel.chi_square_test, dataset, featuresCol, labelCol), "statistic", flatten)


class ANOVATest:
    @staticmethod
    def test(dataset, featuresCol, labelCol, flatten=False):
        """one-way ANOVA F-test of every continuous feature against the categorical label: pValues, degreesOfFreedom,
        fValues."""
        from b200flow import selection as _sel
        return _test_frame(_run_test(_sel.anova_test, dataset, featuresCol, labelCol), "fValue", flatten)


class FValueTest:
    @staticmethod
    def test(dataset, featuresCol, labelCol, flatten=False):
        """F-test of the regression of the continuous label on every continuous feature: pValues, degreesOfFreedom,
        fValues."""
        from b200flow import selection as _sel
        return _test_frame(_run_test(_sel.f_value_test, dataset, featuresCol, labelCol), "fValue", flatten)
