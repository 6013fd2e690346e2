"""Minimal pyspark.ml.stat: MultivariateGaussian, the components of a GaussianMixtureModel, and Correlation (Pearson) on
the PCA kernels' centred Gram matrix (b200flow/pca.py, DESIGN.md §5h)."""


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
