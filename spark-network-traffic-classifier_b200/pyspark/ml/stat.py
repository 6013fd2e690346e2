"""Minimal pyspark.ml.stat: MultivariateGaussian, the components of a GaussianMixtureModel."""


class MultivariateGaussian:
    """mean (DenseVector) and cov (DenseMatrix) of one Gaussian distribution."""

    def __init__(self, mean, cov):
        self.mean, self.cov = mean, cov

    def __repr__(self):
        return "MultivariateGaussian(mean=%r, cov=%r)" % (self.mean, self.cov)
