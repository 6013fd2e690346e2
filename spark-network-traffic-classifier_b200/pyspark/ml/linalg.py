"""Minimal pyspark.ml.linalg: DenseVector / Vectors for host-side inspection of vector columns."""
import numpy as np


class DenseVector:
    def __init__(self, values):
        self.values = np.asarray(values, np.float64)

    def toArray(self):
        return self.values

    def __len__(self):
        return len(self.values)

    def __getitem__(self, i):
        return float(self.values[i])

    def __eq__(self, o):
        return isinstance(o, DenseVector) and np.array_equal(self.values, o.values)

    def __repr__(self):
        return "DenseVector([%s])" % ", ".join(repr(float(v)) for v in self.values)


class Vectors:
    @staticmethod
    def dense(*v):
        return DenseVector(v[0] if len(v) == 1 and hasattr(v[0], "__len__") else v)


class DenseMatrix:
    """numRows x numCols matrix with column-major values, as Spark stores it."""

    def __init__(self, numRows, numCols, values):
        self.numRows, self.numCols = int(numRows), int(numCols)
        self.values = np.asarray(values, np.float64).reshape(-1)
        if self.values.shape[0] != self.numRows * self.numCols:
            raise ValueError("DenseMatrix %dx%d needs %d values, got %d" % (self.numRows, self.numCols,
                                                                           self.numRows * self.numCols, self.values.shape[0]))

    def toArray(self):
        return self.values.reshape(self.numCols, self.numRows).T.copy()

    def __eq__(self, o):
        return isinstance(o, DenseMatrix) and (self.numRows, self.numCols) == (o.numRows, o.numCols) and \
            np.array_equal(self.values, o.values)

    def __repr__(self):
        return "DenseMatrix(%d, %d, [%s], False)" % (self.numRows, self.numCols, ", ".join(repr(float(v)) for v in self.values))


class Matrices:
    @staticmethod
    def dense(numRows, numCols, values):
        return DenseMatrix(numRows, numCols, values)
