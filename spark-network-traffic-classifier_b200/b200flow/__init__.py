"""b200flow — Python host layer over libb200flow.so (hand-written sm_90a kernels, include/b200flow.h).

Only the hot path of biagiom/spark-network-traffic-classifier lives here: fused encode
(StringIndexer + OneHotEncoder + StandardScaler + VectorAssembler) and the RandomForest /
DecisionTree trainer + batch predictor.  The pyspark.ml-shaped API the reference scripts call is in
the sibling `pyspark` package.  No CPU fallback: the CUDA library must be built and a GPU present.
"""
from ._lib import B200FlowError, EXPORTS, LIB_PATH, load  # noqa: F401
