// tree_walk.cuh — the leaf a binned record reaches in one variance tree of a node pool, shared by GBTClassifier's
// margin update (gbt.cu) and GBTRegressor's (regression.cu), so that both walk a tree with the same bin and mask rule.
#pragma once
#include <stdint.h>

namespace b200flow {

// node {feat (< 0: leaf), kind << 16 | bin_thr, left, nid}: a continuous split sends bin <= bin_thr left, a categorical
// split sends the bins of its mask left; the right child is left + 1.  -> pool index of the reached leaf
__device__ __forceinline__ int variance_tree_leaf(const uint8_t* rec, const int4* __restrict__ nodes,
                                                  const unsigned long long* __restrict__ node_mask, int root) {
    int idx = root;
    int4 nd = __ldg(nodes + idx);
    while (nd.x >= 0) {
        const int bin = rec[nd.x];
        const int right = nd.y < 65536 ? (bin > nd.y) : !((node_mask[(int64_t)idx * 4 + (bin >> 6)] >> (bin & 63)) & 1ull);
        idx = nd.z + right;
        nd = __ldg(nodes + idx);
    }
    return idx;
}

}  // namespace b200flow
