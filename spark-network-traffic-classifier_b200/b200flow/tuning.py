"""Model selection over numTrees x maxDepth from one forest fit per fit group (DESIGN.md §5a).

Every random draw of a fit is keyed independently of numTrees and maxDepth (bagging by (seed, row, tree), the findSplits
sample by (seed, row), feature subsets by (seed, tree, nid); featureSubsetStrategy="auto" is "sqrt" for every T > 1), and
a node's split does not depend on how deep the tree may grow.  So for fixed other params and T >= 2, the forest fitted with
(T, d) is the first T trees of the (T_max, d_max) forest cut at depth d, and one fit plus one
ForestModel.grid_confusion pass scores a whole numTrees x maxDepth grid.  Pure Python: no device work here.
"""

_CUT_PARAMS = ("numTrees", "maxDepth")


def _key(values):
    return tuple(sorted((k, repr(v)) for k, v in values.items() if k not in _CUT_PARAMS))


def fit_groups(param_maps, decision_tree=False):
    """partition resolved param maps (dicts name -> value, each holding maxDepth, and numTrees unless decision_tree) into fit
    groups: -> [(T_max, d_max, [(map index, T, d), ...])], groups in order of their first map, members in map order.

    The group key is every param other than numTrees / maxDepth.  A RandomForest point with numTrees == 1 is a group of its
    own (it has no bagging and "auto" becomes "all", so it is not a prefix of a larger forest); DecisionTree points group over
    maxDepth alone (T = 1)."""
    groups, order = {}, []
    for i, values in enumerate(param_maps):
        d = int(values["maxDepth"])
        T = 1 if decision_tree else int(values["numTrees"])
        key = _key(values)
        if not decision_tree and T == 1:
            key = ("numTrees == 1", i)
        if key not in groups:
            groups[key] = []
            order.append(key)
        groups[key].append((i, T, d))
    return [(max(m[1] for m in groups[k]), max(m[2] for m in groups[k]), groups[k]) for k in order]
