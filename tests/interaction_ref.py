"""NumPy restatement of LightGBM 3.2's interaction constraints (`interaction_constraints`), the rule tree_ref.grow_tree applies with
`constraints`, used to pin the engine's pick step (d_pick_block) and the round controller's leaf set masks tree by tree.

Restated from LightGBM 3.2 (ColSampler::GetByNode, Tree::branch_features, SerialTreeLearner::ComputeBestSplitForFeature); not checked
against the native library:
- `constraints` is a list of sets of real feature indices.  A leaf's branch is the real split features on its path from the root.  A set
  is compatible with the leaf when it holds every branch feature (every set is compatible with the root); the features allowed at the
  leaf are the branch features and the union of the compatible sets (`allowed_by_branch`).
- The scans run as without constraints, for every feature the tree's feature_fraction sample holds: the same is_splittable flag updates
  and the same extra_trees draws.  Only the leaf's best split is taken over the allowed features alone.

The engine keeps one bit mask per leaf instead (`allowed_by_mask`): sets_of[f] has bit s set when set s holds f, the root's mask has
every bit, a split on f gives both children parent & sets_of[f], and f is allowed where sets_of[f] & mask != 0.  tree_ref.grow_tree grows
trees with the masks; test_interaction_reference_cpu.py checks that the two forms agree."""
ALL = (1 << 64) - 1      # the root's mask: every set


def allowed_by_branch(constraints, branch, features):
    """GetByNode's rule: the real indices among `features` allowed at a leaf whose path splits on `branch`"""
    allowed = set(branch)
    for c in constraints:
        if all(f in c for f in branch):
            allowed |= set(c)
    return {f for f in features if f in allowed}


def sets_of(constraints, nf):
    """[nf] per real feature, bit s set when set s holds it"""
    out = [0] * nf
    for s, c in enumerate(constraints):
        for f in c:
            out[f] |= 1 << s
    return out


def allowed_by_mask(sets, mask, features):
    return {f for f in features if sets[f] & mask}


def leaf_paths(t):
    """the split features on every root-to-leaf path of a parsed model tree (modeltext.parse_model)"""
    if t["num_leaves"] <= 1:
        return [[]]
    out = []

    def walk(node, path):
        path = path + [int(t["split_feature"][node])]
        for child in (int(t["left_child"][node]), int(t["right_child"][node])):
            if child < 0:
                out.append(path)
            else:
                walk(child, path)
    walk(0, [])
    return out
