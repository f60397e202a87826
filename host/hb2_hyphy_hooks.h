// hb2_hyphy_hooks.h -- glue between a build copy of HyPhy (veg/hyphy) and libhyphy_b200.so.
//
// The reference has no evaluator plugin interface (SURVEY.md §8b), so the binding is a handful of ONE-LINE insertions
// into a build copy of its sources (host/apply_hooks.py lists them with their anchors) that call the functions below;
// everything else -- the logic of the binding -- lives in hb2_hyphy_hooks.cpp, which is compiled with HyPhy's headers
// and linked against the engine's C ABI (include/hyphy_b200.h).  Nothing here is reference code.
//
//   _LikelihoodFunction::SetupLFCaches   (likefunc.cpp:4163)  -> hb2_hooks::create      one engine partition per tree
//   _LikelihoodFunction::ComputeBlock    (likefunc.cpp:10783) -> hb2_hooks::Scope + hb2_hooks::compute_block
//   _CalcNode::SetCompExp                (calcnode.cpp:714)   -> hb2_hooks::intercept   matrices go to the GPU instead of
//                                                                                       _Matrix::Exponentiate
//                                                                                       (called from the OpenMP loop of
//                                                                                       ExponentiateMatrices, tree.cpp:2995:
//                                                                                       the hand-over is serialised inside)
//   _CalcNode::RecomputeMatrix           (calcnode.cpp:526)   -> hb2_hooks::compiled    formula VALUES go to the GPU instead
//                                                                                       of a numeric rate matrix
//   _LikelihoodFunction::DeleteCaches    (likefunc.cpp:10556) -> hb2_hooks::destroy_all
//   _LikelihoodFunction::ReconstructAncestors (likefunc2.cpp:308) -> hb2_hooks::materialize  device -> host copies for the
//                                                                                       ancestral-state readers
//
// Environment: HYPHY_B200=0 disables the engine (the unmodified CPU path runs); HYPHY_B200_TC=1 selects the tensor-core
// pruning path for 33..64-state partitions (error-compensated 3xTF32: every evaluation is within 1e-6*|lnL| of the
// reference, typically ~1e-9, but that rounding noise is not smooth in the parameters and HyPhy's optimiser differentiates
// the likelihood numerically -- SimpleOptimizations/SmallCodon.bf stops short of the optimum with it -- so
// the DEFAULT under the optimiser is the fp64 kernels, whose noise is ~1e-13); HYPHY_B200_DEVICE=n selects the CUDA device (default: MPI rank modulo visible devices, or 0);
// HYPHY_B200_VERBOSE=1 prints one line per partition created / destroyed with evaluation counts.
#pragma once

class _CalcNode;
class _Matrix;
class _TheTree;
class _SimpleList;
class _DataSetFilter;
class _Vector;

namespace hb2_hooks {

// SetupLFCaches: create the engine partition of tree `index` (state = the likelihood function's opaque slot).
void create(void *&state, unsigned long n_trees, unsigned long index, _TheTree *tree, _DataSetFilter const *filter,
            long const *leaf_flags, _Vector const *ambiguities, long n_ambiguities);
// the partition of tree `index`, or nullptr when the engine does not run it (disabled, 2-sequence / numeric filters)
void *partition(void *state, unsigned long index);
// DeleteCaches
void destroy_all(void *&state);

// ComputeBlock: while a Scope is alive, _CalcNode::SetCompExp calls of nodes of its tree are diverted to the engine.
class Scope {
  public:
    explicit Scope(void *part);
    ~Scope();
    void *part() const { return part_; }
  private:
    void *part_, *prev_;
};

// SetCompExp(m, catID, do_exponentiation): returns the matrix to keep as compExp (a placeholder of the right shape for
// rate matrices, `m` itself for host-computed transition matrices) or nullptr when the call is not diverted.
_Matrix *intercept(_CalcNode *node, _Matrix *m, long catID, bool do_exponentiation, _Matrix *existing);

// _CalcNode::RecomputeMatrix (calcnode.cpp:526), queue mode, ordinary (not explicit-form) models whose rate matrix has been
// compiled (_CompiledMatrixData, matrix.h:69-80): evaluates the model's unique formulas with this node's parameters --
// the first half of _Matrix::EvaluateSimple (matrix.cpp:3112-3133) -- and hands the ~50 VALUES to the engine; the scatter
// into the matrix (matrix.cpp:3135-3321), the multiplication by the equilibrium frequencies and the diagonal
// (MultByFreqs, matrix.cpp:1546) and the exponential all happen on the device.  Returns the matrix the node keeps as
// compExp (shape only, NaN filled), or nullptr when the node takes the dense route (SetCompExp interception).
// HYPHY_B200_DENSE=1 disables this route (A/B).
_Matrix *compiled(_CalcNode *node, _Matrix *model_matrix, long model_index, long catID, _Matrix *existing);
// while alive, SetCompExp is NOT intercepted (the node stores the placeholder the call above returned)
class Bypass {
  public:
    Bypass();
    ~Bypass();
};

// ComputeBlock after DetermineNodesForUpdate + ExponentiateMatrices: pruning, root reduction, scaling correction.
double compute_block(void *part, _TheTree *tree, long catID, _SimpleList const &branches, double *siteRes, long *scc,
                     long branchIndex, _SimpleList *branchValues);

// ReconstructAncestors (likefunc2.cpp:308): joint reconstruction and ancestral sampling read the nodes' transition matrices
// (tree.cpp:4273, :4110) and the internal-node conditionals (tree.cpp:4107, FillInConditionals :3335) on the HOST.  With the
// engine those live on the device: this copies them back once -- P of every branch and class into the matrices the nodes
// keep (the NaN placeholders), the conditionals (normalised per node and pattern: both readers are scale-invariant there)
// into conditionalInternalNodeLikelihoodCaches in the host's cache order.
void materialize(void *part, _TheTree *tree, _DataSetFilter const *filter, double *inode_cache, _SimpleList const *site_ordering);
// _TheTree::RecoverNodeSupportStates (tree.cpp:2515; ConstructCategoryMatrix on a tree linked to a likelihood function,
// batchlanruntime.cpp:1198) reads the transition matrices knowing only the tree: same copy-back, matrices only.  (Untested:
// that HBL path segfaults in the unmodified reference at this commit.)
void materialize_tree(_TheTree *tree);

}  // namespace hb2_hooks
