/*
 * hyphy_b200.h -- C ABI of the GPU-native (H100, sm_90a) phylogenetic-likelihood engine (libhyphy_b200.so).
 *
 * This is the drop-in boundary behind the reference's `_LikelihoodFunction::ComputeBlock`
 * (veg/hyphy src/core/likefunc.cpp:10783-11289).  The reference has no plugin interface for its evaluator; the
 * only precedent is the dormant `#ifdef MDSOCL` trio (construct in SetupLFCaches likefunc.cpp:4182-4184, init
 * :4313-4316, destroy :10546-10551).  The entry points below are what a maintainer binds at those three places
 * (INTEGRATION.md shows the patch).  Plain pointers and sizes only; no C++/torch types cross this line.
 *
 * Conventions (all follow the reference so host arrays can be passed unmodified):
 *   - nodes: 0..L-1 leaves in post-order, L..L+I-1 internal nodes in post-order, root = L+I-1;
 *     flatParents[node] = parent's INTERNAL index (0..I-1), root = -1        (tree.cpp:722-766, tree.h:336)
 *   - leafState[l*S + s]: original pattern order; >=0 state index, <0 -> ambiguity row -(code+1)
 *                                                                            (likefunc.cpp:4265-4308)
 *   - matrices: D*D row-major doubles, row = parent(from) state, column = child(to) state
 *                                                                            (tree_evaluator.cpp:232,3674)
 *   - per-pattern results use the reference's scaler convention L_true = L * 2^(-64*count)
 *                                                                            (likefunc2.cpp:828-859,1484-1506)
 *   - errors: every call returns 0 on success, nonzero on failure (hb2_last_error() has the text).  There is NO
 *     CPU fallback: a missing GPU makes hb2_create fail and the host must treat that as fatal
 *     (HandleApplicationError, global_things.cpp:787).  Numerical failures are value-encoded exactly like
 *     tree_evaluator.cpp:4094-4148: lnL = -inf when a pattern has likelihood <= 0, NaN is propagated.
 *   - threading: one host thread per partition handle at a time (ComputeBlock is entered from the single
 *     interpreter thread; OpenMP lives inside it).  Calls block until the result is on the host.
 */
#ifndef HYPHY_B200_H
#define HYPHY_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HB2_ABI_VERSION 1

typedef struct hb2_partition hb2_partition;   /* opaque: one per (likelihood function, partition) */

/* hb2_create flags */
#define HB2_FLAG_DEFAULT        0
#define HB2_FLAG_FORCE_FP64     1   /* always use the fp64 pruning kernels (parity reference), never the tensor path */

/* matrix kinds for hb2_set_matrices */
#define HB2_MATRIX_RATE   0   /* numeric rate matrix Q*t after MultByFreqs: engine exponentiates on device
                                 (replaces _Matrix::Exponentiate matrix.cpp:5537 / ExponentiateMatrices tree.cpp:2932) */
#define HB2_MATRIX_TRANS  1   /* transition matrix P already exponentiated by the host (GetCompExp()->theData) */

int         hb2_abi_version(void);
const char *hb2_last_error(void);              /* thread-local text of the last failure */
int         hb2_device_count(void);            /* number of visible CUDA devices (0 => hb2_create will fail) */

/* Replaces the allocation half of _LikelihoodFunction::SetupLFCaches (likefunc.cpp:4163-4319) for one partition.
 * S patterns, D states, L leaves, I internal nodes, C rate classes (categoryCount, >=1).
 * ambig: nAmb*D doubles of 0/1 (dataset_filter.cpp:1594-1632); patternFreq: theFilter->theFrequencies.
 * All host arrays are copied; the caller keeps ownership.  device = CUDA ordinal. */
int hb2_create(hb2_partition **out, int64_t S, int64_t D, int64_t L, int64_t I, int64_t C,
               const int64_t *flatParents, const int64_t *leafState, const double *ambig, int64_t nAmb,
               const int64_t *patternFreq, int device, int flags);

/* Replaces ExponentiateMatrices (tree.cpp:2932-3113) + _CalcNode::SetCompExp (calcnode.cpp:714): hands the engine
 * the matrices of the nodes in `*matrices` (DetermineNodesForUpdate, tree.cpp:3117) for rate class `cat`
 * (0..C-1; -1 is accepted as 0 for partitions without category variables, likefunc.cpp:10843).
 * nodeIds[k] in 0..L+I-2; M[k] -> D*D doubles.  kind = HB2_MATRIX_RATE | HB2_MATRIX_TRANS.
 * Every hand-over (hb2_set_matrices*, hb2_set_mixture_matrices) checks its whole list first: a refused call (bad class,
 * node id, kind or matrix pointer anywhere in the list) changes nothing -- no slot, no pending matrix, no branch cache. */
int hb2_set_matrices(hb2_partition *p, int64_t cat, int64_t n, const int64_t *nodeIds,
                     const double *const *M, int kind);
/* same, matrices packed back to back (n*D*D doubles) */
int hb2_set_matrices_packed(hb2_partition *p, int64_t cat, int64_t n, const int64_t *nodeIds,
                            const double *M, int kind);

/* Compact hand-over of rate matrices (removes the 8*D*D bytes per matrix of H2D traffic and lets the device do
 * what _Matrix::EvaluateSimple's scatter (matrix.cpp:3094-3321) and MultByFreqs (matrix.cpp:1546-1677) do on the host).
 * The reference compiles a model matrix into _CompiledMatrixData (include/matrix.h:69-80): a list of unique formulas
 * (formulasToEval), per-evaluation numeric formulaValues[], and formulaRefs[] mapping every stored off-diagonal entry
 * to its formula.  hb2_set_rate_template takes that static part once per model:
 *   entryIndex[e]   = row*D + col of stored entry e (theIndex), off-diagonal
 *   entryFormula[e] = formulaRefs[e] in [0, nFormulas)
 *   colFreq         = nullable D doubles: entry (r,c) is multiplied by colFreq[c] (MultByFreqs; NULL when the model
 *                     was declared with the "do not multiply by frequencies" flag)
 * hb2_set_matrices_compiled then hands over, per evaluation, only formulaValues (n * nFormulas doubles, one row per
 * listed node); the engine scatters them, applies colFreq, sets diagonal = -(row sum) and exponentiates. */
int hb2_set_rate_template(hb2_partition *p, int64_t nnz, const int64_t *entryIndex, const int64_t *entryFormula,
                          int64_t nFormulas, const double *colFreq);
int hb2_set_matrices_compiled(hb2_partition *p, int64_t cat, int64_t n, const int64_t *nodeIds,
                              const double *formulaValues);
/* Several models on one tree (foreground / background branches of RELAX and BUSTED, per-branch models of aBSREL; every
 * _CalcNode carries its own model index, calcnode.h): one template per model matrix, ids 0..HB2_MAX_TEMPLATES-1; the two
 * calls above are the id-0 forms.  hb2_set_template_frequencies replaces colFreq when the model's equilibrium
 * frequencies are themselves being estimated (cheap: D doubles, no reallocation). */
#define HB2_MAX_TEMPLATES 16
int hb2_set_rate_template_id(hb2_partition *p, int64_t templateId, int64_t nnz, const int64_t *entryIndex,
                             const int64_t *entryFormula, int64_t nFormulas, const double *colFreq);
int hb2_set_matrices_compiled_id(hb2_partition *p, int64_t templateId, int64_t cat, int64_t n, const int64_t *nodeIds,
                                 const double *formulaValues);
int hb2_set_template_frequencies(hb2_partition *p, int64_t templateId, const double *colFreq);

/* Explicit-form mixtures P = sum_k w_k Exp(Q_k) per branch (BS-REL; tree.cpp:3047-3089):
 * K components for each listed node, M packed [n][K][D*D], w packed [n][K].  Asynchronous like the other hand-overs
 * (two kernel launches on the partition's stream, no host synchronisation); M and w are copied before the call returns. */
int hb2_set_mixture_matrices(hb2_partition *p, int64_t cat, int64_t n, const int64_t *nodeIds, int64_t K,
                             const double *M, const double *w);

/* Replaces likefunc.cpp:10978-11123 (+ ComputeTreeBlockByBranch tree_evaluator.cpp:3556-4171) for ONE rate class:
 * prunes the nodes in updateNodes (nUpdate < 0 or updateNodes == NULL => all nodes) and reduces at the root.
 *   lnL            : sum_s f_s log L_s, already scale-corrected (what ComputeBlock returns at likefunc.cpp:11259)
 *   siteL/siteScale: nullable; per-pattern (original order) L and count with L_true = L*2^(-64*count)
 *                    (the storageVec / siteCorrectionCounts outputs, tree_evaluator.cpp:4080-4092, :84-87) */
int hb2_evaluate(hb2_partition *p, int64_t cat, int64_t nUpdate, const int64_t *updateNodes,
                 const double *rootFreqs, double *lnL, double *siteL, int64_t *siteScale);

/* hb2_evaluate with ONE node pinned to a per-pattern state -- the reference's `branchIndex` / `branchValues` arguments of
 * ComputeBlock (likefunc.cpp:10783), i.e. setBranch / setBranchTo of ComputeTreeBlockByBranch (tree_evaluator.cpp:3624:
 * a pinned leaf has its observed state replaced :173-181, a pinned internal node starts from the indicator vector of its
 * state :585-605, a pinned root contributes only that state :4059-4063).  forcedNode is a FLAT node id (0..L-1 leaves,
 * L..L+I-1 internal nodes; the reference's branchIndex b maps to b + L for b < I and to b - I otherwise), forcedStates[S]
 * in original pattern order, each in 0..D-1.  The caller lists the pinned node (a leaf) or its children (an internal
 * node) in updateNodes exactly as DetermineNodesForUpdate does with `addOne` (tree.cpp:3117,3262), and schedules the
 * recomputation of the affected conditionals afterwards (AddBranchToForcedRecomputeList, likefunc2.cpp:979-1041).
 * Everything PopulateConditionalProbabilities builds on per-class ComputeBlock calls -- ConstructCategoryMatrix run
 * modes, HMM / constant-on-partition categories, ancestral sampling -- only needs this entry point. */
int hb2_evaluate_forced(hb2_partition *p, int64_t cat, int64_t nUpdate, const int64_t *updateNodes,
                        const double *rootFreqs, int64_t forcedNode, const int64_t *forcedStates,
                        double *lnL, double *siteL, int64_t *siteScale);

/* Fused replacement for the whole category loop PopulateConditionalProbabilities(WeightedSum) +
 * SumUpSiteLikelihoods (likefunc2.cpp:484-908, 1446-1506): all C classes pruned in one pass,
 * L_s = sum_c weights[c]*L_{c,s} combined on device, one lnL comes back.  Same outputs as hb2_evaluate.  A class of
 * weight 0 is ignored, as likefunc2.cpp:668 (its likelihoods, NaN included, do not reach the sum); a tiny or subnormal
 * weight on a class far above the others does not hide them.  Negative weights are not supported. */
int hb2_evaluate_classes(hb2_partition *p, const double *weights, int64_t nUpdate, const int64_t *updateNodes,
                         const double *rootFreqs, double *lnL, double *siteL, int64_t *siteScale);

/* Single-branch shortcut (SURVEY 8f row 1; ComputeBranchCache tree_evaluator.cpp:4286-4845 and ComputeLLWithBranchCache
 * tree.cpp:3383-3934, entered from ComputeBlock likefunc.cpp:10984-10993 / :11170-11177).  After a regular evaluation,
 * hb2_branch_cache_build(node) collects, for every owned class and pattern, the likelihood of everything outside the
 * subtree of `node` as seen from the parent end of its branch (the reference's branchCaches[.][1]; the subtree side is
 * the resident conditional).  While only THAT branch's matrix changes (set it with hb2_set_matrices*),
 * hb2_branch_cache_evaluate returns lnL in O(S*D^2) without touching the tree; cat/weights as in hb2_evaluate /
 * hb2_evaluate_classes (weights != NULL selects the all-class form).  Any regular evaluation invalidates the cache; a
 * pending matrix of another node makes the call fail.  Unlike the reference this needs no reversible model: the outside
 * vectors are propagated through transposed transition matrices instead of re-rooting the tree. */
int hb2_branch_cache_build(hb2_partition *p, int64_t node, const double *rootFreqs);
int hb2_branch_cache_evaluate(hb2_partition *p, int64_t cat, const double *weights, double *lnL, double *siteL,
                              int64_t *siteScale);

/* Batched one-pattern likelihoods on the partition's tree (SURVEY 8f row 3).  The site phases of FEL and MEME
 * (res/TemplateBatchFiles/SelectionAnalyses/FEL.bf:1180-1233, MEME.bf:699-746) fit thousands of independent likelihood
 * functions that all use ONE site pattern of the alignment, the same tree, and differ only in a few per-site parameters
 * (alpha, beta, ...); the reference farms them out one by one (mpi.QueueJob).  Here `nSets` such problems are evaluated in
 * one call: set s prunes pattern patternOf[s] of the partition with ITS OWN matrices for every branch, handed over in the
 * compiled form of template `templateId`: formulaValues[s][b][nFormulas], b = 0..B-1 (one rate class per set).
 * branchGroup (nullable, B entries in 0..7) tells the engine which branches of a set share one rate matrix up to a scalar
 * (FEL: tested vs background branches); it is a hint for the shared-powers exponential, proportionality is still checked.
 * siteLnL[s] = log-likelihood of the pattern under set s (NOT multiplied by the pattern's frequency).  fp64 throughout;
 * the partition's resident caches are not touched.  33..64 states only. */
int hb2_batch_site_likelihoods(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf,
                               const double *formulaValues, const int64_t *branchGroup, const double *rootFreqs,
                               double *siteLnL);

/* The same with explicit-form mixtures on the branches (MEME's site model, MEME.bf:381-386 and :656-680): branch b of a
 * set has branchK[b] components (branchK nullable, B entries in 1..K; NULL = K on every branch; K in 1..4) and its
 * transition matrix is sum_k w_k Exp(Q_k), components added in order k = 0..branchK[b]-1.  With R = sum_b branchK[b]
 * component rows per set, in branch order with the components of one branch consecutive:
 *   formulaValues [nSets][R][nFormulas]  (compiled form of template `templateId`, one template for every row)
 *   weights       [nSets][R]             (not normalised or checked; a plain branch is one component of weight 1.0)
 * The shared-powers group of a row is (set, branchGroup[b], k): component k of the tested branches is one rate matrix up
 * to the branch length.  Everything else as hb2_batch_site_likelihoods; a pattern of likelihood 0 gives -inf, a NaN
 * weight NaN for its set only. */
int hb2_batch_site_mixture_likelihoods(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf,
                                       int64_t K, const int64_t *branchK, const double *formulaValues,
                                       const double *weights, const int64_t *branchGroup, const double *rootFreqs,
                                       double *siteLnL);

/* Branch-level empirical Bayes for MEME (meme.compute_branch_EBF, MEME.bf:886-944, called for every tested branch of a
 * site whose fitted beta+ > alpha with a positive weight above 1e-6, :1415-1431): the site's likelihood with each branch
 * pinned to each of its mixture components, for every set in one call.  Arguments as hb2_batch_site_mixture_likelihoods
 * (R = sum_b branchK[b] rows per set, in branch order with the components of one branch consecutive), plus:
 *   rowLnL   [nSets][R]: row r = component k of branch b is the log-likelihood of pattern patternOf[s] under set s with
 *            branch b's transition matrix replaced by that row's exponential alone, Exp(Q_{s,r}) with weight 1, and every
 *            other branch keeping its mixture sum_k w_k Exp(Q_k) as the batch pruning forms it.  NOT multiplied by the
 *            pattern frequency; it does not depend on branch b's own weights (a component of weight 0 still gets its
 *            pinned value); a branch with one component gives the set's own likelihood up to rounding.
 *   siteLnL  nullable [nSets]: the set's mixed log-likelihood, bit for bit what hb2_batch_site_mixture_likelihoods
 *            returns for the same arguments (the same inside pass).
 * MEME's posteriors are post_{b,k} = w_{s,r} exp(rowLnL[s][r] - siteLnL[s]) and the EBF of branch b is its positive
 * component's posterior odds over its prior odds, (post / (1 - post)) / (w / (1 - w)).  The weights are neither normalised
 * nor checked: the host maps MEME's stick-breaking mixture_aux_weight parameters to plain weights.  All values come from
 * one inside and one outside (pre-order) pass per set, fp64, every vector renormalised by exact powers of two; a row of
 * likelihood 0 gives -inf, and a NaN weight gives NaN for its set only.
 * Refusals before anything is launched or written (the partition stays usable): everything
 * hb2_batch_site_mixture_likelihoods refuses; weights == NULL (with one row per branch every row would equal siteLnL);
 * rowLnL == NULL.  nSets == 0 after these checks does nothing.  33..64 states only; not available in class-group mode.
 * Nothing an evaluation reads is touched: conditionals, scalers, walk plans and tags, the branch cache, the staged root
 * vector, the P cache and the resident rate matrices. */
int hb2_batch_branch_component_likelihoods(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf,
                                           int64_t K, const int64_t *branchK, const double *formulaValues,
                                           const double *weights, const int64_t *branchGroup, const double *rootFreqs,
                                           double *siteLnL, double *rowLnL);

/* Leaf state imputation for MEME and PRIME (--impute-states, MEME.bf:1382-1412, PRIME.bf:940-960): what
 * ReconstructAncestors(lf_site, {{0}}, MARGINAL, DOLEAVES) reports for every leaf of a site, for every set in one call.
 * The reference evaluates the site with leaf l forced to each state k (setBranchTo replaces the leaf's observation, so its
 * state or ambiguity is not used, tree_evaluator.cpp:173-181), divides by the site likelihood and normalises over k
 * (_LikelihoodFunction::RecoverAncestralSequencesMarginal, likefunc2.cpp:974-1006 and :1083-1093): the row of leaf l is the
 * predictive distribution of l's state given every other leaf, not the posterior given all the data.
 * Sets as hb2_batch_column_likelihoods, on partition patterns: weights == NULL gives one row per branch, formulaValues
 * [nSets][B][nFormulas] as hb2_batch_site_likelihoods (K must be 1 and branchK NULL; PRIME's and FEL's site models);
 * otherwise rows, weights, K and branchK as hb2_batch_site_mixture_likelihoods (MEME's lf_bsrel).  Outputs:
 *   support  [nSets][L][D]: support[s][l][k] = u[k] / sum_j u[j] with u[k] = sum_p A_l[p] P_l[p][k], A_l the vector at the
 *            parent end of leaf l's branch of everything outside l (the batch outside pass of
 *            hb2_batch_branch_component_likelihoods) and P_l l's transition matrix, mixed as the batch pruning mixes it.
 *            Flat leaf ids, states 0..D-1 (not padded).  A leaf's row does not depend on that leaf's own code; rows sum
 *            to 1 up to rounding; a row whose total sum_j u[j] is 0 or not finite is NaN in every entry (the reference
 *            gives NaN there too, likefunc2.cpp:1084-1086).
 *   siteLnL  nullable [nSets]: bit for bit what hb2_batch_site_likelihoods (weights == NULL) or
 *            hb2_batch_site_mixture_likelihoods returns for the same arguments (the same inside pass).
 * Plain sets give, bit for bit, the support of the mixture layout with one component of weight 1.0 per branch.  A NaN
 * weight or formula value gives NaN for its own set only.  fp64 throughout, every outside vector renormalised by exact
 * powers of two.
 * Refusals before anything is launched or written (the partition stays usable): everything the corresponding likelihood
 * entry point refuses; support == NULL; K != 1 or a non-NULL branchK without weights.  nSets == 0 after these checks does
 * nothing.  33..64 states only; not available in class-group mode.
 * Nothing an evaluation reads is touched: conditionals, scalers, walk plans and tags, the branch cache, the staged root
 * vector, the P cache and the resident rate matrices. */
int hb2_batch_leaf_support(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf,
                           int64_t K, const int64_t *branchK, const double *formulaValues, const double *weights,
                           const int64_t *branchGroup, const double *rootFreqs, double *siteLnL, double *support);

/* Joint maximum-likelihood ancestral states for FEL's, MEME's and PRIME's per-site reconstruction (ancestral.build(lf, 0,
 * FALSE) at every site, FEL.bf:798-801, MEME.bf:1359-1363, PRIME.bf:975 and :1013): what ReconstructAncestors(lf, {{0}})
 * reports for the internal nodes of a site, for every set in one call.  The reference's procedure is Pupko's max-product
 * recursion (_LikelihoodFunction::ReconstructAncestors, likefunc2.cpp:309-480; _TheTree::RecoverAncestralSequences,
 * tree.cpp:4209-4510) without category variables, every branch under its one transition matrix (an explicit-form
 * mixture's mixed matrix):
 *   children in increasing flat id, each parent vector starting at 1 (:4253, :4266-4271); a resolved leaf in state a
 *   multiplies it by P[p][a] (:4315-4327); an ambiguous leaf or internal child with vector x (its 0/1 row, or the child's
 *   joint vector) multiplies it by max_c P[p][c] x[c], the scan over ascending c by strict > against a running maximum
 *   that starts at 0 with index 0, so ties go to the lowest c and a row with no positive product gives 0 with index 0
 *   (:4357-4377); an unresolved child -- a leaf whose row is 1 in all D states, or an internal node all of whose children
 *   are unresolved -- takes state -1 and does not multiply its parent (:4350-4356, :4390-4394); the root state is argmax_c
 *   pi_c J_root[c] by the same rule, -1 when the root is unresolved (:4448-4457, :4484-4486); traceback takes each internal
 *   node's argument at its parent's state, -1 below a -1 (:4458-4470).  The reference's unresolved test compares values
 *   with 1.0; the engine's is structural, which agrees except when a resolved subtree's vector is exactly 1 in all D
 *   states (DESIGN §4.13).
 * Sets as hb2_batch_leaf_support, on partition patterns: weights == NULL gives one row per branch (K must be 1 and branchK
 * NULL; FEL's and PRIME's site models), otherwise MEME's mixture rows.  Outputs:
 *   nodeStates [nSets][I]: entry i is internal node i (root at I-1, as hb2_batch_site_simulate's nodeStates): a state
 *              0..D-1, or -1 for an unresolved node.
 *   jointLnL   nullable [nSets]: log(pi_r J_root[r]) at the returned root state r; -inf for a product of 0, 0.0 for a fully
 *              unresolved column, NaN for a set whose recursion multiplied or compared a NaN (its states are still those
 *              the comparisons give).
 *   siteLnL    nullable [nSets]: bit for bit what hb2_batch_site_likelihoods (weights == NULL) or
 *              hb2_batch_site_mixture_likelihoods returns for the same arguments; its inside pass runs only when given.
 * Plain sets give, bit for bit, the states and jointLnL of the mixture layout with one component of weight 1.0 per branch.
 * A NaN weight or formula value affects its own set only.  fp64 throughout, every joint vector renormalised by exact
 * powers of two (which changes no comparison).
 * Refusals before anything is launched or written (the partition stays usable): everything the corresponding likelihood
 * entry point refuses; nodeStates == NULL; K != 1 or a non-NULL branchK without weights.  nSets == 0 after these checks
 * does nothing.  33..64 states only; not available in class-group mode.
 * Nothing an evaluation reads is touched: conditionals, scalers, walk plans and tags, the branch cache, the staged root
 * vector, the P cache and the resident rate matrices. */
int hb2_batch_joint_ancestors(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf,
                              int64_t K, const int64_t *branchK, const double *formulaValues, const double *weights,
                              const int64_t *branchGroup, const double *rootFreqs,
                              double *siteLnL, double *jointLnL, int64_t *nodeStates);

/* The batch likelihoods of caller-given columns instead of partition patterns (the refits of a parametric bootstrap score
 * columns simulated by hb2_batch_site_simulate, which are not patterns of the partition): set s scores
 * columns[s][0..L-1], in hb2_create's leafState codes (>= 0: a state < D; < 0: ambiguity row -(code+1) < nAmb).
 * weights == NULL: one row per branch, formulaValues [nSets][B][nFormulas] as hb2_batch_site_likelihoods (K must be 1 and
 * branchK NULL); otherwise rows, weights, K and branchK as hb2_batch_site_mixture_likelihoods.  A code out of range is
 * refused on the host with its set and leaf, and nothing is written.  Everything else, outputs included, as
 * hb2_batch_site_mixture_likelihoods: a column that equals pattern q gives exactly what patternOf = q gives. */
int hb2_batch_column_likelihoods(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *columns,
                                 int64_t K, const int64_t *branchK, const double *formulaValues, const double *weights,
                                 const int64_t *branchGroup, const double *rootFreqs, double *siteLnL);

/* Batched one-pattern likelihoods at site-specific relative rates, for nucleotide and protein partitions (2..32 states).
 * LEISR (res/TemplateBatchFiles/LEISR.bf:209-266, :271-290, :420-444) and ProteinAnalyses/relative_prot_rates.bf
 * (:160-192, :286) fit the alignment-wide model once, then one one-site likelihood function per pattern whose only free
 * parameter scales every branch length; a constant site is evaluated at rate 0 (LEISR.bf:411-416).  Set s is the
 * log-likelihood of pattern patternOf[s] under class `cat` (-1 means 0) of the partition's current model with every
 * branch's rate matrix multiplied by rates[s]:  P_b(s) = exp(rates[s] * A_b), A_b the rate matrix last handed over for
 * (cat, b) by hb2_set_matrices* with HB2_MATRIX_RATE or by hb2_set_matrices_compiled* (pending hand-overs are flushed
 * first, as by hb2_read_transition).  Only patternOf and rates cross to the device.
 *   rootFreqs  D values, one root vector for every set.
 *   siteLnL    [nSets], NOT multiplied by the pattern frequency; a pattern of likelihood 0 gives -inf.  fp64 throughout.
 * rates[s] == 0 gives identity matrices exactly (a constant column: log pi_state; any other: -inf).  A product
 * rates[s] * ||A_b|| beyond the exponential's range (scaling shift > 900) gives NaN for that set only.
 * Refusals before anything is launched or written (the partition stays usable): null pointers; nSets < 0; cat out of
 * range; patternOf out of range or a rate that is negative, NaN or infinite (both name the set); class-group mode;
 * 33..64 states (use hb2_batch_site_likelihoods with formula values multiplied by the rate: codon rows are linear in
 * them); a branch of `cat` without a resident rate matrix -- its last hand-over a transition matrix or a mixture, or
 * none -- named with its class.  Nothing an evaluation reads is touched: conditionals, scalers, walk plans and tags, the
 * branch cache, the staged root vector, the P cache and the resident rate matrices. */
int hb2_batch_site_rates(hb2_partition *p, int64_t cat, int64_t nSets, const int64_t *patternOf, const double *rates,
                         const double *rootFreqs, double *siteLnL);

/* FillInConditionals-style read-back (tree.cpp:3335): conditionals of internal node `inode` (0..I-1), class cat,
 * as S*D doubles (original pattern order) and S binary exponents: true value = cond * 2^exp2. */
int hb2_read_conditionals(hb2_partition *p, int64_t cat, int64_t inode, double *cond, int32_t *exp2);

/* Read back the transition matrix currently cached for (cat, node): D*D doubles, row = parent state. */
int hb2_read_transition(hb2_partition *p, int64_t cat, int64_t node, double *P);

/* Simulated alignment columns from the partition's current transition matrices (SimulateDataSet, likefunc.cpp:12584,
 * discrete-category mode: every site draws one rate class and evolves down the tree with that class's matrices).  Site i
 * of the call is global site g = firstSite + i of the stream `seed`, so a replicate may be produced in any number of calls.
 *   weights    C class weights, not necessarily normalised; NULL only when C == 1.  A class of weight 0 is never drawn and
 *              its matrices need not exist.
 *   rootFreqs  D root-state weights.
 *   leafStates [L][nSites]: leafStates[l*nSites + i], hb2_create's leafState layout (a block can be handed to hb2_create as
 *              nSites patterns of frequency 1).
 *   nodeStates nullable [I][nSites]: internal-node states, root at I-1 (the reference's storeIntermediates).
 *   siteClass  nullable [nSites]: the drawn class of every site.
 * The matrices are those hb2_read_transition returns (pending hand-overs are flushed first): dense, compiled and mixture
 * hand-overs alike, on every kernel family.
 * The stream (results depend on matrices, weights, rootFreqs, seed and g only -- not on chunking or launch shape):
 *   - one Philox4x32-10 call per draw: counter = (lo32(g), hi32(g), slot, 0), key = (lo32(seed), hi32(seed));
 *   - slot n in 0..L+I-2: flat node n's state drawn from its parent's row; slot L+I-1: the root state; slot L+I: the class;
 *   - uniform u = (x0 * 2^21 + (x1 >> 11)) * 2^-53 from the first two output words.
 * The draw rule for a weight vector v[0..m-1] (a matrix row: row = parent state, columns 0..D-1):
 *   - entries that are not > 0 (negative, zero, NaN) count as 0;
 *   - c_j = sequential fp64 prefix sum over j = 0..m-1, T = c_{m-1};
 *   - the result is the smallest j with fl(u*T) < c_j, or, when there is none, the largest j with v_j > 0.
 * Refusals (a refused call writes no output): nSites < 0; firstSite < 0; negative or NaN weights or rootFreqs, or a total
 * that is not finite and > 0; NULL weights with C > 1; a class of positive weight with a branch that never received a
 * matrix; a matrix row of such a class whose total is not finite and > 0 (checked on the device, reported with class,
 * node and row); class-group mode (hb2_comm_class_groups: a rank does not hold the other groups' matrices).  Pattern-sharded
 * ranks simulate from their own copy of the matrices.  nSites == 0 after these checks does nothing.
 * Nothing an evaluation reads is touched: conditionals, scalers, walk plans and tags, the branch cache, the root vector. */
int hb2_simulate(hb2_partition *p, const double *weights, const double *rootFreqs, int64_t nSites, uint64_t seed,
                 int64_t firstSite, int64_t *leafStates, int64_t *nodeStates, int32_t *siteClass);

/* Site-level parametric bootstrap (FEL.bf:803-818, MEME.bf:1445-1458, --resample N): nReps replicate columns simulated
 * from EACH set's own model (SimulateDataSet on the one-site likelihood function).  Sets have the layout of the batch
 * entry points: weights == NULL: one row per branch, formulaValues [nSets][B][nFormulas], K must be 1 and branchK NULL;
 * otherwise rows, weights, K, branchK as hb2_batch_site_mixture_likelihoods.  branchGroup is the same shared-powers hint.
 * The matrix simulated from is the one the likelihood entry points use for the set: entry (k, j) of a mixture branch is
 * e = w_0 P_0[k][j], then e = fma(w_c, P_c[k][j], e) for c = 1..n-1 (the order of the batch pruning and of
 * hb2_set_mixture_matrices), exponentials from the same batched pipeline.
 *   rootFreqs  D root-state weights, one vector for every set.
 *   leafStates [nSets][nReps][L]: leaf states 0..D-1, column by column -- directly the `columns` of
 *              hb2_batch_column_likelihoods for nSets*nReps sets.
 *   nodeStates nullable [nSets][nReps][I]: internal-node states, root at I-1.
 * The stream is hb2_simulate's with the set in the fourth counter word: one Philox4x32-10 call per draw on counter
 * (lo32(g), hi32(g), slot, t), key (lo32(seed), hi32(seed)), g = firstRep + r for replicate r, t = firstSet + s for set s
 * of the call; slot n < L+I-1 is flat node n's state, slot L+I-1 the root (no class slot: a set has one model); uniform and
 * draw rule as hb2_simulate.  Results depend only on the set's matrices, rootFreqs, seed, t and g: splitting sets or
 * replicates across calls or chunks changes nothing, and set t = 0 draws exactly hb2_simulate's stream.
 * Refusals before anything runs (nothing is written): everything hb2_batch_site_mixture_likelihoods refuses; nSets < 0 or
 * nReps < 0; firstRep < 0 or firstRep > INT64_MAX - nReps; firstSet < 0 or firstSet + nSets > 2^32; root frequencies
 * refused by hb2_simulate's rule.  A set whose matrix has a row whose total is not finite and > 0 (NaN formula values,
 * for example) is found on the device: the call fails naming the first such (set of the call, branch, row) in call
 * order, and the output of the set chunks finished before it is unspecified.  nSets == 0 or nReps == 0 after the checks
 * does nothing.  As with the other batch entry points, nothing an evaluation reads is touched: conditionals, scalers,
 * walk plans, the branch cache, the staged root vector.  33..64 states only. */
int hb2_batch_site_simulate(hb2_partition *p, int64_t templateId, int64_t nSets, int64_t K, const int64_t *branchK,
                            const double *formulaValues, const double *weights, const int64_t *branchGroup,
                            const double *rootFreqs, int64_t nReps, uint64_t seed, int64_t firstSet, int64_t firstRep,
                            int64_t *leafStates, int64_t *nodeStates);

/* Multi-GPU (one process per GPU, patterns sharded by the caller: each rank creates its partition with its own
 * pattern shard).  After hb2_comm_init every hb2_evaluate* returns the SUM over ranks of the partial lnL
 * (a single fp64 ncclAllReduce on the partition's stream; per-pattern outputs stay local to the shard).
 * uniqueId: the 128 bytes of an ncclUniqueId produced by hb2_comm_unique_id on rank 0 and broadcast by the host. */
int hb2_comm_unique_id(void *uniqueId128);
int hb2_comm_init(hb2_partition *p, int nRanks, int rank, const void *uniqueId128);

/* Optional second sharding axis for partitions with rate classes (the per-class loop of
 * ComputeSiteLikelihoodsForABlock, likefunc2.cpp:912, iterates independent ComputeBlock calls): the nRanks ranks are
 * arranged as (nRanks/nGroups pattern shards) x (nGroups class groups); rank r belongs to class group r % nGroups and
 * pattern shard r / nGroups, i.e. the nGroups consecutive ranks of one shard are created with the SAME pattern slice.
 * Group g owns classes [g*C/nGroups, (g+1)*C/nGroups): matrices handed over for other classes are ignored on this
 * rank (no expm, no pruning), hb2_evaluate_classes prunes the owned classes only, and the per-pattern class partials
 * (value, binary exponent) of all ranks are exchanged before the logarithm with ONE collective per evaluation: every
 * rank writes its partials into its own slot of a buffer that is zero elsewhere and a sum ncclAllReduce acts as the
 * gather; every rank then merges every shard and holds the complete, bit-identical lnL (no second collective).
 * Requires C % nGroups == 0 and nRanks % nGroups == 0; hb2_evaluate (single class) is refused in this mode.  Call after
 * hb2_comm_init, before the first matrix is set. */
int hb2_comm_class_groups(hb2_partition *p, int nGroups);
/* Per-pattern outputs of ALL pattern shards on every rank (SURVEY 8e: "per-pattern outputs, when requested, are gathered";
 * what the host needs for ConstructCategoryMatrix / SITE_LOG_LIKELIHOODS on a sharded partition, likefunc.cpp:1791).
 * siteL / siteScale: this rank's S values as returned by the last hb2_evaluate*; allSiteL / allSiteScale: room for
 * `capacity` patterns, filled in shard order (= pattern order of the unsharded partition when shards are contiguous
 * slices); *total = patterns over all shards.  Collective over the partition's communicator (two ncclAllGather). */
int hb2_comm_gather_sites(hb2_partition *p, const double *siteL, const int64_t *siteScale, double *allSiteL,
                          int64_t *allSiteScale, int64_t capacity, int64_t *total);

/* Pair of SetupLFCaches in DeleteCaches (likefunc.cpp:10556-10601). */
void hb2_destroy(hb2_partition *p);

/* Host-side planner of the tensor-core pruning pass, callable WITHOUT a GPU (tests/test_planner.py): for a tree (same
 * flatParents as hb2_create), a dirty set given as hb2_evaluate's updateNodes (NULL or nUpdate < 0 = whole tree) and a
 * number of lanes (1..15), returns the lanes' step lists exactly as the kernel receives them: laneStart[lanes+1] and
 * 2 ints per step -- child id | HB2_STEP_WAIT (1<<30: produced by another lane) | HB2_STEP_CHAIN (1<<29: produced by
 * the lane's previous job, taken from registers) | HB2_STEP_MUL (1<<28: side product, multiply without a matrix); job's
 * node slot (>= I: side product of node slot-I) | HB2_STEP_FIRST (1<<28) | HB2_STEP_LAST (1<<29).  `steps` must hold
 * 2*(L+2I) ints.  splitNodes: bit 0 = side products on; bit 1 = the fp64 lanes kernel's rule for nodes with more than
 * two children (never split or chained, children in tree order), which makes conditionals independent of the plan. */
int hb2_plan_walk(int64_t L, int64_t I, const int64_t *flatParents, int64_t nUpdate, const int64_t *updateNodes, int lanes,
                  int splitNodes, int32_t *laneStart, int32_t *steps, int64_t stepCapacity, int64_t *nSteps);

/* Introspection for tests/bench: kernel launches issued so far by this partition, and device pointers/timing. */
int64_t hb2_launch_count(const hb2_partition *p);
/* 0: fp64 pruning kernels (4/20-state register kernels, or HB2_FLAG_FORCE_FP64);
 * 1: tensor-core (wgmma) pruning, error-compensated 3xTF32 split with fp32 conditionals (33..64 states). */
int hb2_precision_mode(const hb2_partition *p);
/* Name of the pruning kernel this partition launches, and the kernel launches per evaluation of the three stages
 * {expm, pruning, root reduction} as counted during the last hb2_time_resident (bench.py's roofline object). */
const char *hb2_pruning_kernel(const hb2_partition *p);
int hb2_stage_launches(const hb2_partition *p, int64_t *out3);
/* Runs the same work as hb2_evaluate_classes `iters` times with inputs already resident on the device
 * (re-exponentiating every cached rate matrix and re-pruning the whole tree each time) and returns the mean
 * device time per evaluation in milliseconds (CUDA events on the partition's stream).  stageMs (nullable, 3 doubles)
 * receives the mean per-stage times {expm, pruning, root reduction}. */
int hb2_time_resident(hb2_partition *p, const double *weights, const double *rootFreqs, int iters,
                      double *msPerEval, double *stageMs, double *lnL);

#ifdef __cplusplus
}
#endif
#endif /* HYPHY_B200_H */
