/* skdist_b200.h -- C-ABI of libskdist_b200.so (hand-written sm_90a CUDA, no torch types).
 *
 * This is the drop-in boundary for the hot path of Ibotta/sk-dist (reference v0.1.9):
 * the per-task fits that skdist.distribute fans out over Spark executors.  The
 * reference has no FFI (it is pure Python); each entry point below names the Python
 * call site whose work it replaces ("ref:" = path under the reference tree, "SK/" =
 * site-packages/sklearn 1.9.0, the third-party code that executes the arithmetic).
 * INTEGRATION.md shows the ctypes stub a maintainer would add on the reference side.
 *
 * Conventions: every function returns 0 on success, non-zero on error; the message is
 * available from skd_last_error(ctx) (ctx may be NULL for creation failures).  All
 * pointers are HOST pointers owned by the caller unless the name says `_device`.
 * A context is bound to one GPU and must be used from one host thread at a time.
 */
#ifndef SKDIST_B200_H
#define SKDIST_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct skd_ctx skd_ctx;

/* Library version (major*10000 + minor*100 + patch). */
int skd_version(void);

/* Create / destroy a context on CUDA device `device`.
 * ref: replaces the SparkContext `sc` argument of every Dist* estimator
 * (skdist/distribute/search.py:309-313). */
int skd_ctx_create(int device, skd_ctx** out);
int skd_ctx_destroy(skd_ctx* ctx);
const char* skd_last_error(skd_ctx* ctx);

/* Number of CUDA devices visible (0 if none / driver missing). */
int skd_device_count(void);

/* Stage the design matrix once in HBM (fp32, row-major, n rows, d features, leading
 * dimension ldx >= d in elements).
 * ref: replaces shipping X in the task closure / sc.broadcast
 * (skdist/distribute/search.py:414-421, multiclass.py:35-50). */
int skd_stage_x(skd_ctx* ctx, const float* X, int64_t n, int64_t d, int64_t ldx);
/* Same, from a DEVICE pointer on ctx's device (e.g. the buffer an NCCL broadcast filled). */
int skd_stage_x_device(skd_ctx* ctx, const float* dX, int64_t n, int64_t d, int64_t ldx);
/* The staged matrix in HBM (device pointer owned by ctx, valid until the next staging call): the source
 * of the NCCL broadcast that replicates X on the other ranks' GPUs over NVLink.
 * ref: the sc.broadcast of search.py:414-421. */
int skd_staged_x(skd_ctx* ctx, const float** dX, int64_t* n, int64_t* d, int64_t* ldx);

/* Sliced staging when every rank holds X on the host (SPMD fit under torchrun): begin allocates the
 * device buffer for n rows (n_alloc >= n rows of capacity, so that N equal slices fit) and returns it;
 * rows copies this rank's slice [row0, row0 + n_rows) host -> device through its own PCIe link; the
 * caller all-gathers the slices in place over NVLink (torch.distributed / NCCL); commit validates the
 * matrix (NaN / infinity check as skd_stage_x) and makes it the staged X.
 * ref: the sc.broadcast of search.py:414-421, with the host -> device copy divided over the GPUs. */
int skd_stage_x_begin(skd_ctx* ctx, int64_t n, int64_t d, int64_t n_alloc, const float** dX, int64_t* ldx);
int skd_stage_x_rows(skd_ctx* ctx, const float* X_rows, int64_t ld, int64_t row0, int64_t n_rows);
int skd_stage_x_commit(skd_ctx* ctx);

/* Stage integer class ids (0..K-1), one per row.  Column j of a batch treats rows with
 * y_class == col_pos[j] as positive, the rest as negative.
 * ref: y in the closure (search.py:416-421); LabelBinarizer columns (multiclass.py:289-317). */
int skd_stage_labels(skd_ctx* ctx, const int32_t* y_class, int64_t n);

/* Stage real-valued targets (regression; Ridge).  ref: same as above. */
int skd_stage_targets(skd_ctx* ctx, const float* y, int64_t n);

/* Stage the cross-validation layout as one int8 fold id per row (0..n_folds-1; test fold
 * of the row).  Replaces the per-task (train_idx, test_idx) index arrays and the
 * X[train]/X[test] copies.  ref: search.py:378-383 (fit_sets), utils.py:171-209 (_safe_split). */
int skd_stage_folds(skd_ctx* ctx, const int8_t* fold_id, int64_t n, int32_t n_folds);

/* Per-column feature masks for the NEXT skd_logreg_fit_batch call (one-shot): mask[j*d + k] = 1
 * if feature k takes part in column j's fit, 0 if it is left out (its weight stays exactly 0, which
 * equals fitting on X with those columns dropped).  B must equal the batch size of that call;
 * mask = NULL clears.  ref: replaces the `_drop_col(X, index)` copies of eliminate.py:22-38
 * (_fit_and_score_one) -- one feature set x fold per column. */
int skd_stage_column_masks(skd_ctx* ctx, int32_t B, const uint8_t* mask);

/* Row bit matrices for the NEXT skd_logreg_fit_batch call (one-shot; NULL / B = 0 clears): bit r of
 * column j in `label_bits` = the binary label of row r in that column (instead of class id == col_pos[j]:
 * multilabel targets), in `train_bits` = row r takes part in the column's fit (instead of every row: the
 * reference's negative down-sampling).  Packed little-endian, `bytes_per_col` bytes per column (>= n / 8);
 * either matrix may be NULL.  Not combinable with folds or pair columns.
 * ref: the label columns of multiclass.py:288-297 (LabelBinarizer output of a multilabel y) and
 * `_negatives_mask` (multiclass.py:76-106). */
int skd_stage_row_bits(skd_ctx* ctx, int32_t B, const uint8_t* label_bits, const uint8_t* train_bits,
                       int64_t bytes_per_col);

/* Class weights for the NEXT skd_logreg_fit_batch, skd_logreg_loss_grad or skd_logreg_multinomial_fit_batch
 * call (one-shot; w = NULL or B = 0 clears).  w [B x K] float32, finite and >= 0: weight of each class in
 * column j (binary calls: K = 2, w[2j] for label 0 and w[2j + 1] for label 1; multinomial: K = n_classes,
 * indexed by class id).  sw_sum [B] > 0: the sum of the per-row weights over the column's training rows.
 * The call that reads them fails unless its B (and K) match.  Each training row's loss and gradient entry
 * is multiplied by its weight, and sw_sum takes the place of n_train in the mean and in the l2 strength
 * 1 / (C sw_sum).  ref: `class_weight` of LogisticRegression (SK/linear_model/_logistic.py:429-474). */
int skd_stage_class_weights(skd_ctx* ctx, int32_t B, int32_t K, const float* w, const double* sw_sum);

/* Per-row sample weights for the NEXT skd_logreg_fit_batch, skd_logreg_loss_grad,
 * skd_logreg_multinomial_fit_batch or skd_logreg_multinomial_loss_grad call (one-shot, cleared by that call
 * even when it fails; w = NULL clears).  w [n] float32, one per staged row, finite and >= 0; the call fails
 * unless n equals the staged row count.  Every column of that call weighs training row i by w[i] times the
 * class weight of the row's label in that column (a float32 product), so the call also needs class weights
 * staged for it (all ones without class_weight): their sw_sum must be the sum of those products over the
 * column's training rows.  Rows of weight 0 add nothing to the loss or the gradient.  The scoring entries do
 * not use sample weights: scores stay unweighted.  ref: `sample_weight` of LogisticRegression.fit
 * (SK/linear_model/_logistic.py:409-474), indexed by each fit's training rows (ref search.py:208-211). */
int skd_stage_sample_weights(skd_ctx* ctx, const float* w, int64_t n);

/* Class weights for the NEXT skd_forest_fit (classification; one-shot, cleared by that call even when it
 * fails; n_classes <= 0, or w = NULL without balanced_subsample, clears).  Tree t is fitted with
 * sample_weight count_i * cw[y_i]: w [n_classes] float64, finite and >= 0, the same for every tree, or
 * balanced_subsample != 0 (w unused): per tree cw_k = n / (K_present * N_k) from the tree's bootstrap class
 * counts N_k (compute_class_weight("balanced") of the bootstrap sample; absent classes 0).  Rows of weight 0
 * leave the tree.  min_weight_fraction_leaf replaces the fit's min_weight_leaf: per tree, fraction * (sum of
 * the tree's weights).  The fit fails if its n_classes differs or it is a regression fit.
 * ref: `class_weight` of the forest classifiers (ensemble.py:68-109, 229-238). */
int skd_stage_forest_class_weights(skd_ctx* ctx, int32_t n_classes, const double* w, int32_t balanced_subsample,
                                   double min_weight_fraction_leaf);

/* Split criterion of the NEXT skd_forest_fit (one-shot, cleared by that call even when it fails): 0 = Gini
 * (classification) / squared error (regression), the default; 1 = entropy in bits (classification only:
 * the fit fails with a regression target).  Entropy fits always run the general tree builder.  The forest's
 * `impurity` arrays are formed on the host with the host's log from the nodes' class sums, as scikit-learn
 * forms them.  ref: `criterion="entropy"` / "log_loss" of the forest classifiers (SK/tree/_criterion.pyx
 * Entropy). */
int skd_stage_forest_criterion(skd_ctx* ctx, int32_t criterion);

/* Batched binary L2 logistic regression (lbfgs), B independent columns sharing X.
 * Column j: positives = rows with y_class == col_pos[j]; training rows = rows whose fold id
 * != col_fold[j] (col_fold[j] < 0: all rows); l2 strength = 1 / (C[j] * n_train_j).
 * col_neg (may be NULL): col_neg[j] >= 0 restricts column j to the rows of class col_pos[j] or
 * col_neg[j] -- the one-vs-one pair fit of multiclass.py:155-173 (_fit_ovo_binary) without the
 * X[cond] copy; col_neg[j] < 0 keeps every other class as negatives (one-vs-rest).
 * Outputs: coef_out[j*(d+1) + k] (k<d weights, k==d intercept, 0 if !fit_intercept),
 * n_iter_out[j] = min(nit, max_iter), status_out[j] (1,2 converged; 3 max_iter; 4 abnormal
 * line search; 5 non-finite), loss_out[j] final objective, n_evals_out[j] number of
 * loss+gradient evaluations, gpu_seconds_out (CUDA-event time of the whole call; may be NULL).
 * ref: replaces B invocations of search.py:180-288 (_fit_and_score -> estimator.fit,
 * line 230) / multiclass.py:109-152 (_fit_binary) for LogisticRegression(solver="lbfgs",
 * penalty="l2"): SK/linear_model/_logistic.py:219-717, SK/linear_model/_linear_loss.py:291-379,
 * scipy L-BFGS-B with maxiter=max_iter, maxls=50, gtol=tol, ftol=64*eps. */
int skd_logreg_fit_batch(skd_ctx* ctx, int32_t B, const double* C, const int32_t* col_fold,
                         const int32_t* col_pos, const int32_t* col_neg, int32_t fit_intercept,
                         double tol, int32_t max_iter, float* coef_out, int32_t* n_iter_out,
                         int32_t* status_out, double* loss_out, int32_t* n_evals_out,
                         double* gpu_seconds_out);

/* Objective and gradient of B columns at caller-supplied points w_in[j*(d+1)+k] (float64;
 * cast to fp32 for the products as sklearn does).  loss_out[j], grad_out[j*(d+1)+k] follow
 * SK/linear_model/_linear_loss.py:291-379 exactly (mean loss + 0.5*l2*|w|^2, intercept last).
 * Diagnostic / test entry: it runs the evaluation kernel skd_logreg_fit_batch would run on the same
 * columns, in the same slot layout (on the tensor cores: sorted by held-out fold into groups of 128
 * slots, with the per-fold tile lists; TC_FIT_UNI when every column has the same col_pos and at most
 * 32 folds are staged, TC_FIT otherwise).  Outputs are in column order. */
int skd_logreg_loss_grad(skd_ctx* ctx, int32_t B, const double* w_in, const double* C,
                         const int32_t* col_fold, const int32_t* col_pos, int32_t fit_intercept,
                         double* loss_out, double* grad_out);

/* Accuracy counts of B linear binary classifiers on their held-out rows.
 * Column j is scored on rows whose fold id == col_fold[j] (col_fold[j] == -2: all rows;
 * col_fold[j] == -3-f: rows NOT in fold f, i.e. the training rows, for return_train_score);
 * prediction = (x.w + b > 0) compared with (y_class == col_pos[j]).
 * ref: replaces search.py:264 (_score -> ClassifierMixin.score -> accuracy_score). */
int skd_linear_score_batch(skd_ctx* ctx, int32_t B, const float* coef, const int32_t* col_fold,
                           const int32_t* col_pos, int64_t* correct_out, int64_t* count_out);

/* B multinomial (n_classes >= 2) L2 logistic regressions sharing the staged X and class ids
 * 0..n_classes-1 (the call fails, naming the staged range, when a class id lies outside it): candidate j minimises mean_i[logsumexp(W x_i + b) - (W x_i + b)_{y_i}] +
 * 0.5 / (C[j] * n_train) * ||W||^2 over the rows whose fold id != col_fold[j] (col_fold[j] < 0: all
 * rows) with L-BFGS-B from W = 0 (m = 10, maxls = 50, gtol = tol, ftol = 64 eps, like scikit-learn's
 * call).  coef_out[(j * n_classes + k) * (d+1) + i]: i < d weights of class k, i == d its intercept.
 * Column masks staged with skd_stage_column_masks apply to the candidates (a masked feature keeps weight 0 in
 * every class row) and are consumed by this call.
 * ref: replaces the estimator.fit of search.py:228-230 for a multiclass target
 * (SK/linear_model/_logistic.py:523-547,584-598; SK/_loss/_loss.pyx.tp:1293-1327). */
int skd_logreg_multinomial_fit_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const double* C,
                                     const int32_t* col_fold, int32_t fit_intercept, double tol, int32_t max_iter,
                                     float* coef_out, int32_t* n_iter_out, int32_t* status_out, double* loss_out,
                                     int32_t* n_evals_out, double* gpu_seconds_out);

/* Objective and gradient of B multinomial candidates at caller-supplied points
 * w_in[(j * n_classes + k) * (d+1) + i] (float64, the layout of coef_out above; cast to fp32 for the products as
 * scikit-learn does, intercepts read as 0 without fit_intercept).  loss_out[j], grad_out (same layout as w_in)
 * follow SK/linear_model/_linear_loss.py:291-379, multiclass branch (mean loss + 0.5*l2*|W|^2, intercepts
 * unpenalised).  Staged class weights and column masks apply as in skd_logreg_multinomial_fit_batch and are
 * consumed by this call.  Diagnostic / test entry: it runs the passes, buffers, evaluation kernels and gradient
 * reduction of one round of skd_logreg_multinomial_fit_batch on the same batch, every candidate active.  Fails
 * like the fit on class ids outside 0..n_classes-1, C <= 0, an empty training set or staged inputs that do not
 * match B (x d, x n_classes). */
int skd_logreg_multinomial_loss_grad(skd_ctx* ctx, int32_t B, int32_t n_classes, const double* w_in, const double* C,
                                     const int32_t* col_fold, int32_t fit_intercept, double* loss_out,
                                     double* grad_out);

/* Accuracy counts of B multiclass linear classifiers (coef laid out as above): prediction =
 * first arg max_k (W x + b)_k compared with the staged class id, on the rows selected by the fold
 * codes of skd_linear_score_batch.  This entry, the confusion counts below and the multiclass log loss fail
 * when a staged class id lies outside 0..n_classes-1.
 * ref: replaces search.py:264 (_score -> ClassifierMixin.score -> accuracy_score). */
int skd_multinomial_score_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const float* coef,
                                const int32_t* col_fold, int64_t* correct_out, int64_t* count_out);

/* Confusion counts of the same classifiers on the same rows: confusion_out[(j * K + t) * K + p] = rows of
 * true class t predicted as class p (K = n_classes).  Every count-based multiclass scorer (f1 / precision /
 * recall with micro, macro or weighted averaging, balanced accuracy) is a function of this matrix.
 * ref: replaces search.py:264 (_score -> scorer(estimator, X_test, y_test)) for those scorers
 * (the reference's examples/search/hand_written_digits.py uses scoring="f1_weighted"). */
int skd_multinomial_confusion_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const float* coef,
                                    const int32_t* col_fold, int64_t* confusion_out);

/* Area under the ROC curve of B linear binary classifiers on the rows selected by the fold codes of
 * skd_linear_score_batch, as exact integer counts: u2_out[j] = 2 * U with U = #{(p, q): z_p > z_q} +
 * 0.5 * #{z_p == z_q} over positive rows p (y_class == col_pos[j]) and negative rows q of the fp32 decision
 * values z = x.w + b; auc = u2 / (2 * n_pos * n_neg) (== roc_auc_score(y, decision_function(X))).
 * ref: replaces search.py:264 for scoring="roc_auc" (the reference's examples/search/basic_usage.py). */
int skd_linear_auc_batch(skd_ctx* ctx, int32_t B, const float* coef, const int32_t* col_fold,
                         const int32_t* col_pos, int64_t* u2_out, int64_t* n_pos_out, int64_t* n_neg_out);

/* Ranked counts of B linear classifiers on the rows selected by the fold codes of skd_linear_score_batch, per
 * SEGMENT: u2_out = 2U (U = #{(p, q): s_p > s_q} + 0.5 * #{s_p == s_q} over positive rows p and negative rows q),
 * n_pos_out, n_neg_out, and ap_out = average precision (sum over the tie groups in descending score of
 * pos_g * tp_g / (tp_g + fp_g), divided by n_pos; 0 without positives).  auc = u2 / (2 * n_pos * n_neg).
 *   n_classes == 1: coef [B][d+1] binary columns, one segment per column, positives y_class == col_pos[j].
 *   n_classes = K > 2: coef [B][K][d+1], class ids 0..K-1; pairs == 0: K one-vs-rest segments per column
 *     (segment k: positives y == k, score s_k); pairs == 1: K (K - 1) one-vs-one segments, ordered pair (a, b)
 *     at a * (K - 1) + (b < a ? b : b - 1): the rows with y in {a, b}, positives y == a, score s_a.
 * score_kind: 0 the fp32 decision values z = x.w + b, 1 their negation (pos_label = classes_[0]), 2 the float32
 * predict_proba of LogisticRegression (expit for binary columns, softmax for K > 2; K <= 128), within
 * (K + 10) * 2^-23 relative of numpy's (the device exp is correctly rounded, numpy's float32 exp within 4 ulp).
 * Outputs are [B][segments].
 * ref: replaces search.py:264 for scoring="roc_auc_ovr", "roc_auc_ovr_weighted", "roc_auc_ovo",
 * "roc_auc_ovo_weighted" (predict_proba) and "average_precision" (decision_function). */
int skd_linear_rank_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const float* coef, const int32_t* col_fold,
                          const int32_t* col_pos, int32_t score_kind, int32_t pairs, int64_t* u2_out,
                          int64_t* n_pos_out, int64_t* n_neg_out, double* ap_out);

/* Log loss of the predicted probabilities on the rows selected by the fold codes of
 * skd_linear_score_batch: loss_sum_out[j] = sum_i -log(clip(p_i[y_i], eps, 1 - eps)), eps = float32 epsilon,
 * p = softmax of the fp32 decision values; count_out[j] = rows.  n_classes == 1: B binary columns
 * (coef [B][d+1], true class = y_class == col_pos[j], p = [1 - expit(z), expit(z)]); n_classes > 2: coef
 * [B][n_classes][d+1], col_pos unused.  log_loss = loss_sum / count.
 * ref: replaces search.py:264 for scoring="neg_log_loss" (log_loss(y_test, predict_proba(X_test))). */
int skd_linear_logloss_batch(skd_ctx* ctx, int32_t B, int32_t n_classes, const float* coef, const int32_t* col_fold,
                             const int32_t* col_pos, double* loss_sum_out, int64_t* count_out);

/* Batched Ridge: B independent (alpha, fold) columns from one pass over the staged X and the
 * staged real targets.  Column j trains on rows whose fold id != col_fold[j] (col_fold[j] < 0: all
 * rows).  coef_out[j*(d+1)+k] (k<d weights, k==d intercept); status_out[j] 1 = ok, 4 = matrix not
 * positive definite.  Supports d <= 338 (each column's Cholesky factor is held in shared memory);
 * larger d fails with an error before any work is launched.
 * ref: replaces B invocations of search.py:180-288 with estimator = Ridge (dense, solver
 * auto->cholesky): SK/linear_model/_base.py:113-220 (centring), SK/linear_model/_ridge.py:215-234
 * (_solve_cholesky: X^T X, X^T y, LAPACK posv). */
int skd_ridge_fit_batch(skd_ctx* ctx, int32_t B, const double* alpha, const int32_t* col_fold,
                        int32_t fit_intercept, float* coef_out, int32_t* status_out,
                        double* gpu_seconds_out);

/* Exact-order column-batched SGD: B one-vs-rest label columns (positives of column j = rows with
 * y_class == col_pos[j]) trained with the SAME shuffled sample order, one warp per column.
 * loss: 0 hinge, 1 log_loss; penalty l2; lr_type: 0 optimal, 1 constant, 2 invscaling; `seed` and
 * `optimal_init` are computed by the host exactly as scikit-learn does.  coef_out [B x d] float32
 * (after reset_wscale), intercept_out [B] float64, n_iter_out epochs run, t_out = 1 + n_iter * n,
 * status_out 1 = converged (n_iter_no_change), 3 = max_iter reached, 5 = non-finite.
 * ref: replaces B invocations of multiclass.py:109-152 (_fit_binary -> SGDClassifier.fit):
 * SK/linear_model/_stochastic_gradient.py:387-515, SK/linear_model/_sgd_fast.pyx.tp:274-640. */
int skd_sgd_fit_batch(skd_ctx* ctx, int32_t B, const int32_t* col_pos, int32_t loss, double alpha,
                      int32_t fit_intercept, int32_t max_iter, double tol, int32_t shuffle,
                      uint32_t seed, int32_t lr_type, double eta0, double power_t, double optimal_init,
                      int32_t n_iter_no_change, float* coef_out, double* intercept_out,
                      int32_t* n_iter_out, double* t_out, int32_t* status_out, double* gpu_seconds_out);

/* The same exact-order SGD for cross-validation: B binary columns in G order groups.  Column j fits
 * group col_group[j] with its own col_alpha[j] (> 0) and col_optimal_init[j] (computed by the host per alpha,
 * as for skd_sgd_fit_batch); positives = rows with y_class == col_pos[j].  Group g walks the rows
 * group_rows[group_offsets[g] .. group_offsets[g+1]) (a fold's training rows, in the splitter's order; int32
 * row ids, every group non-empty, group_offsets[0] = 0) and shuffles that list every epoch with its own
 * group_seeds[g]; its t and per-epoch objective use n_g = its row count, so t_out = 1 + n_iter * n_g.
 * Every other argument and output as skd_sgd_fit_batch.  All groups run side by side in one launch per epoch
 * on the warp-per-column kernels (never on the tensor cores).
 * ref: replaces B invocations of search.py:180-288 (_fit_and_score: estimator.fit(X[train], y[train])) with
 * estimator = SGDClassifier: SK/linear_model/_stochastic_gradient.py:387-515 (binary) and :795-830 (one
 * seed per class, seeds = RandomState(random_state).randint(MAX_INT, size=K)),
 * SK/linear_model/_sgd_fast.pyx.tp:274-640. */
int skd_sgd_fit_groups(skd_ctx* ctx, int32_t B, const int32_t* col_pos, const int32_t* col_group,
                       const double* col_alpha, const double* col_optimal_init, int32_t G, const int64_t* group_offsets,
                       const int32_t* group_rows, const uint32_t* group_seeds, int32_t loss, int32_t fit_intercept,
                       int32_t max_iter, double tol, int32_t shuffle, int32_t lr_type, double eta0, double power_t,
                       int32_t n_iter_no_change, float* coef_out, double* intercept_out, int32_t* n_iter_out,
                       double* t_out, int32_t* status_out, double* gpu_seconds_out);

/* Host-only helper (no CUDA, no context): bootstrap multiplicities and splitter seeds of n_trees trees
 * from their integer seeds, spread over host threads (n_threads <= 0: all cores, at most 64).
 * counts_out[t * n + i] = how often row i is drawn by RandomState(seeds[t]).randint(0, n, n) (needed only
 * when bootstrap != 0); rand_r_out[t] = RandomState(seeds[t]).randint(0, 2^31 - 1).  Bit-identical to numpy's
 * legacy generator.  Returns 0, 1 if a multiplicity exceeds 255 (device format), 2 on bad arguments.
 * ref: replaces the per-task `_generate_sample_indices` + `bincount` of ensemble.py:51-55, 97-99 and the seed draw
 * of SK/tree/_splitter.pyx:155. */
int skd_bootstrap_counts(int32_t n_trees, const uint32_t* seeds, int64_t n, int32_t bootstrap,
                         uint8_t* counts_out, uint32_t* rand_r_out, int32_t n_threads);

/* Forest classifier trees, one persistent CTA per tree (depth-first, exact scikit-learn
 * splitter semantics).  sample_counts[t*n + i] is the
 * bootstrap multiplicity of row i in tree t (the reference's sample_weight, uint8; NULL = no
 * bootstrap, every row once), rand_states[t] the splitter's xorshift seed; both are derived by the
 * host exactly as the reference does.  splitter:
 *   0 = best split of the drawn features (RandomForest, SK/tree/_splitter.pyx:262-504) on per-feature
 *       value histograms: every feature must have <= 256 distinct values, else the call fails;
 *   1 = one uniformly drawn threshold per drawn feature (ExtraTrees, node_split_random :507-736),
 *       any finite values;
 *   2 = as 0, and a feature with more than 256 distinct values is split by sorting the node's raw
 *       float32 values (the same trees; when every feature has <= 256 distinct values, exactly 0).
 * Trees come back through an opaque handle: sizes first, then caller-allocated arrays.
 * ref: replaces n_trees invocations of ensemble.py:68-109 (_build_trees -> tree.fit):
 * SK/tree/_tree.pyx:139-337, SK/tree/_splitter.pyx:262-504, SK/tree/_criterion.pyx:605-680. */
typedef struct skd_forest skd_forest;
int skd_forest_fit(skd_ctx* ctx, int32_t n_trees, const uint8_t* sample_counts, const uint32_t* rand_states,
                   int32_t n_classes, int32_t max_features, int32_t max_depth, int32_t min_samples_split,
                   int32_t min_samples_leaf, double min_weight_leaf, double min_impurity_decrease,
                   int32_t splitter, const double* y_regression, skd_forest** out, double* gpu_seconds_out);
/* Device time (CUDA events) of the tree-builder kernels of the last skd_forest_fit on ctx, without the
 * copies of bootstrap counts in and node arrays out: the numerator of the builder's HBM roofline. */
int skd_forest_kernel_seconds(skd_ctx* ctx, double* seconds_out);
int skd_forest_tree_size(skd_forest* f, int32_t tree, int32_t* node_count, int32_t* max_depth);
int skd_forest_tree_copy(skd_forest* f, int32_t tree, int32_t* left, int32_t* right, int32_t* feature,
                         double* threshold, double* impurity, int32_t* n_node_samples,
                         double* weighted_n_node_samples, uint8_t* missing_go_to_left, double* value);
/* One tree as scikit-learn `Node` records (64 bytes each: left, right, feature int64; threshold, impurity
 * float64; n_node_samples int64; weighted_n_node_samples float64; missing_go_to_left uint8 + padding;
 * SK/tree/_tree.pxd:15-25) plus value [node_count][n_classes]: the state `Tree.__setstate__` takes. */
int skd_forest_tree_nodes(skd_forest* f, int32_t tree, void* nodes64, double* value);
void skd_forest_free(skd_forest* f);

/* Sum of squared residuals and row counts of B linear regressors on the rows selected by the
 * same fold codes as skd_linear_score_batch; the host forms r2 = 1 - sse / sst.
 * ref: replaces search.py:264 (_score -> RegressorMixin.score -> r2_score). */
int skd_linear_r2_batch(skd_ctx* ctx, int32_t B, const float* coef, const int32_t* col_fold,
                        double* sse_out, int64_t* count_out);

/* Streaming batched inference on NEW host rows: out[i*B + j] = Xnew[i,:].coef_j + intercept_j.
 * Rows are moved in <= 256 MiB chunks; pageable sources go through a threaded pinned bounce so the
 * copy engine, not a single host memcpy, sets the pace.  gpu_seconds_out: time of the whole call.
 * ref: replaces skdist/distribute/predict.py:160-179 (pandas_udf around model.predict). */
int skd_predict_linear(skd_ctx* ctx, const float* Xnew, int64_t m, int64_t d, int64_t ld, int32_t B,
                       const float* coef, float* out, double* gpu_seconds_out);

/* Class-probability inference of a fitted forest on NEW host rows (soft voting):
 *   proba_out[i*C + c] = (1/n_trees) * sum_t value_t[leaf_t(x_i)][c]
 * with the trees given as concatenated sklearn `Tree` arrays: node k of tree t lives at index
 * tree_offset[t] + k of left/right/feature/threshold, its C class fractions at value[(..)*C].
 * A row goes left iff (double)x[feature] <= threshold (SK/tree/_tree.pyx:960-986); the per-tree
 * values are added in tree order in float64, i.e. exactly what
 * RandomForestClassifier.predict_proba computes with n_jobs=1 (SK/ensemble/_forest.py:947-966).
 * ref: replaces skdist/distribute/predict.py:160-179 for forest models (model.predict[_proba]). */
int skd_forest_predict(skd_ctx* ctx, const float* Xnew, int64_t m, int64_t d, int64_t ld,
                       int32_t n_trees, const int64_t* tree_offset, const int32_t* left,
                       const int32_t* right, const int32_t* feature, const double* threshold,
                       const double* value, int32_t n_classes, double* proba_out,
                       double* gpu_seconds_out);


/* Decision values out[i*B + j] = X[i,:].coef_j + intercept_j for the staged X (all rows).
 * ref: estimator.decision_function / predict inside scorers (utils.py:45-72) and
 * skdist/distribute/predict.py:160-179 (model.predict over row batches). */
int skd_linear_decision(skd_ctx* ctx, int32_t B, const float* coef, float* out);

/* Which evaluation kernel skd_logreg_fit_batch uses: 0 = auto, 1 = SIMT fp32, 2 = tensor-core (wgmma)
 * (fp16x2-split, fp32 accumulate).  Returns the previous value. */
int skd_set_kernel(skd_ctx* ctx, int32_t which);

/* Counters since context creation: kernels launched by this library, bytes H2D, bytes D2H. */
int skd_get_counters(skd_ctx* ctx, int64_t* launches, int64_t* h2d_bytes, int64_t* d2h_bytes);

/* Per-evaluation timing for the roofline report: reads the accumulators (summed CUDA-event
 * time of the evaluation launches of skd_logreg_fit_batch, their algorithmic FLOPs
 * (4 * n_train * d per active column per launch), launch and round counts) and then, if
 * enable >= 0, resets them and switches collection on (1) or off (0).  enable < 0: read only. */
int skd_profile(skd_ctx* ctx, int32_t enable, double* eval_ms, double* eval_flops,
                int64_t* eval_launches, int64_t* rounds);

/* CUDA-event stopwatch on the context's stream (the stream every kernel of this library is
 * launched on): start records an event, stop records a second one, waits for it and returns
 * the elapsed device time in milliseconds.  Used by bench.py to time K steps on the device. */
int skd_timer_start(skd_ctx* ctx);
int skd_timer_stop(skd_ctx* ctx, double* ms_out);

/* Host-side optimiser object exposing the same L-BFGS-B core the device kernels run
 * (csrc/lbfgs_core.h); used by the CPU tests that pin it against scipy's setulb.
 * ref: scipy/optimize/_lbfgsb_py.py:393-437 reverse-communication loop. */
typedef struct skd_lbfgs skd_lbfgs;
skd_lbfgs* skd_lbfgs_create(int32_t n, int32_t m, int32_t maxiter, int32_t maxls, double pgtol,
                            double ftol);
double* skd_lbfgs_x(skd_lbfgs* h);
double* skd_lbfgs_g(skd_lbfgs* h);
int skd_lbfgs_advance(skd_lbfgs* h, double f); /* returns status (0 = evaluate at x again) */
int skd_lbfgs_nit(skd_lbfgs* h);
int skd_lbfgs_nfev(skd_lbfgs* h);
/* the core's whole state, struct LbfgsScalars of csrc/lbfgs_core.h, as raw bytes; set_state writes it back
 * (tests: a core that loses one pair update, to show that the device comparison would notice) */
void skd_lbfgs_state(skd_lbfgs* h, void* out);
void skd_lbfgs_set_state(skd_lbfgs* h, const void* in);
int skd_lbfgs_state_bytes(void);
void skd_lbfgs_free(skd_lbfgs* h);

/* Diagnostic / test entry: the device optimiser of skd_logreg_fit_batch (K == 1) and
 * skd_logreg_multinomial_fit_batch (K >= 2) driven by caller-supplied evaluation partials
 * instead of an evaluation kernel.  It needs a staged X: d and the row pitch come from it.
 * create: B columns of K * (d + 1) variables, x0 = 0, memory 10; grouped = 1 runs the fold-grouped
 *   slot layout of the tensor-core fit (K == 1, d <= 256, labels staged; col_fold in -1..127),
 *   grouped = 0 slot s = column s; nz partials per slot; use_reduce = 1 reduces the gradient partials
 *   with the whole device first when nz > 8, as the tensor-core fit does; l2[B], inv_n[B];
 *   gscale[d] (K == 1) or NULL; fmask[B x d] (1 = feature takes part) or NULL.
 *   dims_out[4] = {variables per column, slot-list capacity, row pitch ldw, floats of rows_out}.
 * step: one optimiser round.  loss_parts[B][nz] and gsum_parts[B*K][nz] (float64) and
 *   grad_parts[B*K][nz][d] (fp32) are scattered by the current slot list into the partial buffers
 *   with stride n_act_in (between the live slot count and the capacity); slots that hold no live
 *   column get NaN.  Returns x_out[B][K*(d+1)], state_out[B] (struct LbfgsScalars), slot_out[cap][4]
 *   ({col, fold, pos, pad}), counts_out[4] = {slots, running, round record} and, if not NULL and
 *   dims_out[3] > 0, the exported fp32 rows (weights [slots x ldw], then one bias per slot).
 * finish: coef[B][K*(d+1)] (fp32), n_iter, status and loss of every column. */
typedef struct skd_lbfgs_dev skd_lbfgs_dev;
skd_lbfgs_dev* skd_lbfgs_dev_create(skd_ctx* ctx, int32_t B, int32_t K, int32_t d, int32_t fit_intercept,
                                    int32_t grouped, const int32_t* col_fold, int32_t nz, int32_t use_reduce,
                                    int32_t maxiter, int32_t maxls, double pgtol, double ftol, const double* l2,
                                    const double* inv_n, const double* gscale, const uint8_t* fmask,
                                    int32_t* dims_out);
int skd_lbfgs_dev_step(skd_lbfgs_dev* h, int32_t n_act_in, const double* loss_parts, const double* gsum_parts,
                       const float* grad_parts, double* x_out, void* state_out, int32_t* slot_out,
                       int32_t* counts_out, float* rows_out);
int skd_lbfgs_dev_finish(skd_lbfgs_dev* h, float* coef_out, int32_t* n_iter_out, int32_t* status_out,
                         double* loss_out);
void skd_lbfgs_dev_free(skd_lbfgs_dev* h);

#ifdef __cplusplus
}
#endif
#endif /* SKDIST_B200_H */
