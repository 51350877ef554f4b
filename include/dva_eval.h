/*
 * dva_eval.h -- C ABI of libdva_eval.so: segmentation evaluation on the H100 (sm_90a).
 *
 * The entry points replace the per-batch confusion update, the vote accumulation and the
 * full-resolution nearest-neighbour prediction of the reference's trackers
 * (torch_points3d/metrics/segmentation_tracker.py, s3dis_tracker.py, scannet_segmentation_tracker.py,
 * kitti360_tracker.py).  libdva_eval.so links against libdva_b200.so (rpath $ORIGIN): it reports its
 * errors through dva_last_error() and counts its launches in dva_launch_count() of that library.
 *
 * Conventions: those of dva_b200.h (device pointers, sizes, dtype code, the stream last, DVA_E*
 * return codes: <0 = argument error, nothing launched; >0 = cudaError_t of the failed launch).
 *   - K is the number of classes, 1 <= K <= DVA_EVAL_MAX_CLASSES; a larger K is DVA_EUNSUPPORTED.
 *   - the confusion matrix `cm` is int64 [K, K], row = ground truth, column = prediction; every
 *     update adds to it with integer atomics, so the result does not depend on the launch order.
 *   - `status` is one int32 word on the device.  A range error inside a kernel is not counted and
 *     ORs one of the DVA_EVAL_BAD_* bits into it; no entry point reads it back.
 *   - `has_ignore` = 0: every label counts; otherwise rows labelled `ignore_label` are skipped.
 */
#ifndef DVA_EVAL_H_
#define DVA_EVAL_H_

#include "dva_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define DVA_EVAL_MAX_CLASSES 64

/* status bits */
enum { DVA_EVAL_BAD_LABEL = 1, DVA_EVAL_BAD_PRED = 2, DVA_EVAL_BAD_ID = 4 };

/* full-resolution modes of dva_eval_nn_vote */
enum {
  DVA_EVAL_NN_INTERPOLATE = 0,      /* every query from its nearest voted point (s3dis_tracker.py:94-118) */
  DVA_EVAL_NN_INTERPOLATE_MEAN = 1, /* the same, voted rows divided by their counts first
                                       (scannet_segmentation_tracker.py:122-135) */
  DVA_EVAL_NN_OWN_VOTES = 2         /* a voted query keeps its own votes, the others are interpolated
                                       (kitti360_tracker.py:219-222) */
};

/* cm += confusion(labels, argmax(scores)) over rows i with counts[i] != 0 (counts may be NULL) and
 * labels[i] != ignore_label.  scores [n, K] of `dtype`; argmax takes numpy's rule: the first index of
 * the maximum, and the first NaN wins.  A label outside [0, K) sets DVA_EVAL_BAD_LABEL.
 * replaces: metrics/segmentation_tracker.py:76-85, s3dis_tracker.py:68-75 */
int dva_eval_confusion_scores(const void* scores, int dtype, const int64_t* labels, const int* counts, int64_t n,
                              int K, int64_t ignore_label, int has_ignore, int64_t* cm, int* status, void* stream);

/* cm += confusion(labels, pred), pred int64 [n]; a prediction outside [0, K) sets DVA_EVAL_BAD_PRED.
 * replaces: metrics/confusion_matrix.py:21-33 (count_predicted_batch) */
int dva_eval_confusion_pred(const int64_t* pred, const int64_t* labels, int64_t n, int K, int64_t ignore_label,
                            int has_ignore, int64_t* cm, int* status, void* stream);

/* votes[ids] += outputs; counts[ids] += 1, the last occurrence of a duplicated id winning.
 * votes fp32 [N, K], counts int32 [N], stamp int32 [N] all -1 on entry and on return (after a failed launch the
 * caller puts them back to -1: a claim left behind would drop a later vote); outputs [n, K] of
 * `dtype`, added in fp32 (one round-to-nearest add per element).  An id outside [0, N) is skipped and
 * sets DVA_EVAL_BAD_ID.  n < 2^31.
 * replaces: metrics/s3dis_tracker.py:76-80, scannet_segmentation_tracker.py:117-118 */
int dva_eval_vote(const void* outputs, int dtype, const int64_t* ids, int64_t n, int64_t N, int K, float* votes,
                  int* counts, int* stamp, int* status, void* stream);

/* Fused k = 1 knn_interpolate + argmax (+ confusion) over the queries.  votes fp32 [N, K], counts int32
 * [N], pos fp32 [N, 3]; voted int64 [nv] = the search set (table ids, in the order of the search);
 * query int64 [nq] table ids; nbr int64 [nq] the nearest search index of each query (unread for a voted
 * query in DVA_EVAL_NN_OWN_VOTES mode).  Writes pred int64 [nq]; with labels != NULL (int64 [N], read at
 * the query's id) also cm += confusion(labels, pred).  An id or neighbour index out of range sets
 * DVA_EVAL_BAD_ID and that query predicts 0 and is not counted.
 * replaces: torch_geometric knn_interpolate(k=1) + argmax in s3dis_tracker.py:107-113,
 * scannet_segmentation_tracker.py:124-135, kitti360_tracker.py:219-222 */
int dva_eval_nn_vote(const float* votes, const int* counts, const float* pos, int64_t N, int K, const int64_t* voted,
                     int64_t nv, const int64_t* query, const int64_t* nbr, int64_t nq, int mode,
                     const int64_t* labels, int64_t ignore_label, int has_ignore, int64_t* pred, int64_t* cm,
                     int* status, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* DVA_EVAL_H_ */
