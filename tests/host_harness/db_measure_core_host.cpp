// Host-side harness: runs the PRODUCT's geometry of the DB validation measure (megreader_b200/csrc/db_measure_core.cuh, the
// code the CUDA kernels in db_measure.cu execute) on the CPU, so that tests can compare it with the exact oracle without a GPU.
// Built on demand by tests/test_db_measure_cpu.py with g++.
#include "db_measure_core.cuh"

using namespace mr_dbmeas;

extern "C" {

// validity of the n [4, 2] float64 rings q
void host_valid(const double *q, int n, int *valid) {
    for (int i = 0; i < n; ++i) valid[i] = ring_prepare(q + 8 * i).valid;
}

// for n pairs (gt[i], det[i]) of [4, 2] float64 rings: both valid flags, and where both are valid the IoU and the
// intersection / area(det) the evaluator's don't-care test uses (0 elsewhere)
void host_pairs(const double *gt, const double *det, int n, int *valid_gt, int *valid_det, double *iou, double *precision) {
    for (int i = 0; i < n; ++i) {
        const Ring g = ring_prepare(gt + 8 * i), d = ring_prepare(det + 8 * i);
        valid_gt[i] = g.valid;
        valid_det[i] = d.valid;
        iou[i] = precision[i] = 0.;
        if (g.valid && d.valid) iou_precision(g, d, iou + i, precision + i);
    }
}

// evaluate_image's precision, recall and hmean from the counts
void host_metrics(int gt_care, int det_care, int matched, double *out) { image_metrics(gt_care, det_care, matched, out, out + 1, out + 2); }

}  // extern "C"
