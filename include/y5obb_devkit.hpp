// y5obb_devkit.hpp - the DOTA devkit's GPU entry points, exported by liby5obb.so under the reference's own C++ names, so that
// DOTA_devkit/poly_nms_gpu/poly_nms.pyx and poly_overlaps.pyx link against liby5obb.so instead of poly_nms_kernel.cu /
// poly_overlaps_kernel.cu with no source change (`cdef extern from "poly_nms.hpp"` -> this header).
// Replaces DOTA_devkit/poly_nms_gpu/poly_nms.hpp:9-10 and poly_overlaps.hpp:1.  Host pointers in and out,
// synchronous on the default stream of `device_id`; CUDA errors are printed to stdout, not returned (poly_nms_kernel.cu:20-27).
#ifndef Y5OBB_DEVKIT_HPP_
#define Y5OBB_DEVKIT_HPP_

// keep_out[0 .. *num_out) = indices of the kept polygons; polys_host [polys_num][polys_dim = 9] = x1 y1 .. x4 y4 score, ALREADY
// sorted by descending score (poly_nms.pyx:21-24 sorts before the call); a polygon is dropped when its IoU with an earlier kept
// one is > nms_overlap_thresh.
void _poly_nms(int* keep_out, int* num_out, const float* polys_host, int polys_num, int polys_dim, float nms_overlap_thresh,
               int device_id);
// overlaps[i * k + j] = IoU(boxes[i], query_boxes[j]); boxes are (x_ctr, y_ctr, w, h, angle_rad).
void _overlaps(float* overlaps, const float* boxes, const float* query_boxes, int n, int k, int device_id);

#endif  // Y5OBB_DEVKIT_HPP_
