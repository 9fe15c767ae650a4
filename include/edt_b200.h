/* include/edt_b200.h -- C ABI of the H100-native multi-label Euclidean distance transform.
 *
 * This is the drop-in boundary for the reference's hot path
 *     pyedt::_edt3dsq<T>(labels, sx,sy,sz, wx,wy,wz, black_border, parallel, workspace)
 *                                                    (reference src/edt.hpp:411-484)
 * and its 2-D / 1-D siblings (src/edt.hpp:632-678, 70-119), which the reference's Cython
 * layer binds in src/edt.pyx:63-87 (`cdef extern from "edt.hpp" namespace "pyedt"`).
 * Plain pointers and sizes only; no C++/torch types cross this boundary.
 *
 * Conventions shared by every entry point
 *   - volumes are x-fastest ("Fortran order" in the reference's words, README.md:100);
 *     C-ordered numpy arrays are handled by the caller swapping axes (src/edt.pyx:651-664);
 *   - labels are compared for equality only, as raw 1/2/4/8-byte unsigned integers
 *     (the reference instantiates uint8/16/32/64, float, double and bool: src/edt.pyx:670-732;
 *     float labels must be canonicalised by the caller so that -0.0 == +0.0);
 *   - the output is float32, same shape; with EDTB200_OUT_ON_DEVICE the transform runs in
 *     place in `out` (the reference's `workspace` argument has the same role);
 *   - every function returns 0 on success or a negative EDTB200_E* code;
 *     edtb200_last_error() gives the message (thread-local).  Nothing throws.
 *   - there is NO CPU fallback: without a usable CUDA device every transform fails with
 *     EDTB200_ECUDA.
 */
#ifndef EDT_B200_H
#define EDT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 100: round 1 (transform, per-axis passes, slab face kernels).  200: additions only --
 * edtb200_transform_multi, edtb200_slab_step / _stage_bytes / _pack, edtb200_label_stats / _extract,
 * edtb200_host_alloc / _free; every 100-level entry point keeps its signature and meaning.
 * 201: additions only -- edtb200_last_later_launch.  202: additions only -- edtb200_feature_transform.
 * Entry points added since (edtb200_transform_chunked, edtb200_feature_transform_chunked,
 * edtb200_transform_voxel_graph_chunked, edtb200_transform_stack, edtb200_feature_transform_stack,
 * edtb200_expand_gather, edtb200_surface_count, edtb200_surface_distances, edtb200_morphology,
 * edtb200_parabolic, edtb200_parabolic_sites, edtb200_nearest_labels, edtb200_nearest_labels_plan,
 * edtb200_medial_axis, edtb200_skeletonize, edtb200_pass_window, edtb200_local_thickness,
 * edtb200_geodesic, edtb200_noise_planes, edtb200_watershed, edtb200_connected_components,
 * edtb200_extended_maxima, edtb200_fill_holes, edtb200_dust)
 * keep the number: every 202-level entry point
 * keeps its signature and meaning, and a caller that needs a newer one looks its symbol up.  One
 * exception: edtb200_last_later_launch fills info[0..9) since the settled-tile skip (it filled
 * info[0..8) before), so its buffer must hold 9 ints. */
#define EDTB200_VERSION 202

/* flags */
#define EDTB200_SQRT             1  /* emit sqrt(edtsq): reference _edt3d (src/edt.hpp:591-604) /
                                       np.sqrt in edt() (src/edt.pyx:241-242), fused in the last store */
#define EDTB200_SIGNED           2  /* signed distance: background (label 0) is transformed as an
                                       ordinary label and its result negated -- equal to the
                                       reference's sdf()/sdfsq() = f(data) - f(data==0)
                                       (src/edt.pyx:121-202) */
#define EDTB200_LABELS_ON_DEVICE 4  /* `labels` is a device pointer on `device` */
#define EDTB200_OUT_ON_DEVICE    8  /* `out` is a device pointer on `device` */
#define EDTB200_LABELS_FLOAT    16  /* edtb200_transform_voxel_graph: the 4- / 8-byte labels are
                                       IEEE floats and foreground means value > 0, as the reference's
                                       float instantiations test it (src/edt_voxel_graph.hpp:76, 151);
                                       edtb200_expand_gather: background means value == 0 */

/* Residency, shared by edtb200_transform, edtb200_feature_transform and
 * edtb200_transform_voxel_graph: without EDTB200_LABELS_ON_DEVICE / EDTB200_OUT_ON_DEVICE the
 * inputs / outputs are host memory (pageable or pinned).  `stream` is a cudaStream_t (as void*) or
 * NULL.  A call with both flags is asynchronous on `stream`; a call that touches host memory
 * returns after its results have landed. */

/* error codes */
#define EDTB200_EINVAL  (-1)   /* bad argument */
#define EDTB200_ECUDA   (-2)   /* CUDA runtime / driver error, or no device */
#define EDTB200_ENOMEM  (-3)   /* device or host allocation failed */
#define EDTB200_ELIMIT  (-4)   /* size outside what the kernels support */

int edtb200_version(void);
const char *edtb200_last_error(void);

/* Number of visible CUDA devices (0 if none or on error). */
int edtb200_device_count(void);

/* Whole transform: edtsq / edt / sdfsq / sdf of a 1-D, 2-D or 3-D volume.
 *
 * Replaces  pyedt::_edt3dsq<T>        src/edt.hpp:411-484   (ndim == 3)
 *           pyedt::_edt2dsq<T>        src/edt.hpp:632-678   (ndim == 2; sz ignored)
 *           squared_edt_1d_multi_seg  src/edt.hpp:70-119    (ndim == 1; sy, sz ignored)
 *           pyedt::_edt3d / _edt2d    src/edt.hpp:591-604, 764-778  (EDTB200_SQRT)
 *           edt.sdf / edt.sdfsq       src/edt.pyx:121-202   (EDTB200_SIGNED)
 * For ndim < 3 the missing axis passes are skipped (not run on size-1 axes), exactly as the
 * reference's lower-dimensional drivers do.
 *
 *   labels       sx*sy*sz labels of `label_bytes` (1, 2, 4 or 8) bytes each; never written
 *   wx, wy, wz   anisotropy (voxel size) per axis
 *   black_border non-zero: the volume faces count as background
 *   out          sx*sy*sz float32
 *   device       CUDA device ordinal
 *   stream       see Residency above
 */
int edtb200_transform(const void *labels, int label_bytes, int ndim,
                      int64_t sx, int64_t sy, int64_t sz,
                      float wx, float wy, float wz,
                      int black_border, int flags,
                      float *out, int device, void *stream);

/* Feature transform: for every voxel p the coordinates of its nearest SITE, and optionally the
 * distance to it -- what scipy.ndimage.distance_transform_edt(return_indices=True) returns, for
 * multi-label volumes.
 *
 * A site of p is a voxel q whose label differs from p's, or with black_border a face position
 * (one coordinate -1 or n on its axis, the others inside the volume).
 *   foreground p                   a nearest site;
 *   background p, no EDTB200_SIGNED p itself (distance 0, as edtb200_transform gives it);
 *   background p, EDTB200_SIGNED   background is an ordinary label (as for sdf): the nearest voxel
 *                                  of any non-zero label, or a face position;
 *   no site at all                 every coordinate -1, distance +inf (-inf for signed
 *                                  background).  Only possible without black_border.
 * "Nearest" is in the transform's own float32 arithmetic: the distance from p to its site,
 * evaluated as the passes evaluate it (the X step table, then each later axis's term added in
 * double and rounded once to float32), is bit for bit what edtb200_transform returns for p.  Among
 * equally near sites any one may be returned, the same one on every run.
 *
 *   idx_out   ndim int32 planes laid out like the labels: idx_out[0] the x coordinate of the site,
 *             idx_out[1] y, idx_out[2] z.  One pointer per plane, so a caller may hand over the
 *             planes of an array in any order.
 *   dist_out  NULL, or sx*sy*sz float32 distances: EDTB200_SQRT / EDTB200_SIGNED as for
 *             edtb200_transform, equal to its result bit for bit
 *   flags     EDTB200_SIGNED, EDTB200_SQRT, EDTB200_LABELS_ON_DEVICE, and EDTB200_OUT_ON_DEVICE,
 *             which covers dist_out and every index plane (Residency above)
 * Every pass runs the one-thread-per-line kernels (no tile kernel).
 * Device memory of one call, for V voxels: the labels (V * label_bytes, when uploaded), the
 * distances (4V), one scratch volume for the passes' ping-pong (4V, ndim >= 2), the long-line
 * kernel's hull (4V, ndim >= 2), ndim code planes (4V each) and ndim index planes (4V each, when
 * downloaded): 36 bytes per voxel beyond the labels in 3-D, so 512^3 with uint32 labels needs
 * 40 * 2^27 bytes, about 5.4 GB.  An allocation that fails returns EDTB200_ENOMEM. */
int edtb200_feature_transform(const void *labels, int label_bytes, int ndim,
                              int64_t sx, int64_t sy, int64_t sz,
                              float wx, float wy, float wz,
                              int black_border, int flags, float *dist_out,
                              int32_t *const *idx_out, int device, void *stream);

/* Bounded transforms: only the distances up to max_distance = d, for callers that clamp, grow or
 * query within a radius.  Let L = (double)d * (double)d and S the squared value the unbounded call
 * gives a voxel (its edtsq, or |sdfsq| with EDTB200_SIGNED).
 *   transform          the bounded result is the unbounded one bit for bit where (double)S <= L, and
 *                      +inf elsewhere (-inf on signed background); unsigned background stays 0.  The
 *                      cut is made on the squared value, before sqrt and sign, as expand_labels'
 *                      (double)|sqdist| <= limit_sq.  This holds for edtsq, edt, sdfsq and sdf.
 *   feature transform  inside the band distances as above and sites as edtb200_feature_transform's
 *                      (the distance to the site is the distance returned, bit for bit); outside it
 *                      every coordinate -1 and the distance +inf (-inf on signed background), the "no
 *                      site" encoding; unsigned background maps to itself.  Among equally near sites
 *                      any one may be returned, the same one on every run.
 *   d = +inf           the unbounded call, unchanged.  d = 0 is allowed; a negative or NaN d is
 *                      EDTB200_EINVAL.
 * How: with B the largest float32 with (double)B <= L, a later-axis pass along axis k only needs the
 * samples within R_k rows of a voxel, R_k the largest r >= 0 with (double)w2_k * r * r <
 * nextafterf(B, +inf), w2_k = fl32(w_k * w_k).  A pass with R_k up to a limit runs a window kernel
 * (2 R_k + 1 rows, no hull, no scratch beyond one ping-pong volume); any other pass runs the unbounded
 * kernel, and a streaming kernel applies the cut.  The limits were measured on an H100
 * (records/h100/bounded_bench.txt): the window kernel beats the feature transform's long-line kernel
 * at every radius measured (up to 32), but the distance transform's tile kernels only at radii of 2
 * or less, and not on blocky labels.  edtb200_last_later_launch reports a window pass as kernel 2 with its radius in info[1]. */
#define EDTB200_BOUNDED_WINDOW_MAX 2         /* edtb200_transform_bounded */
#define EDTB200_BOUNDED_SITES_WINDOW_MAX 32  /* edtb200_feature_transform_bounded */

/* edtb200_transform with max_distance (the bounded transform above).  Residency, staging and
 * asynchrony as edtb200_transform; device memory: one more float32 volume of scratch when a later
 * pass takes the window kernel.  An allocation that fails returns EDTB200_ENOMEM (there is no
 * chunked retry).  Checks, in order: as edtb200_transform (label width, ndim, sizes, emptiness,
 * pointers), then max_distance, then the device. */
int edtb200_transform_bounded(const void *labels, int label_bytes, int ndim,
                              int64_t sx, int64_t sy, int64_t sz,
                              float wx, float wy, float wz,
                              int black_border, int flags,
                              float *out, int device, void *stream, double max_distance);

/* edtb200_feature_transform with max_distance (the bounded feature transform above).  Residency and
 * checks as there, then max_distance, then the device.  A window pass needs no long-line hull (4 bytes
 * per voxel while a long-line pass runs), so in 3-D, when every later pass takes the window kernel,
 * the device memory beyond the labels is 32 bytes per voxel instead of 36. */
int edtb200_feature_transform_bounded(const void *labels, int label_bytes, int ndim,
                                      int64_t sx, int64_t sy, int64_t sz,
                                      float wx, float wy, float wz,
                                      int black_border, int flags, float *dist_out,
                                      int32_t *const *idx_out, int device, void *stream,
                                      double max_distance);

/* The plan of a bounded transform, pure host logic (no device needed): radius[k] = R_k for every axis
 * k < ndim (capped at 2^62, which also stands for "no bound": d = +inf, or w2_k = 0), and in windowed[k]
 * bit 0 where edtb200_transform_bounded's later pass along axis k (k >= 1) takes the window kernel
 * (R_k <= EDTB200_BOUNDED_WINDOW_MAX), bit 1 where edtb200_feature_transform_bounded's does
 * (R_k <= EDTB200_BOUNDED_SITES_WINDOW_MAX).  Entries k >= ndim are 0.
 * Checks, in order: ndim, sizes (as edtb200_transform), max_distance, pointers. */
int edtb200_bounded_plan(int ndim, int64_t sx, int64_t sy, int64_t sz,
                         float wx, float wy, float wz, double max_distance,
                         int64_t radius[3], int windowed[3]);

/* Spherical morphology of label volumes: erosion, dilation, opening and closing with the Euclidean
 * ball B = {v : sum_j (w_j v_j)^2 <= radius^2}, each a threshold on a bounded transform with
 * max_distance = radius.  "Within" is (double)d2 <= (double)radius * radius on the float32 squared
 * distance d2 as edtb200_transform computes it (+inf where there is no site): the rule of the bounded
 * transforms' cut and of expand_labels.  L is the labels, 0 background.
 *   EDTB200_ERODE  multi-label: p keeps L(p) iff L(p) != 0 and its edtsq (with black_border) is not
 *                  within radius; else 0.  Per label k: scipy binary_erosion(L == k, B,
 *                  border_value = black_border ? 0 : 1).
 *   EDTB200_OPEN   multi-label: with E the erosion above, p keeps L(p) iff L(p) != 0 and d2(p, E != 0)
 *                  is within radius, that transform without black_border; else 0.  Per label k:
 *                  binary_dilation(eroded_k, B, border_value = 0).  One transform of E opens every
 *                  label at once: the ball around E's voxel nearest p lies in that voxel's own label.
 *   EDTB200_DILATE binary: out[p] = 1 iff L(p) != 0 or |sdfsq(L)|(p) is within radius (no
 *                  black_border; black_border is ignored); binary_dilation(L != 0, B, border_value = 0).
 *   EDTB200_CLOSE  binary: D = the dilation above, then out[p] = 1 iff D(p) and the edtsq of D as a
 *                  two-label volume (with black_border) is not within radius: binary_erosion(D, B,
 *                  border_value = black_border ? 0 : 1).
 * radius 0 is the identity for erosion and opening; a voxel with no site at all (one label, no
 * black_border) is never within any radius.
 *
 *   labels   count * sx*sy*sz labels of label_bytes (1, 2, 4 or 8) bytes, volumes back to back as for
 *            edtb200_transform_stack (count 1: one volume), each transformed on its own
 *   flags    the residency flags, and EDTB200_LABELS_FLOAT for 4- / 8-byte IEEE labels: -0.0 is then
 *            background and compares equal to +0.0; every other value compares by its bits
 *   out      erode / open: count * sx*sy*sz labels of label_bytes, a kept voxel's bits copied exactly
 *            and every other voxel all-zero bits; dilate / close: count * sx*sy*sz bytes, 0 or 1.
 *            It must not overlap labels.
 * Residency, staging and asynchrony as edtb200_transform_bounded: host buffers are staged whole (there
 * is no chunked path; EDTB200_ENOMEM when they do not fit).  Each transform is the bounded transform's
 * passes with one launch per pass for the whole stack; the last store writes the labels or mask -- in
 * the window kernel where the last pass takes it (EDTB200_BOUNDED_WINDOW_MAX), else in one select kernel
 * after it.  Opening and closing run their two transforms back to back on one stream, the first writing
 * a 1-byte mask that the second transforms.  Device memory beyond the labels and out: 4 bytes per voxel
 * of distances, 4 more when a pass other than the last takes the window kernel, 1 for the mask of
 * opening and closing, and label_bytes for the folded labels with EDTB200_LABELS_FLOAT.
 * Checks, in order: label width, ndim, sizes (as edtb200_transform), count >= 0, op, radius (finite,
 * >= 0), flags, EDTB200_LABELS_FLOAT width, the stack's size (within 2^62 voxels), emptiness (returns 0
 * touching nothing), pointers, device. */
#define EDTB200_ERODE  0
#define EDTB200_DILATE 1
#define EDTB200_OPEN   2
#define EDTB200_CLOSE  3
int edtb200_morphology(const void *labels, int label_bytes, int ndim,
                       int64_t sx, int64_t sy, int64_t sz, int64_t count,
                       float wx, float wy, float wz, int op, double radius,
                       int black_border, int flags, void *out, int device, void *stream);

/* Local thickness of every label at once: for each labelled voxel, the radius of the largest ball of a
 * given ladder of levels that lies inside the voxel's own label and covers it (Hildebrand & Ruegsegger's
 * thickness is twice this value, BoneJ's included; porespy's local_thickness returns the radius).  For
 * labels L (0 is background), weights w, black_border and levels r_1 > ... > r_m of a volume:
 *   1. D2 = edtb200_transform's edtsq of L with black_border, bit for bit;
 *   2. the seeds of level r are S_r = { x : (double)D2(x) > r*r } -- exactly the voxels EDTB200_ERODE at
 *      radius r keeps; background has D2 = 0 and is never a seed;
 *   3. d2_r = the edtsq of the 1-byte mask that is 0 on S_r and 1 elsewhere, WITHOUT black border (the
 *      second transform of EDTB200_OPEN);
 *   4. out[p] = fl32(max{ r_i : L(p) != 0 and (double)d2_r_i(p) <= r_i*r_i }), and 0 where no level
 *      qualifies or L(p) == 0.
 * So out equals the maximum over i of (r_i where edtb200_morphology's EDTB200_OPEN at r_i is non-zero), bit
 * for bit: the ball around a seed lies inside the seed's own label, so one pass handles every label.
 * Exact Hildebrand thickness (every distinct D2 as a level) is not offered: each level costs a transform.
 *
 *   labels     count * sx*sy*sz labels of label_bytes (1, 2, 4 or 8) bytes, volumes back to back as for
 *              edtb200_transform_stack (count 1: one volume), each on its own
 *   wx..wz     the weights of the first ndim axes: finite and > 0
 *   flags      the residency flags, and EDTB200_LABELS_FLOAT for 4- / 8-byte IEEE labels (-0.0 is then
 *              background), as edtb200_morphology takes them
 *   sizes      a host array of nsizes radii, finite and >= 0, in any order and with repeats: the levels of
 *              every volume (sorted descending; a repeat is run once).  NULL: nsizes default levels per
 *              volume, computed on the device in double from R = sqrt(the largest finite D2 over the
 *              volume's labelled voxels) -- R = h/2 where there is none (no labelled voxel, or one label
 *              without black_border) -- and h = the least weight of the first ndim axes (a float):
 *                  r_i = (h/2) * (2R/h)^(i/n),  i = 0 .. n-1,  n = nsizes
 *              so every labelled voxel gets at least h/2 (it is its own seed) and the top level stays
 *              below R, which leaves it seeds.  pow may differ from another library's in the last bit:
 *              the result is defined relative to the levels sizes_out returns.
 *   nsizes     1 .. EDTB200_THICKNESS_MAX_SIZES
 *   out        count * sx*sy*sz float32 radii in the units of w; must not overlap labels
 *   sizes_out  NULL, or count * nsizes doubles on the side of out: the levels volume v used, descending, at
 *              sizes_out[v * nsizes ...] (repeats kept)
 * Residency, staging and asynchrony as edtb200_morphology: both sides on the device run asynchronously on
 * `stream` with no host wait, default levels included; host buffers are staged whole (EDTB200_ENOMEM when
 * they do not fit; there is no chunked path).  Kernels, on one stream, one launch per pass for the whole
 * stack: the edtsq (edtb200_transform's passes); with default levels a per-volume maximum of the finite
 * labelled D2 and one kernel that writes the levels and their float cuts B = the largest float32 whose
 * double is at most r*r to the device; then per level a seed kernel (D2 > B -> 0), the unbounded passes on
 * the mask, and a store that keeps the maximum (d2_r <= B -- the rule of the bounded transforms' cut, so
 * equal to them bit for bit).  Device memory beyond the labels and out: 9 bytes per voxel (D2, the mask,
 * its distances), label_bytes more with EDTB200_LABELS_FLOAT, 12 bytes per default level and volume plus 4
 * per volume, the staged levels of a host sizes_out, and the edtsq's own scratch where its plan takes it.
 * Checks, in order: label width, ndim, sizes (as edtb200_transform), count >= 0, weights, nsizes, each
 * radius (finite, >= 0), flags, EDTB200_LABELS_FLOAT width, the stack's size (within 2^62 voxels),
 * emptiness (returns 0 touching nothing), pointers (labels, out) and overlap (out with labels on the same
 * side; sizes_out with out, and with labels on the same side), device.  EDT_B200_VERBOSE=1 prints the
 * device time of the edtsq and of the levels on stderr. */
#define EDTB200_THICKNESS_MAX_SIZES 4096
int edtb200_local_thickness(const void *labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                            int64_t count, float wx, float wy, float wz, int black_border, int flags,
                            const double *sizes, int nsizes, float *out, double *sizes_out,
                            int device, void *stream);

/* Parabolic erosion and dilation of float volumes: the distance transform of a sampled function
 * (Felzenszwalb-Huttenlocher), ITK's ParabolicErode / DilateImageFilter.  Volumes are x-fastest, as
 * everywhere here.  Erosion: g0 = f as float32, then one pass per axis a in the order x, y, z:
 *     g_a(i) = min over j on i's line of cand(i, j)
 *     cand(i, i) = g_{a-1}(i)                                    (the sample itself, never w2 * 0)
 *     cand(i, j) = fl32(fl64(fl64(w2 * fl64((i-j)^2)) + fl64(g_{a-1}(j)))),  j != i
 *     w2 = fl64(fl32(w_a * w_a))
 * -- w2 rounded in float, the sum formed in double and rounded once to float32: what numpy computes in
 * float64 followed by .astype(np.float32).  Lines never cross the volume (nor one volume of a stack
 * into the next) and there are no border terms.  A NaN sample is read as +inf (never a site), -0.0 is
 * read and written as +0.0, so every zero result is +0.0.  When w_a * w_a overflows float32 (w2 = +inf)
 * every j != i candidate is +inf and the pass leaves its samples as they are; with a finite w2, a -inf
 * sample makes its whole line -inf.  Dilation is -erosion(-f), with the same NaN and zero rules.  The
 * result equals this definition bit for bit for every input.
 *
 * Uses: with integer weights, f = 0 on sites and +inf elsewhere gives the edtsq of the mask; a dilation
 * of r^2 (-inf off the medial points) gives the reverse distance transform, > 0 on the union of balls;
 * ITK's scale t is the weight spacing / sqrt(2 t).
 *
 *   f, out   count * sx*sy*sz float32, volumes back to back as for edtb200_transform_stack (count 1:
 *            one volume).  out == f is allowed (in place); any other overlap is EDTB200_EINVAL.
 *   wx..wz   the weights of the first ndim axes: finite and > 0 (the others are ignored)
 *   op       EDTB200_PARABOLIC_ERODE or EDTB200_PARABOLIC_DILATE
 *   flags    EDTB200_LABELS_ON_DEVICE (f is a device pointer) and EDTB200_OUT_ON_DEVICE only.  Both on
 *            the device: asynchronous on `stream`, no lock and no host wait.  Host buffers are staged
 *            whole through the device (there is no chunked path; EDTB200_ENOMEM when they do not fit).
 * One launch per pass for the whole stack; the first pass runs f -> out, the others in place on out.
 * Lines of at most 1024 samples take tile kernels that read and write every value once per pass and
 * need no device memory beyond f and out.  Longer lines of at most 23170 samples take a one-thread-
 * per-line hull with 8 bytes of device scratch per sample of the lines in flight (at most about 1 GiB);
 * longer lines than that take a brute-force minimum over every candidate (O(n^2) per line), which in
 * place needs a copy of the volume.  The hull is exact: its predicates fall back to exact expansion
 * arithmetic where a double evaluation cannot decide.
 * Checks, in order: ndim, sizes (as edtb200_transform), count >= 0, op, weights, flags, the stack's size
 * (within 2^62 voxels), emptiness (returns 0 touching nothing), pointers and overlap, device. */
#define EDTB200_PARABOLIC_ERODE  0
#define EDTB200_PARABOLIC_DILATE 1
int edtb200_parabolic(const float *f, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                      float wx, float wy, float wz, int op, int flags, float *out, int device, void *stream);

/* edtb200_parabolic with the minimising sample q of every voxel p (the maximising one for a dilation):
 * the seed of p's power (Laguerre) cell, the best placement of a part, the ball that decides p.
 *
 * Each pass a also picks a site s_a(i) on the line of every voxel i among its candidates (j = i
 * included, with the value g_{a-1}(i)):
 *   - lines of at most 23170 samples (tile kernels and the long-line hull): the least j among the REAL
 *     minimisers of w2 (i-j)^2 + g_{a-1}(j);
 *   - longer lines (the brute-force minimum): the least j among the minimisers of the double
 *     fl64(fl64(w2 * fl64((i-j)^2)) + g_{a-1}(j)), the candidate before its float32 rounding;
 *   - NaN and +inf samples are never sites; with a finite w2 a line holding -inf takes the least j with
 *     g_{a-1}(j) = -inf; with w2 = +inf s_a(i) = i; a voxel whose whole line is +inf or NaN has no site.
 * Rounding is monotone, so the value written is the site's own rounded candidate in both tiers.  A
 * dilation is the erosion of -f and so names the least maximiser.  The passes' sites compose as the
 * feature transform's: q_z = s_z(p), q_y = s_y at (p_x, p_y, q_z), q_x = s_x at (p_x, q_y, q_z).  A voxel
 * without a site gets -1 in every coordinate; its value is +inf (-inf for a dilation).  (A value can also
 * be +inf with a site, where a finite candidate rounds past the float32 range.)  So f(q) is finite or
 * +-inf at every q returned, and the value at p is the chain of rounded candidates from f(q): the X
 * pass's, then the Y pass's, then the Z pass's.
 *
 *   f, out, ..., flags, device, stream   as edtb200_parabolic; out is bit for bit its result
 *   idx   ndim x-fastest int32 planes of count * sx*sy*sz voxels, back to back: idx[0 .. V) the x
 *         coordinate, then y, then z (V = count * sx*sy*sz), each within its voxel's own volume.  It is on
 *         the device with EDTB200_OUT_ON_DEVICE, on the host otherwise, and must not overlap f or out.
 * Device memory beyond edtb200_parabolic's: the code planes of every pass but the last (4 bytes per voxel
 * each, so 8 in 3-D, 4 in 2-D and none in 1-D; the last pass writes its codes into its index plane), and
 * for a host idx the staged planes (4 ndim bytes per voxel).  With sites, X rows of 1009 to 1024 samples
 * take 2 warps per tile CTA instead of 4 (the codes need a second transpose buffer).
 * Checks, in order: as edtb200_parabolic up to the stack's size, then the line length (a line of more
 * than 2^26 samples is EDTB200_ELIMIT: beyond it (i-j)^2 is not exact in double), emptiness, pointers
 * (idx included) and overlap (idx with out, and with f when f is on the same side), device. */
int edtb200_parabolic_sites(const float *f, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                            float wx, float wy, float wz, int op, int flags, float *out,
                            int32_t *idx, int device, void *stream);

/* The medial axis of every label at once: the balls that rebuild each label exactly, the input of the
 * reverse distance transform (edtb200_parabolic's dilation of D^2 on the medial voxels, -inf elsewhere).
 * For labels L (0 is background) with weights w and black_border:
 *   1. D2 = edtb200_transform's edtsq of L (with black_border), bit for bit;
 *   2. (V, q) = edtb200_parabolic_sites' dilation of D2 as it is -- 0 on the background, not masked to
 *      -inf -- so q(p) is p's power (Laguerre) site, the maximiser of D2(y) - |p - y|^2_w;
 *   3. medial[y] = 1 iff y = q(p) for some voxel p with L(p) != 0.
 * The tie rule is edtb200_parabolic_sites': on lines of at most 23170 samples each pass takes the least j
 * among the REAL maximisers.  With integer weights and values below 2^24 nothing rounds, and q(p) is the
 * lexicographically least (z, y, x) among the real maximisers of D2(y) - |p - y|^2_w over the volume, x
 * the fastest axis in memory (so a caller's memory order decides which of tied maximisers is marked).  The
 * marked set is the reduced discrete medial axis (Coeurjolly & Montanvert, 2007): the balls B(y, D(y))
 * that are the power maximiser of at least one labelled voxel.  It is neither thin nor connected: not a
 * topological skeleton and not the minimal medial axis.
 *   reconstruction  for any weights, at every p with L(p) != 0, the dilation of (D2 on medial, -inf
 *                   elsewhere) equals V(p) bit for bit and is > 0: it is <= V(p) because every pass is
 *                   monotone, and >= the chain of rounded candidates from q(p), which is medial and, by the
 *                   sites' definition, gives V(p).
 *   integer weights the reconstruction is <= 0 on every background voxel, so "> 0" is exactly L != 0; q(p)
 *                   carries L(p); per label M the balls of M's medial voxels rebuild exactly the voxels of M,
 *                   so every non-empty label has a medial voxel.
 * Examples (1-D, background on both sides): a run of 5 has D2 = 1 4 9 4 1 and medial {2}; a run of 4 has
 * D2 = 1 4 4 1 and medial {1, 2}.  A volume of one non-zero label without black_border has D2 = +inf, and
 * its only medial voxel is its first one (a -inf line takes its first -inf position).
 *
 *   labels      count * sx*sy*sz labels of label_bytes (1, 2, 4 or 8) bytes, volumes back to back as for
 *               edtb200_transform_stack (count 1: one volume), each on its own; q(p) lies in p's volume
 *   wx..wz      the weights of the first ndim axes: finite and > 0
 *   flags       the residency flags (both on the device: asynchronous on `stream`, no lock and no host wait;
 *               host buffers are staged whole, EDTB200_ENOMEM when they do not fit -- there is no chunked
 *               path), and EDTB200_LABELS_FLOAT for 4- / 8-byte IEEE labels: -0.0 is then background and
 *               compares equal to +0.0, as in edtb200_morphology
 *   medial_out  count * sx*sy*sz bytes, 0 or 1
 *   dist_out    NULL, or count * sx*sy*sz float32: edt (sqrt of D2, correctly rounded), bit for bit
 *               edtb200_transform's with EDTB200_SQRT; on the same side as medial_out
 * Kernels, on one stream: the edtsq of the stack (one launch per pass, into dist_out or scratch), the
 * parabolic dilation with site codes (edtb200_parabolic_sites' instances; with distances the X pass runs
 * out of place from D2 into a value scratch, without them every pass runs in place over the D2 scratch;
 * the codes go to one plane per axis and no index plane is written), then the mask is zeroed and
 * medial_mark_kernel has every labelled voxel follow its codes to q(p) and store 1 there, taking the
 * square root of dist_out in the same pass.  Device memory beyond the labels and the outputs: 4 + 4 ndim
 * bytes per voxel (16 in 3-D: one value volume and ndim code planes; the folded labels of
 * EDTB200_LABELS_FLOAT live in the code planes until the edtsq has read them, so a 1-D call with 8-byte
 * float labels takes 4 + 8), plus the edtsq's long-line scratch where its plan takes that kernel, the
 * parabolic long-line hull on lines of 1025 to 23170 samples, and the staged host buffers.
 * Checks, in order: label width, ndim, sizes (as edtb200_transform), count >= 0, weights, flags,
 * EDTB200_LABELS_FLOAT width, the stack's size (within 2^62 voxels), the line length (a line of more than
 * 2^26 samples is EDTB200_ELIMIT, as for edtb200_parabolic_sites), emptiness (returns 0 touching nothing),
 * pointers (labels, medial_out) and overlap (neither output may overlap the labels when on the same side,
 * nor the other output), device.  EDT_B200_VERBOSE=1 prints each step's device time on stderr. */
int edtb200_medial_axis(const void *labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                        int64_t count, float wx, float wy, float wz, int black_border, int flags,
                        uint8_t *medial_out, float *dist_out, int device, void *stream);

/* Topology-preserving curve skeletons of every label at once, thinned in the order of the distance
 * transform, so that the skeleton is centred in physical units even on anisotropic voxels.
 * Terms.  Coordinates are taken within one volume (x the fastest axis in memory).  The voxels of a label
 * M are 26-connected (2-D: 8-); everything that is not M -- background, other labels, and the voxels
 * outside the volume -- is 6-connected (2-D: 4-).  All labels are thinned at once; deleting a voxel of M
 * never changes the topology of another label N, for which it was already "not N".
 *   simple     p of label M is simple iff the M-voxels of N26(p) \ {p} form exactly one 26-component
 *              and the non-M voxels of N18(p) \ {p} (6-connected within that set) have exactly one
 *              6-component that contains a 6-neighbour of p.  2-D: the M-pixels of N8(p) \ {p} form
 *              exactly one 8-component and the non-M pixels of N8(p) \ {p} have exactly one 4-component
 *              4-adjacent to p.
 *   end point  p of label M is an end point iff exactly one voxel of N26(p) \ {p} (2-D: N8) is of M.
 *   subfield   k = (x & 1) | (y & 1) << 1 | (z & 1) << 2 (2-D: (x & 1) | (y & 1) << 1).
 * Rounds.  R = edtb200_transform's edtsq of the labels (with black_border), float32, bit for bit; h = the
 * least weight of the first ndim axes; theta_t = (t h)^2 in double for t = 1, 2, ... (t below 2^53).
 * Round t admits the labelled voxels still present whose (double) R <= theta_t.  Rounds run up to the
 * first t with theta_t >= the largest finite R of a labelled voxel; then one final round admits every
 * voxel still present, R = +inf included (a label that touches the volume's edge without black_border).
 * A round that admits no new voxel changes nothing, and the kernel skips it.
 * Inside a round cycles repeat; a cycle runs the steps k = 0, 1, ..., 7 (2-D: 0 .. 3) in order, and step
 * k deletes, all at once, every present admitted voxel of subfield k that is simple on the image at the
 * start of the step and was not an end point at the start of the CYCLE.  The round ends after the first
 * cycle that deletes nothing.  The skeleton is the set of voxels present after the final round.  No two
 * voxels of one subfield are 26-neighbours, so a step equals any sequential order of its deletions.
 *   topology   each label keeps its number of 26-components (2-D: 8-), the number of 6-components of its
 *              complement (2-D: 4-) and its Euler characteristic, so also its cavities and tunnels.
 *   thinness   no voxel of the result is simple and not an end point.
 *   order      the result depends on which axis is fastest in memory, through the subfield order: an
 *              F-ordered array gives the C-ordered call on its transpose with the weights reversed, and
 *              the same labels in the two orders can give different, equally valid skeletons.
 * Examples: a straight line one voxel thick is its own skeleton; an isolated voxel stays; a 3x3x3 cube
 * in background gives exactly its centre; a hollow spherical shell keeps a closed surface around its
 * cavity; a 4x6x12 box (z, y, x) in background gives the line x = 4 .. 10 at (z, y) = (3, 4) of the box
 * padded by one voxel, along its long axis; a 2-D disc of radius 6 gives its centre pixel.
 *
 *   labels        count * sx*sy*sz labels of label_bytes (1, 2, 4 or 8) bytes, integers (no float
 *                 labels), volumes back to back as for edtb200_transform_stack (count 1: one volume),
 *                 each thinned on its own
 *   ndim          2 or 3; wx..wz the weights of the first ndim axes: finite and > 0
 *   flags         the residency flags only (both on the device: asynchronous on `stream`, no lock and no
 *                 host wait; host buffers are staged whole, EDTB200_ENOMEM when they do not fit -- there
 *                 is no chunked path)
 *   skeleton_out  count * sx*sy*sz bytes, 0 or 1
 *   dist_out      NULL, or count * sx*sy*sz float32: edt (sqrt of R, correctly rounded), bit for bit
 *                 edtb200_transform's with EDTB200_SQRT; on the same side as skeleton_out
 * Kernels, on one stream: the edtsq of the stack (one launch per pass, into dist_out or scratch), then
 * ONE cooperative launch of skeleton_thin_kernel, which runs every round, cycle and step with a grid
 * barrier between them: a sweep per round admits voxels into a compact list with one segment per
 * subfield, each cycle's first pass drops the deleted entries and the end points (an end point at the
 * start of a cycle can never be deleted later, so it is retired for good), each step tests only its
 * segment, and the last sweep writes the skeleton and the square roots.  Device memory beyond the labels
 * and the outputs: 4 + 8 bytes per voxel for volumes of even sides (12 in 2-D and 3-D; 8 with dist_out,
 * which holds R): R (4, without dist_out) and two list buffers of one 4-byte entry per voxel (a segment
 * holds count * ceil(sx/2) * ceil(sy/2) * ceil(sz/2) entries); the state byte of each voxel lives in
 * skeleton_out's device buffer.  The lists are taken after the edtsq has returned its long-line scratch
 * (where its plan takes that kernel), so the two do not add up; plus the staged host buffers.
 * Checks, in order: label width, ndim, sizes (as edtb200_transform), ndim of 2 or 3, count >= 0, weights,
 * flags, the stack's size (within 2^62 voxels), a subfield's size (below 2^32 voxels, else
 * EDTB200_ELIMIT), emptiness (returns 0 touching nothing), pointers (labels, skeleton_out) and overlap
 * (neither output may overlap the labels when on the same side, nor the other output), device.
 * EDT_B200_VERBOSE=1 prints the edtsq's and the thinning's device times, and the rounds, cycles and
 * steps run, on stderr. */
int edtb200_skeletonize(const void *labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                        int64_t count, float wx, float wy, float wz, int black_border, int flags,
                        uint8_t *skeleton_out, float *dist_out, int device, void *stream);

/* Geodesic distance: the length of the shortest path from a seed to each voxel that stays inside the
 * voxel's own label (connectomics path lengths, seed splitting of touching objects, geodesic maps from clicks,
 * tortuosity).  Volumes are x-fastest, as everywhere here; coordinates are taken within one volume.
 *   graph     every voxel with a non-zero label is a node; two nodes are joined when they are 26-neighbours
 *             (2-D: 8, 1-D: 2) with the SAME label.  Label 0 and the outside of the volume cannot be crossed
 *             (there is no black_border).  A step (dx, dy, dz), each in {-1, 0, 1}, has the length
 *             w = sqrt((dx*wx)^2 + (dy*wy)^2 + (dz*wz)^2): each (float) weight promoted to double, the squares summed
 *             in double in the order x, y, z, the square root correctly rounded.  The host forms the 7
 *             distinct lengths (one per non-zero (|dx|, |dy|, |dz|)) once; no device code forms a weight.
 *   seeds     a voxel is a seed when its seed value AND its label are non-zero (seeds on background are
 *             ignored).
 *   distance  D is the least fixed point of D[v] = min(D[v], fl64(D[u] + w(u, v))) over the graph neighbours u
 *             of v, from D = 0 on the seeds and +inf elsewhere -- what Dijkstra computes in double.  dist_out
 *             = float32(D), rounded once to nearest; label-0 voxels and voxels with no seed in their component
 *             get +inf.
 *   indices   S[v] is the least linear seed index c (x-fastest within the volume) with a TIGHT path c = u0 ..
 *             uk = v: every step has D[u_{i+1}] == fl64(D[u_i] + w).  Deterministic, independent of the order of
 *             evaluation.  idx_out holds S as ndim int32 coordinate planes laid out like the labels (idx_out[0]
 *             the x coordinate, idx_out[1] y, idx_out[2] z), -1 in every plane where D is +inf.
 * Examples: along a straight one-voxel corridor D is the number of steps times its axis weight; in an
 * L-shaped corridor D at the far end is the sum of both legs, larger than the edt's straight line.
 *
 *   labels, label_bytes  count * sx*sy*sz labels of 1, 2, 4 or 8 bytes (integers: compared by their bits),
 *                        volumes back to back as for edtb200_transform_stack (count 1: one volume)
 *   seeds, seed_bytes    count * sx*sy*sz values of 1, 2, 4 or 8 bytes, laid out like the labels and on the
 *                        same side (EDTB200_LABELS_ON_DEVICE covers both)
 *   wx..wz               the weights of the first ndim axes: finite and > 0
 *   flags                the residency flags only (both on the device: asynchronous on `stream`, no lock and
 *                        no host wait; host buffers are staged whole, EDTB200_ENOMEM when they do not fit --
 *                        there is no chunked path)
 *   dist_out             count * sx*sy*sz float32
 *   idx_out              NULL, or ndim pointers to count * sx*sy*sz int32 planes on the side of dist_out
 * Kernels, on one stream.  The distances: a seed kernel writes D as doubles (0 / +inf) and queues the tiles
 * that hold a seed; then ONE cooperative launch of geodesic_relax_kernel runs every round with a grid barrier
 * between them.  Tiles are 8x8x8 voxels (2-D 16x16, 1-D 256).  A round's CTAs each take tiles of the
 * worklist, stage a tile and a one-voxel halo of D and labels in shared memory, relax it in sweeps until a
 * sweep lowers nothing, write back the voxels that went down, and queue each neighbour tile (up to 26) that a
 * lowered voxel on a face, edge or corner touches (in round 1, whose tiles are those the seed kernel queued,
 * the seeds count as lowered, so a seed on a tile's border reaches past it); a per-tile flag holding the round it is queued for makes
 * each list hold a tile at most once.  The rounds end when one queues nothing.  A halo value read while its
 * owner writes it is an 8-byte load, never torn; D only decreases, so a stale value is an upper bound and the
 * owner's write queues the reader again.  Termination follows from monotone decrease over finitely many
 * doubles; there is no round cap.  With idx_out the same rounds then run on S with D fixed: S starts at the
 * seed's own index and relaxes by min over tight edges only, evaluated with the same double add.  A store
 * kernel writes float32(D) and the coordinate planes.  The rounds grow with how often shortest paths turn
 * across tile boundaries: a handful for a convex object, thousands for a maze.
 * Device memory beyond the labels, seeds and outputs: 8 bytes per voxel for D, 8 more for S with idx_out,
 * 12 bytes per tile (its flag and its entries in the two worklists), 64 bytes of control blocks, and the
 * staged seeds and index planes of a host call.
 * Checks, in order: label width, seed width, ndim and sizes (as edtb200_transform), count >= 0, weights,
 * flags, the stack's size (within 2^62 voxels, so that a linear seed index fits S's 8 bytes), its tiles
 * (fewer than 2^32, else EDTB200_ELIMIT: the worklists hold 4-byte tile numbers), emptiness (returns 0
 * touching nothing), pointers (labels, seeds, dist_out, and each of the ndim planes when idx_out is given),
 * overlaps (no output may overlap the labels or seeds when on the same side, nor another output), device.
 * EDT_B200_VERBOSE=1 prints the device time of the distances, indices and store, and the rounds and tile
 * visits of each phase, on stderr. */
int edtb200_geodesic(const void *labels, int label_bytes, const void *seeds, int seed_bytes, int ndim,
                     int64_t sx, int64_t sy, int64_t sz, int64_t count, float wx, float wy, float wz,
                     int flags, float *dist_out, int32_t *const *idx_out, int device, void *stream);

/* Watershed: marker-controlled flooding of an altitude image inside each label (splitting touching objects:
 * markers at the maxima of edt(mask), then the watershed of -edt).  Volumes are x-fastest, as everywhere here.
 *   graph     every voxel with a non-zero label is a node (label_bytes 0: every voxel, all with one label);
 *             two nodes are joined when they are neighbours under `connectivity` with the SAME label: an
 *             offset in {-1, 0, 1}^ndim counts when at most `connectivity` of its components are non-zero
 *             (3-D 1/2/3: 6/18/26 neighbours, 2-D 1/2: 4/8, 1-D 1: 2), as in scipy and skimage.  Label 0 and
 *             the outside of the volume cannot be crossed.
 *   altitude  f = image as float32, NaN read as +inf and -0.0 as +0.0; +inf and -inf are valid altitudes.
 *   seeds     a voxel is a seed when its marker AND its label are non-zero (markers on label 0 are ignored).
 *             Marker values are compared as unsigned integers of marker_bytes.
 *   level     L is the least fixed point of L[v] = min(L[v], max(f[v], L[u])) over the graph neighbours u of
 *             v, from f on the seeds and +inf elsewhere: the lowest flood level at which water from some seed
 *             reaches v.  min and max round nothing, so L is exact.
 *   result    an edge u -> v is TIGHT when v is not a seed and L[v] == max(f[v], L[u]).  W[s] = marker[s] on
 *             the seeds; elsewhere W[v] is the least marker m with a tight path from a seed of marker m to
 *             v whose voxels after the first are non-seeds, and 0 where there is none and on label 0.
 *             Deterministic, independent of the order of evaluation, also on plateaus.  Ties (a voxel reached
 *             at the same level from two markers) go to the smaller marker; plateaus are not split by
 *             distance.
 *
 *   labels, label_bytes    count * sx*sy*sz labels of 1, 2, 4 or 8 bytes (integers: compared by their bits),
 *                          volumes back to back as for edtb200_transform_stack; label_bytes 0: no labels
 *                          (labels is not read)
 *   markers, marker_bytes  count * sx*sy*sz markers of 1, 2, 4 or 8 bytes, laid out like the volume
 *   image                  count * sx*sy*sz float32 altitudes, laid out like the volume
 *   connectivity           1 to ndim
 *   flags                  the residency flags only (EDTB200_LABELS_ON_DEVICE covers every input; both on
 *                          the device: asynchronous on `stream`, no lock and no host wait; host buffers are
 *                          staged whole, EDTB200_ENOMEM when they do not fit -- there is no chunked path)
 *   out                    count * sx*sy*sz markers of marker_bytes: W
 *   level_out              NULL, or count * sx*sy*sz float32 on the side of out: L (+inf on label 0)
 * Kernels, on one stream, on the tiles and worklists of edtb200_geodesic (8x8x8 voxels, 2-D 16x16, 1-D 256).
 * The levels: a seed kernel writes L (f / +inf) and queues the tiles that hold a seed; then ONE cooperative
 * launch of watershed_relax_kernel runs every round with a grid barrier between them.  A round's CTAs each
 * stage a tile and a one-voxel halo of L and labels in shared memory, relax it in sweeps of min over the
 * neighbours of max(f[v], L[u]) until a sweep lowers nothing, write back the voxels that went down and queue
 * each neighbour tile that a lowered voxel on a face, edge or corner touches through the connectivity (in
 * round 1 the seeds count as lowered, so a seed on a tile's border reaches past it).  The labels: the same
 * rounds on W = marker - 1 (all ones: none) with L fixed, by min over the tight edges, queued on changes of W
 * (a voxel of altitude +inf has L = +inf and can still take a W); the seeds are never written.  A store kernel
 * writes W in the markers' width and L.  Every halo read is an aligned 4- or 8-byte load (W is 4 bytes for
 * markers of up to 4 bytes, 8 for 8-byte markers), never torn; values only decrease, so a stale value is an
 * upper bound and the owner's write queues the reader again; there is no round cap.
 * Device memory beyond the inputs and outputs: 4 bytes per voxel for L, 4 for W (8 with 8-byte markers),
 * 12 bytes per tile, 64 bytes of control blocks, and the staged markers, image and result of a host call.
 * Checks, in order: label width, marker width, ndim and sizes (as edtb200_transform), count >= 0,
 * connectivity, flags, the stack's size (within 2^62 voxels), its tiles (fewer than 2^32, else
 * EDTB200_ELIMIT: the worklists hold 4-byte tile numbers), emptiness (returns 0 touching nothing), pointers
 * (labels unless label_bytes is 0, markers, image, out), overlaps (no output may overlap an input when on the
 * same side, nor the other output), device.
 * EDT_B200_VERBOSE=1 prints the device time of the levels, labels and store, and the rounds and tile visits
 * of each phase, on stderr. */
int edtb200_watershed(const void *labels, int label_bytes, const void *markers, int marker_bytes,
                      const float *image, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                      int connectivity, int flags, void *out, float *level_out, int device, void *stream);

/* Connected components and extended maxima (the markers of a watershed split: dist = edt(mask), markers =
 * extended_maxima(dist, h), watershed(-dist, markers, mask)).  Volumes are x-fastest, as everywhere here.
 *   graph      the watershed's: every voxel with a non-zero label is a node (label_bytes 0, extended_maxima
 *              only: every voxel, all with one label); two nodes are joined when they are neighbours under
 *              `connectivity` with the SAME label: an offset in {-1, 0, 1}^ndim counts when at most
 *              `connectivity` of its components are non-zero.  Label 0 and the outside of the volume cannot be
 *              crossed.
 *   numbering  each component is numbered 1..n in increasing order of its least voxel index in memory order,
 *              everything else 0; each volume of a stack is numbered on its own from 1.  For a C-ordered array
 *              this is scipy.ndimage.label's numbering.
 *
 * edtb200_connected_components: the components of the graph, numbered.
 * edtb200_extended_maxima: the regional maxima of the h-maxima transform (Soille's EMAX_h):
 *   f = image, NaN read as -inf and -0.0 as +0.0; h finite and >= 0; m = fl32(fl64(f) - h), -0.0 as +0.0.
 *   R is the least fixed point of R[v] = max(R[v], min(f[v], R[u])) over the joined neighbours u of v, from m:
 *   the reconstruction by dilation of m under f, exact because min and max round nothing (h = 0: R = f).
 *   A plateau is a component of the graph restricted to the edges with R[u] == R[v]; it is a maximum when no
 *   node in it has a joined neighbour of larger R and its R is not -inf.  The result is the maximum plateaus,
 *   numbered.  When f - h is exact in float32, a peak survives exactly when its dynamic (its height above the
 *   highest pass to a higher voxel of its label) exceeds h.
 *
 *   labels, label_bytes  count * sx*sy*sz labels of 1, 2, 4 or 8 bytes (integers: compared by their bits),
 *                        volumes back to back as for edtb200_transform_stack; label_bytes 0: no labels
 *                        (extended_maxima only; labels is not read)
 *   image                count * sx*sy*sz float32, laid out like the volume
 *   connectivity         1 to ndim
 *   flags                the residency flags only (EDTB200_LABELS_ON_DEVICE covers every input; both on the
 *                        device: asynchronous on `stream`, no lock and no host wait; host buffers are staged
 *                        whole, EDTB200_ENOMEM when they do not fit -- there is no chunked path)
 *   out, out_bytes       count * sx*sy*sz numbers of 4 bytes (int32; volumes of fewer than 2^31 voxels) or 8
 * Kernels, on one stream (edt_components.cuh).  Parents are 4-byte indices within a volume.  A tile pass
 * (one CTA per 16x8x8 tile, 2-D 32x32, 1-D 1024) runs union-find on the tile's keys in shared memory; a border
 * pass joins the joined edges that leave a tile by lock-free union in global memory, always hanging the larger
 * root under the smaller (atomicMin), so that the final root of every component is its least index whatever
 * order the races take; a flatten pass points every voxel at its root and flags the roots in out; for the
 * plateaus a mark pass drops the root of every plateau with a larger joined neighbour or R = -inf; a prefix
 * sum in place over out (cub::DeviceScan, per volume) and a number pass copy each kept root's number to its
 * component.  For h > 0, R comes first from the level phase of edtb200_watershed on negated values
 * (altitude -f, every node seeded at -m), on its tiles and worklists.
 * Device memory beyond the inputs and outputs: 4 bytes per voxel of parents and the scan's scratch (8 bytes
 * per volume of a stack and cub's); with h > 0 another 4 + 4 bytes per voxel (-R and -f) and 12 bytes per
 * tile; and the staged image and result of a host call.
 * Checks, in order: label width (extended_maxima also takes 0), ndim and sizes (as edtb200_transform),
 * count >= 0, h (extended_maxima: finite and >= 0), connectivity, flags, out_bytes (4 or 8), the stack's size
 * (within 2^62 voxels), the volume's size (fewer than 2^32 voxels, else EDTB200_ELIMIT), out_bytes 4 with a
 * volume of 2^31 voxels or more (EDTB200_EINVAL), for extended_maxima with h > 0 the tiles (fewer than 2^32,
 * else EDTB200_ELIMIT), emptiness (returns 0 touching nothing), pointers (labels unless label_bytes is 0,
 * image, out), overlaps (out may not overlap an input on the same side), device.
 * EDT_B200_VERBOSE=1 prints the device time of the reconstruction (with its rounds and tile visits), the
 * union, the flatten and mark, and the numbering, on stderr. */
int edtb200_connected_components(const void *labels, int label_bytes, int ndim, int64_t sx, int64_t sy,
                                 int64_t sz, int64_t count, int connectivity, int flags, void *out,
                                 int out_bytes, int device, void *stream);
int edtb200_extended_maxima(const void *labels, int label_bytes, const float *image, int ndim, int64_t sx,
                            int64_t sy, int64_t sz, int64_t count, double h, int connectivity, int flags,
                            void *out, int out_bytes, int device, void *stream);

/* Hole filling and dust removal: decide per component, then write every voxel.  Volumes are x-fastest, as
 * everywhere here.  The graph and `connectivity` are connected_components': an offset in {-1, 0, 1}^ndim
 * counts when at most `connectivity` of its components are non-zero.  Labels compare by their bits.
 *
 * edtb200_fill_holes: every hole of a label L takes L.
 *   background component  a component of the label-0 voxels under `connectivity`; all background
 *                         neighbours are joined.
 *   open                  it contains a voxel on a face of its volume (in a stack each volume has its own
 *                         faces).
 *   bordering labels      the non-zero labels of the voxels that neighbour it under `connectivity`.
 *   hole of L             a background component that is not open, whose only bordering label is L, and, when
 *                         max_size >= 0, that has at most max_size voxels.
 *   result                the labels with every hole of L set to L; everything else unchanged.  For one label
 *                         this is scipy.ndimage.binary_fill_holes with generate_binary_structure(ndim,
 *                         connectivity).  A background gap bordered by two labels (the gap between a cell and
 *                         a nucleus inside it) stays 0.
 *   fill_counts           NULL, or count int64: the voxels filled in each volume, on the side of out.
 * edtb200_dust: every component (same label, joined under `connectivity`) of fewer than `threshold` voxels is
 *   set to 0; with invert = 1 only those components are kept and every other labelled voxel is set to 0.
 *
 *   labels, label_bytes  count * sx*sy*sz labels of 1, 2, 4 or 8 bytes, volumes back to back as for
 *                        edtb200_transform_stack
 *   connectivity         1 to ndim
 *   max_size             fill_holes: -1 (no bound) or >= 0
 *   threshold, invert    dust: threshold >= 0 (0 keeps everything), invert 0 or 1
 *   flags                the residency flags only (EDTB200_LABELS_ON_DEVICE covers the labels; both on the
 *                        device: asynchronous on `stream`, no lock and no host wait; host buffers are staged
 *                        whole, EDTB200_ENOMEM when they do not fit -- there is no chunked path)
 *   out                  count * sx*sy*sz labels of label_bytes; it may not overlap the labels (no in-place call)
 * Kernels, on one stream (edt_holes.cuh).  The union is the tile and border passes of
 * edtb200_connected_components (edt_components.cuh): with the label key for dust, and for fill_holes with a
 * key whose nodes are the label-0 voxels inside the volume, all joined.  A tally pass (one thread per voxel)
 * points every node at its root and adds it to its root's 4-byte size, one atomic per run of equal roots in a
 * warp; for fill_holes a node on a face sets an OPEN bit at its root, and a node with a neighbour of label
 * L != 0 claims L at its root by atomicCAS(claim, 0, L) (4 bytes, 8 for 8-byte labels), setting a MIXED bit
 * when the CAS returns another label.  Sums, ORs and "the claimed labels are one" do not depend on the order
 * of the races.  An apply pass (one thread per voxel) writes out, and counts the filled voxels per volume by
 * a block reduction and one atomic per block.
 * Device memory beyond the inputs and outputs: 4 bytes per voxel of parents; 4 bytes per voxel of sizes for
 * dust and for fill_holes with max_size >= 0; for fill_holes 4 bytes per voxel of claims (8 with 8-byte
 * labels) and 1 byte per voxel of state; and the staged labels, result and fill counts of a host call.
 * Checks, in order: label width, ndim and sizes (as edtb200_transform), count >= 0, connectivity, max_size
 * (fill_holes) or threshold and invert (dust), flags, the stack's size (within 2^62 voxels), the volume's
 * size (fewer than 2^32 voxels, else EDTB200_ELIMIT), emptiness (returns 0 touching nothing, fill_counts
 * included), pointers (labels, out), overlaps (out may not overlap the labels on the same side; fill_counts
 * may overlap neither), device.
 * EDT_B200_VERBOSE=1 prints the device time of the union, the tally and the apply on stderr. */
int edtb200_fill_holes(const void *labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                       int64_t count, int connectivity, int64_t max_size, int flags, void *out,
                       int64_t *fill_counts, int device, void *stream);
int edtb200_dust(const void *labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                 int64_t count, int connectivity, int64_t threshold, int invert, int flags, void *out,
                 int device, void *stream);

/* The k nearest distinct labels of every voxel within a distance: which objects are near p, and how far
 * away each is (the d1, d2 of the U-Net weight map w0 exp(-(d1 + d2)^2 / 2 sigma^2), contacts between
 * segments, Voronoi boundaries where d2 - d1 is small).
 *
 * Sites: every voxel with a non-zero label is a site of that label; label 0 is background, whose voxels
 * ask the query but are never sites.  There is no border term.  For a voxel p and a label M,
 *     D_M(p) = edtb200_parabolic's erosion of (0 on the voxels of M, +inf elsewhere) at p, bit for bit:
 * one pass per axis in the order x, y, z, each candidate fl32(fl64(w2 (i-j)^2) + fl64(g(j))) with
 * w2 = fl64(fl32(w * w)).  With integer weights and values below 2^24 it is exactly the squared distance
 * from p to the nearest voxel of M.  B is the largest float32 with (double)B <= (double)d * d, the B of the
 * bounded transforms; only labels with D_M(p) <= B count.
 *   values  the k distances of p, ascending, are the k smallest D_M(p) over the distinct counted labels M;
 *           where fewer than k labels count, the missing entries are +inf with label 0.
 *   labels  are fixed by the per-pass rule: the X pass sees the voxel itself at 0 (when its label is
 *           non-zero) and each site j != i within its window at fl32(w2 (i-j)^2); every later pass sees its
 *           own row's list unchanged and row j's entries each as fl32(fl64(w2 (i-j)^2) + fl64(v)); each pass
 *           keeps per voxel the k least (value, label) pairs with distinct labels -- a label keeps its least
 *           value, ties are ordered by the label read as an unsigned integer of its width, pairs above B are
 *           dropped -- and stores them in that order.  So the labels are the k least (D_M(p), M) pairs
 *           wherever no rounding merges two candidates, which always holds for integer weights with values
 *           below 2^24; otherwise a label can differ only among labels whose value equals the k-th value.
 * The values are exact because the per-pass truncation is: a label B dropped at an intermediate voxel q on
 * the path of its least value at p had k other labels no larger at q, and each pass adds w2 d^2 and rounds,
 * which is monotone, so those k are no larger at p either.  A voxel of label A has entry 0 = (0, A).
 *
 *   labels     count * sx*sy*sz labels of label_bytes (1, 2, 4 or 8) bytes, volumes back to back as for
 *              edtb200_transform_stack (count 1: one volume), each on its own
 *   wx..wz     the weights of the first ndim axes: finite and > 0
 *   max_distance  d, finite and >= 0: the cost is O(R) per voxel per pass, so there is no unbounded call
 *   k          1 to 4
 *   flags      the residency flags (both on the device: asynchronous on `stream`; host buffers are staged
 *              whole, EDTB200_ENOMEM when they do not fit -- there is no chunked path) and
 *              EDTB200_NEAREST_SQUARED: the values D; without it sqrtf of each, correctly rounded, as edt
 *   dist_out   k x-fastest float32 planes of count * sx*sy*sz voxels, back to back (entry q of every voxel
 *              is plane q)
 *   label_out  k planes of labels of label_bytes, laid out as dist_out; neither output may overlap the
 *              other or the labels
 * Kernels: the X pass stages runs of voxels with R_x labels either side in shared memory; each later pass
 * walks a window of R_a rows either side with lanes on 32 adjacent lines, staged in shared memory when
 * (64 + 2 R_a) 32 k (4 + label_bytes) bytes fit the 227 KB of a CTA and read from global memory otherwise
 * (equal bit for bit).  R_a is the bounded transforms' radius (edtb200_bounded_plan) and may not exceed
 * 256 rows.  The passes write out of place: 3-D X -> out, Y -> scratch, Z -> out; 2-D X -> scratch,
 * Y -> out; 1-D X -> out.  So the device memory beyond the labels and the outputs is k (4 + label_bytes)
 * bytes per voxel in 2-D and 3-D, and none in 1-D.
 * Checks, in order: label width, ndim, sizes (as edtb200_transform), count >= 0, weights, k, max_distance,
 * a pass radius above 256 (EDTB200_ELIMIT), flags, the stack's size (within 2^62 values), emptiness
 * (returns 0 touching nothing), pointers and overlap, device. */
#define EDTB200_NEAREST_SQUARED 32
int edtb200_nearest_labels(const void *labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                           int64_t count, float wx, float wy, float wz, double max_distance, int k, int flags,
                           float *dist_out, void *label_out, int device, void *stream);

/* The plan of edtb200_nearest_labels, pure host logic (no device needed): radius[a] = R_a, the bounded
 * transforms' rule (the largest r with (double)w2_a r^2 < nextafterf(B, +inf), as edtb200_bounded_plan
 * gives it), and variant[a] the kernel of the pass along axis a: EDTB200_NEAREST_ROWS (the X pass),
 * EDTB200_NEAREST_STAGED or EDTB200_NEAREST_GLOBAL (a later pass with its window in shared memory or read
 * from global memory), -1 for an axis a >= ndim (radius 0) or a radius above 256, which the call refuses.
 * Checks, in order: as edtb200_nearest_labels up to max_distance, then the pointers. */
#define EDTB200_NEAREST_ROWS   0
#define EDTB200_NEAREST_STAGED 1
#define EDTB200_NEAREST_GLOBAL 2
int edtb200_nearest_labels_plan(int ndim, int64_t sx, int64_t sy, int64_t sz, float wx, float wy, float wz,
                                double max_distance, int k, int label_bytes, int64_t radius[3], int variant[3]);

/* A stack of `count` volumes of one geometry (sx, sy, sz), laid back to back (volume b starts at
 * voxel b * sx * sy * sz), each transformed on its own as edtb200_transform would: its result is
 * that call's bit for bit.  No line crosses from one volume into the next, black_border applies to
 * every volume's own faces, and every pass keeps one volume's extents for its arithmetic.  Each pass
 * is ONE launch over the whole stack (the X pass over count * sy * sz rows; the Y pass walks
 * count * sz slices; the Z pass walks the volumes), so many small volumes cost what one volume of
 * their total size costs -- for example the 2-D transform of every z slice of an anisotropic stack
 * (ndim 2, count = depth), or a batch of masks of a training step.
 *
 *   labels, out   count * sx*sy*sz labels / float32; BOTH on the device (EDTB200_LABELS_ON_DEVICE |
 *                 EDTB200_OUT_ON_DEVICE) or both on the host: mixed residency is EDTB200_EINVAL
 *   flags         EDTB200_SQRT / EDTB200_SIGNED and the residency flags
 *   device_bytes  host buffers only (ignored on the device): the budget B of the call's device memory,
 *                 0 = the memory free on the device less EDTB200_CHUNK_RESERVE
 *   groups        NULL, or int64_t[1] that receives the number of groups the call ran (1 on the device;
 *                 0 on an error or an empty stack)
 * On the device the call is asynchronous on `stream` and takes no lock.  Host buffers go through the
 * device in groups of whole volumes, pipelined through two device slots as edtb200_transform_batch
 * pipelines its volumes, planned as one phase of edtb200_transform_chunked whose slices are volumes:
 * a volume costs V (label_bytes + 4 + s) bytes, s = 8 when a later pass takes the long-line kernel
 * (its two scratch volumes); a group holds at most 512 MiB of those bytes (at least one volume), so
 * that the copies of one group overlap the passes of the next; one group when the whole stack fits B
 * and that cap, else two slots of min(cap, floor(B / (2 * that))) volumes each; EDTB200_ENOMEM when
 * not even one volume fits, and the message names the least budget that works.  On label noise the X pass may also take the run-start planes of
 * at most 1/4 byte per voxel outside the budget (none when there is no room).  The device's cached
 * whole-volume buffers are freed first, as edtb200_transform_chunked does, and the host call returns
 * when every result has landed; labels and out must not overlap.
 * Checks, in order: label width, ndim, sizes (as edtb200_transform), count >= 0, emptiness (count 0 or
 * an empty volume returns 0 touching nothing), pointers, residency, overlap, device. */
int edtb200_transform_stack(const void *labels, int label_bytes, int ndim,
                            int64_t sx, int64_t sy, int64_t sz, int64_t count,
                            float wx, float wy, float wz,
                            int black_border, int flags, float *out,
                            int device, size_t device_bytes, int64_t *groups, void *stream);

/* edtb200_feature_transform of a stack of `count` volumes laid back to back, as for
 * edtb200_transform_stack: each volume on its own, one launch per pass for the whole stack.  Every
 * plane (idx_out[k], dist_out) covers the whole stack, and the coordinates are those within the
 * voxel's own volume (a face site is -1 or n on its axis of that volume; no site is -1 everywhere).
 * Residency and device memory as edtb200_feature_transform, for count * sx*sy*sz voxels: host buffers
 * are staged in one shot, with no grouping and no chunking. */
int edtb200_feature_transform_stack(const void *labels, int label_bytes, int ndim,
                                    int64_t sx, int64_t sy, int64_t sz, int64_t count,
                                    float wx, float wy, float wz,
                                    int black_border, int flags, float *dist_out,
                                    int32_t *const *idx_out, int device, void *stream);

/* expand_labels' gather (skimage.segmentation.expand_labels): every background voxel whose nearest
 * labelled voxel lies within the limit takes that voxel's label, every other voxel keeps its own.
 * The inputs are what edtb200_feature_transform_stack (or edtb200_feature_transform, count 1) returns
 * with EDTB200_SIGNED, without EDTB200_SQRT and without black_border, for `count` volumes of
 * (sx, sy, sz) laid back to back (volume b starts at voxel b * sx * sy * sz).
 *   labels   count * sx*sy*sz labels of `label_bytes` (1, 2, 4 or 8) bytes, as given to that transform
 *            but with float labels left as they are (not canonicalised)
 *   sqdist   the transform's float32 squared distances (signed: negative on background)
 *   idx      ndim int32 planes, idx[0] x, idx[1] y, idx[2] z: every voxel's site within its own
 *            volume, idx[0] -1 where there is none
 *   limit_sq the squared limit: a background voxel p grows iff idx[0][p] >= 0 and
 *            (double)|sqdist[p]| <= limit_sq.  A caller with a distance d passes d * d, so a negative d
 *            acts as |d|, NaN grows nothing and +inf grows every voxel that has a site.  A site
 *            outside its volume (a face position of a black_border transform) grows nothing.
 *   flags    EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE (every buffer is on `device`: host
 *            buffers are not accepted), optionally with EDTB200_LABELS_FLOAT
 *   out      count * sx*sy*sz labels; the grown volume.  It may be `labels` itself (in place).
 * Background is a label whose bits are all zero; with EDTB200_LABELS_FLOAT (4- / 8-byte IEEE labels)
 * a label whose value is zero, so -0.0 is background too.  Labels are copied as raw bits: -0.0 and
 * NaN payloads survive exactly.  In place is exact because only background voxels change, and a
 * background voxel reads only its own label and its site's, which is always a labelled voxel.
 * One launch, asynchronous on `stream`, no lock, no allocation; it reads each input once: the
 * labels, and for background voxels their first plane, and only where they have a site their
 * distance, and only where they grow the other planes and the site's label.
 * Checks, in order: label width, ndim, sizes (as edtb200_transform), count >= 0, emptiness (count 0
 * or an empty volume returns 0 touching nothing), pointers (labels, sqdist, idx, idx[k] for k < ndim,
 * out: "null pointer" / "null index plane k"), residency and flags, EDTB200_LABELS_FLOAT width, device. */
int edtb200_expand_gather(const void *labels, int label_bytes, int ndim,
                          int64_t sx, int64_t sy, int64_t sz, int64_t count,
                          const float *sqdist, const int32_t *const *idx,
                          double limit_sq, int flags, void *out, int device, void *stream);

/* Surface distances between two label volumes a (prediction) and b (reference) of one geometry, the
 * inputs of the Hausdorff distance, the average surface distance and surface Dice; `count` volumes of
 * (sx, sy, sz) each, laid back to back as for edtb200_transform_stack.
 *   surface S_v(k)  the voxels p of volume v with v[p] == k that have a face neighbour (2 ndim of them,
 *                   never in the next volume of the stack) of another label or lie on a face of their
 *                   volume: scipy's mask ^ binary_erosion(mask) with border_value 0
 *   d_v,k(q)        the float32 distance from q to the nearest voxel of S_v(k): edtb200_transform with
 *                   EDTB200_SQRT and no black_border of the 1-byte mask that is 0 on S_v(k) and 1
 *                   elsewhere, bit for bit; +inf when S_v(k) is empty
 *   segments        one per (volume, key, direction), numbered (volume * nkeys + key) * 2 + direction:
 *                   direction 0 (A->B) holds d_b,k(q) for every q in S_a(k), direction 1 (B->A) holds
 *                   d_a,k(q) for every q in S_b(k)
 *   keys            HOST array of nkeys labels of `label_bytes` bytes, non-zero and strictly ascending
 *                   as unsigned integers; read before the call returns
 *   flags           EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE: every other buffer is on `device`
 * Labels are compared as raw bits, as in the transforms.  Both calls are asynchronous on `stream`,
 * take no lock and free what they allocate (stream-ordered) on every exit.  An empty volume, count 0
 * or nkeys 0 returns 0 touching nothing.
 * Checks, in order: label width, ndim, sizes (as edtb200_transform), count >= 0, nkeys >= 0, the keys
 * ("null pointer (keys)" when nkeys > 0; no key 0; strictly ascending), count * nkeys within 2^60,
 * emptiness, pointers, residency (flags exactly the two residency flags), device. */

/* counts: count * nkeys * 2 int64, the length of every segment (|S_a(k)| for A->B, |S_b(k)| for
 * B->A), in segment order.  One pass over both volumes. */
int edtb200_surface_count(const void *a, const void *b, int label_bytes, int ndim,
                          int64_t sx, int64_t sy, int64_t sz, int64_t count,
                          const void *keys, int64_t nkeys, int flags, int64_t *counts,
                          int device, void *stream);

/* The distances of every segment.
 *   wx, wy, wz    anisotropy, as for edtb200_transform
 *   offsets       count * nkeys * 2 + 1 int64: the exclusive scan of edtb200_surface_count's counts,
 *                 the total last; segment s is written to values[offsets[s] .. offsets[s + 1]) in
 *                 unspecified order
 *   values        offsets[last] float32
 *   device_bytes  the budget of the call's device memory, 0 = the memory free on the device less
 *                 EDTB200_CHUNK_RESERVE
 *   groups        NULL, or int64_t[1] that receives the number of groups run (0 on an error or when
 *                 there is nothing to do)
 * The segments' slots go through the transform in groups: a group is a contiguous range of slots
 * whose masks are one stack through the transform of edtb200_transform_stack (one launch per pass),
 * one pass over the volumes writes the masks and one more gathers the distances.  A slot costs
 * V (1 + 4 + s) bytes for V = sx*sy*sz, s as for edtb200_transform_stack (8 when a later pass takes
 * the long-line kernel); a group holds at most floor(budget / slot) slots and at most 2^31 mask voxels
 * (at least one slot), and the call runs the fewest such groups, their sizes differing by one at
 * most (one group when every slot fits both); EDTB200_ENOMEM when not even one
 * slot fits, and the message names that least budget.  Outside the budget: the keys and one int64
 * cursor per segment. */
int edtb200_surface_distances(const void *a, const void *b, int label_bytes, int ndim,
                              int64_t sx, int64_t sy, int64_t sz, int64_t count,
                              float wx, float wy, float wz,
                              const void *keys, int64_t nkeys, int flags,
                              const int64_t *offsets, float *values,
                              int device, size_t device_bytes, int64_t *groups, void *stream);

/* The same transform of ONE host volume spread over several GPUs of this process
 * (`devices[0..ndevices)`, distinct ordinals): SURVEY.md section 8b's `devices[] / ndevices`.
 * Every device uploads one Z slab over its own PCIe link and runs the X and Y passes on it; the
 * distances and labels are then re-partitioned into Y slabs (whole z lines per device) by
 * peer-to-peer 3-D copies over NVLink, the Z pass runs, the result goes back the same way and
 * down to `out`.  Exact for any input (no halo, no verdict); `labels` and `out` are HOST pointers
 * (the *_ON_DEVICE flags are rejected).  Volumes that are not 3-D, or too thin to split, run on
 * devices[0].  Device memory per GPU: 2 * (label_bytes + 4) * voxels / ndevices.  Calls on
 * disjoint device sets may run concurrently from different threads. */
int edtb200_transform_multi(const void *labels, int label_bytes, int ndim,
                            int64_t sx, int64_t sy, int64_t sz,
                            float wx, float wy, float wz,
                            int black_border, int flags,
                            float *out, const int *devices, int ndevices);

/* Many volumes of one geometry, HOST buffers, pipelined: while volume k is being transformed,
 * volume k+1 is on its way to the device and volume k-1 on its way back (two device slots,
 * separate copy streams, PCIe used in both directions at once).  This is what a caller of the
 * reference does in a loop over the chunks of a dataset (README.md:191, the skeletonisation use
 * case); per volume the result is exactly what edtb200_transform returns.
 *   labels[k], outs[k]  host pointers (pinned memory is copied directly, pageable memory is staged
 *                       by two groups of host threads); outs[k] must not alias any labels[j]
 *   flags               EDTB200_SQRT / EDTB200_SIGNED; the *_ON_DEVICE flags are rejected
 * Returns when every result has landed. */
int edtb200_transform_batch(const void *const *labels, float *const *outs, int count,
                            int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                            float wx, float wy, float wz, int black_border, int flags, int device);

/* The same transform as edtb200_transform for a 2-D or 3-D HOST volume larger than the device's
 * memory, streamed through one device in chunks; the result is edtb200_transform's bit for bit.
 *
 * Two phases, exact for any input, no halo.  The passes along the first axes couple only the
 * voxels of one slice across the last axis, the last pass only the voxels of one line along it:
 *   phase 1  chunks of whole slices across the last axis (z slabs in 3-D, row ranges in 2-D): the
 *            labels go up, the X pass (and in 3-D the Y pass) runs, the distances come down into
 *            `out`, which holds the intermediate result;
 *   phase 2  chunks of whole lines along the last axis (y ranges in 3-D, x ranges in 2-D): the
 *            labels and the intermediate distances go up, the last pass runs with the sqrt / sign
 *            epilogue, the result comes down into `out`.
 * Every pass sees whole lines and runs with the whole volume's weights and extents, so it makes the
 * one-shot transform's arithmetic choices; the only borders are the volume's faces.  Each phase
 * pipelines its chunks through two device slots as edtb200_transform_batch does.  PCIe traffic is
 * (2 label_bytes + 4) bytes per voxel up and 8 down, against label_bytes and 4 for edtb200_transform:
 * this is for volumes that do not fit.
 *
 * The plan, per phase, from the budget B:
 *   slice   one slice (phase 1) or one line-set of the cut axis (phase 2: sx * sz voxels in 3-D, sy
 *           in 2-D) costs slice = voxels * (label_bytes + 4 + s) bytes, with s = 8 when the phase's
 *           later pass, over a chunk of the largest size allowed below, takes the long-line kernel
 *           (its two scratch volumes) and 0 otherwise (2-D phase 1 has no later pass);
 *   cap     phase-2 chunks hold fewer than 2^32 - 64 voxels, so that the last pass can take the
 *           tile kernel where the one-shot transform could not;
 *   chunks  one chunk when the whole extent fits B (and the cap); otherwise two slots with
 *           c = min(cap, floor(B / (2 slice))) slices per chunk, EDTB200_ENOMEM when c == 0 in
 *           either phase (the message names the smallest budget that works: the larger of the
 *           two phases' min(extent, 2) * slice);
 *   count   ceil(extent / c) chunks whose sizes differ by one at most.
 *
 *   labels, out   HOST buffers, pageable or pinned, that must not overlap; the *_ON_DEVICE flags
 *                 are rejected.  flags: EDTB200_SQRT / EDTB200_SIGNED.  ndim is 2 or 3.
 *   device_bytes  the device-memory budget B of the call; 0: the memory free on the device, less
 *                 EDTB200_CHUNK_RESERVE.  Either way the device's cached whole-volume buffers (those
 *                 edtb200_transform / _batch keep between calls) are freed first and its scratch
 *                 pool trimmed, so a call that follows a one-shot EDTB200_ENOMEM finds that memory.
 *   chunks        NULL, or int64_t[2] that receives {phase-1 chunks, phase-2 chunks}.
 * Returns when the result has landed; after an error the contents of `out` are unspecified.  Nothing
 * the call allocates on the device outlives it.  Calls on one device are serialised. */
#define EDTB200_CHUNK_RESERVE 536870912   /* 512 MiB left free under a budget of 0 */
int edtb200_transform_chunked(const void *labels, int label_bytes, int ndim,
                              int64_t sx, int64_t sy, int64_t sz,
                              float wx, float wy, float wz,
                              int black_border, int flags, float *out,
                              int device, size_t device_bytes, int64_t *chunks);

/* The same feature transform as edtb200_feature_transform for a 2-D or 3-D HOST volume larger than
 * the device's memory, streamed through one device in the two phases of edtb200_transform_chunked;
 * the distances and every index plane are edtb200_feature_transform's bit for bit.
 *
 * The site chain splits along the same phases: the last axis's code at p names a row of p's own line
 * (or no site), and the codes of the first axes at that row only touch its slice.
 *   phase 1  z slabs (3-D) / row ranges (2-D): the labels go up, the site-tracking X pass (and in 3-D
 *            the Y pass) runs, and every voxel's site within its slice is resolved -- (qx, qy) in 3-D,
 *            qx in 2-D -- and comes down with the intermediate distances: qx into idx_out[0], qy into
 *            idx_out[1], the distances into dist_out (when NULL: bit-cast into idx_out[ndim - 1], which
 *            phase 2 reads them from before it writes it).  "No site" stays apart from a face
 *            coordinate -1 in those planes until phase 2 turns it into -1;
 *   phase 2  y ranges of whole z lines (3-D) / x ranges of whole y lines (2-D): the labels, the
 *            intermediate distances and the partial sites go up, the last pass runs with the sqrt /
 *            sign epilogue, and each voxel's code along the last axis is followed to the partial site
 *            on its own line; the index planes (and the distances when dist_out is given) come down.
 * Every pass sees whole lines with the whole volume's weights and extents, so the site codes are the
 * one-shot codes.  Both phases pipeline their chunks through two device slots.  PCIe traffic per
 * voxel, in 3-D with distances: (2 label_bytes + 12) bytes up and 28 down, against label_bytes and 16
 * for edtb200_feature_transform (2-D: 2 label_bytes + 8 up, 20 down): this is for volumes that do not
 * fit.
 *
 * The plan is edtb200_transform_chunked's (slice, chunks, count; the ENOMEM message names the least
 * budget that works) with these bytes per voxel, each slot's buffers plus the later pass's hull
 * scratch of 4 bytes (every feature pass runs on the long-line kernel, so there is no phase-2 cap):
 *   phase 1  3-D: label_bytes + 20 (two distance volumes, two code planes, hull); 2-D: label_bytes + 8
 *            (distances, X codes; no later pass);
 *   phase 2  3-D: label_bytes + 28 (intermediate and final distances, two partial site planes, the Z
 *            codes, one more index plane, hull); 2-D: label_bytes + 20 (the same without qy and the
 *            extra plane).
 *
 *   labels, dist_out, idx_out[0..ndim)  HOST buffers, pageable or pinned, no two of which overlap;
 *                 dist_out may be NULL, no index plane may.  flags: EDTB200_SQRT / EDTB200_SIGNED;
 *                 the *_ON_DEVICE flags are rejected.  ndim is 2 or 3.
 *   device_bytes, chunks  as for edtb200_transform_chunked.
 * Returns when the result has landed; after an error the contents of the outputs are unspecified.
 * Calls on one device are serialised. */
int edtb200_feature_transform_chunked(const void *labels, int label_bytes, int ndim,
                                      int64_t sx, int64_t sy, int64_t sz,
                                      float wx, float wy, float wz,
                                      int black_border, int flags, float *dist_out,
                                      int32_t *const *idx_out, int device,
                                      size_t device_bytes, int64_t *chunks);

/* Transform under a voxel connectivity graph (2-D or 3-D only).
 *
 * Replaces  pyedt::_edt2dsq_voxel_graph<T, uint8_t>   src/edt_voxel_graph.hpp:54-123
 *           pyedt::_edt3dsq_voxel_graph<T, uint8_t>   src/edt_voxel_graph.hpp:125-214
 *           pyedt::_edt3d_voxel_graph  (EDTB200_SQRT) src/edt_voxel_graph.hpp:216-236
 * as bound by __edt2dsq_voxel_graph / __edt3dsq_voxel_graph, src/edt.pyx:514-620, 736-844.
 *
 *   graph   sx*sy*sz bytes, laid out like the labels; bit 0 / 2 / 4 set = the step to the +x / +y /
 *           +z neighbour is allowed (the cc3d voxel-connectivity bit field; other bits are not read)
 * Labels only say foreground (non-zero; > 0 with EDTB200_LABELS_FLOAT) or background here, as in
 * the reference.  The foreground is drawn on a doubled grid in which a forbidden edge is a
 * background cell, transformed with half the anisotropy, and sampled back; all of it on the device
 * (scratch: 1 + 4 bytes per doubled cell).  Residency as above; EDTB200_LABELS_ON_DEVICE covers
 * `labels` AND `graph`.
 * EDTB200_SIGNED is rejected: the reference's sdf with a graph is the difference of two such
 * transforms (src/edt.pyx:147-158), which the caller forms.
 */
int edtb200_transform_voxel_graph(const void *labels, int label_bytes, const unsigned char *graph,
                                  int ndim, int64_t sx, int64_t sy, int64_t sz,
                                  float wx, float wy, float wz,
                                  int black_border, int flags,
                                  float *out, int device, void *stream);

/* The same transform as edtb200_transform_voxel_graph for a 2-D or 3-D HOST volume whose doubled
 * grid does not fit the device, streamed through one device in the two phases of
 * edtb200_transform_chunked; the result is edtb200_transform_voxel_graph's bit for bit.
 *
 * Every pass of the doubled grid couples only the cells of one line, and the result samples the even
 * cells only; so only the Y pass's columns at even x and the last pass's lines at even (x, y) matter,
 * and each voxel carries two cells from the first phase into the second: those of its doubled line
 * along the last axis, (2x, 2y, 2z) and (2x, 2y, 2z + 1) in 3-D, (2x, 2y) and (2x, 2y + 1) in 2-D.
 * Both cells of that line's mask come from the voxel alone: cell 2l is foreground iff the voxel is,
 * cell 2l + 1 iff the voxel is, its +z (3-D, bit 4) / +y (2-D, bit 2) edge is allowed, and it does not
 * lie on the volume's last slice under a black border.
 *   phase 1  z slabs (3-D) / row ranges (2-D): the labels and the graph go up, the slab's doubled
 *            mask is drawn (the black border on the volume's last slice, not the slab's), the X pass
 *            runs over every doubled row and in 3-D the Y pass over every doubled column (the odd-x
 *            columns are not compacted away: that would cost a copy of the X distances for a pass
 *            that is not the bottleneck), and the two cells come down: cell 2l into `out`, cell
 *            2l + 1 into a host scratch of 4 bytes per voxel that the call allocates and frees
 *            (EDTB200_ENOMEM when the host refuses it);
 *   phase 2  y ranges of whole z lines (3-D) / x ranges of whole y lines (2-D): the labels, the graph
 *            and both cells go up, are interleaved into the box's doubled lines beside their mask, the
 *            last pass runs, and the even cells (through sqrt under EDTB200_SQRT) come down into `out`.
 * Every pass runs with the one-shot call's transform of the whole doubled grid (half the weights,
 * doubled extents), so it makes the one-shot arithmetic choices.  PCIe traffic per voxel:
 * (2 label_bytes + 10) bytes up and 12 down, against label_bytes + 1 and 4 for
 * edtb200_transform_voxel_graph: this is for volumes that do not fit.
 *
 * The plan is edtb200_transform_chunked's (slice, cap, chunks, count; the ENOMEM message names the
 * least budget that works: the larger of the two phases' min(extent, 2) * slice) with these bytes per
 * voxel, the slot's buffers plus the long-line kernel's two scratch volumes of doubled cells where the
 * phase's later pass takes it (s1 = 64 in 3-D, s2 = 16):
 *   phase 1  3-D: label_bytes + 49 (+ s1): labels, graph, 8 doubled distances, the two cells, the
 *            doubled mask; 2-D: label_bytes + 29: the same with 4 doubled cells, and no later pass;
 *   phase 2  label_bytes + 21 (+ s2): labels, graph, 2 doubled distances, the two cells, the mask of
 *            the doubled lines (2 bytes held in 4);
 *   cap      phase-2 chunks hold fewer than 2^32 - 64 doubled cells (sx * 2 sz per y in 3-D, 2 sy per
 *            x in 2-D), so that the last pass can take the tile kernel where the one-shot call's could
 *            not.
 *
 *   labels, graph, out  HOST buffers, pageable or pinned; out must not overlap labels or graph (the
 *                 two inputs may overlap each other).  flags: EDTB200_SQRT, EDTB200_LABELS_FLOAT;
 *                 EDTB200_SIGNED and the *_ON_DEVICE flags are rejected.  ndim is 2 or 3.
 *   device_bytes, chunks  as for edtb200_transform_chunked.
 * Returns when the result has landed; after an error the contents of `out` are unspecified.  Calls on
 * one device are serialised. */
int edtb200_transform_voxel_graph_chunked(const void *labels, int label_bytes, const unsigned char *graph,
                                          int ndim, int64_t sx, int64_t sy, int64_t sz,
                                          float wx, float wy, float wz,
                                          int black_border, int flags, float *out,
                                          int device, size_t device_bytes, int64_t *chunks);

/* Single axis passes on DEVICE-resident data, for callers that split a volume into Z slabs
 * across GPUs (SURVEY.md section 8e): every rank runs the first- and second-axis passes on
 * its slab, exchanges what the third axis needs, then runs the third-axis pass.
 *
 * edtb200_pass_first : replaces the X loop of _edt3dsq          src/edt.hpp:430-440
 * edtb200_pass_later : replaces the Y or Z loop of _edt3dsq     src/edt.hpp:450-475
 *     axis 1 = Y (stride sx), axis 2 = Z (stride sx*sy).
 *     flags: on pass_first EDTB200_SIGNED means "background is an ordinary label" (needed for
 *     sdf, no sign is applied there); on pass_later EDTB200_SQRT / EDTB200_SIGNED are applied
 *     in that pass's store (sqrt, negate background) -- use them on the last pass only.
 *     border_lo / border_hi say independently whether the low / high end of the axis is a
 *     volume face with black_border (an interior slab face is neither).
 *     pass_later works IN PLACE on f_dev (input = the previous pass's output) and only writes
 *     the elements whose value it changes.  f_dev may hold any samples: pass_later first reduces
 *     them on `stream` and waits for that (one small kernel) to learn whether every candidate
 *     w^2 d^2 + f is exact in double; when one may not be, the pass forms every candidate in
 *     double and rounds it once, as the reference does.
 */
int edtb200_pass_first(const void *labels_dev, int label_bytes,
                       int64_t sx, int64_t sy, int64_t sz, float wx,
                       int black_border, int flags,
                       float *f_dev, int device, void *stream);

int edtb200_pass_later(const void *labels_dev, int label_bytes, int axis,
                       int64_t sx, int64_t sy, int64_t sz, float w,
                       int border_lo, int border_hi, int flags,
                       float *f_dev, int device, void *stream);

/* edtb200_pass_window : one later pass of the bounded transforms (edtb200_transform_bounded) in their
 *     window kernel, for tests of that kernel alone.  B and R are the bounded transforms' for an axis of
 *     weight w and max_distance (edtb200_bounded_plan), and the window kernel runs whatever R is, up to
 *     its limit of 128 rows.  Out of place: fout_dev = the pass over the samples fin_dev (any
 *     non-negative floats), with every row above B written as +inf; codes_dev (may be NULL) = the
 *     feature transform's site codes of the pass.  axis, borders and flags as edtb200_pass_later; the
 *     arithmetic is decided from the samples as there (one reduction, and a wait for it).
 *     edtb200_last_later_launch reports the launch (kernel 2, R in info[1]).  Checks, in order: label
 *     width and sizes, axis, w (finite and > 0), max_distance (>= 0), R (at most 128), emptiness,
 *     pointers, fin / fout / codes overlapping, then the device. */
int edtb200_pass_window(const void *labels_dev, int label_bytes, int axis,
                        int64_t sx, int64_t sy, int64_t sz, float w,
                        int border_lo, int border_hi, int flags, double max_distance,
                        const float *fin_dev, float *fout_dev, int *codes_dev,
                        int device, void *stream);

/* edtb200_noise_planes : the X pass that a transform runs on label noise, for tests of that pass alone:
 *     the pass that also writes the run-start and settled planes of the later passes (DESIGN.md section
 *     4.1), over `count` volumes of (sx, sy, sz) laid end to end (2-D: images of (sx, sy)), on device
 *     buffers, asynchronous on `stream`.  f_dev gets the distances, planes_dev the planes, in the layout
 *     the transform uses, per later axis (y; in 3-D then z) the run-start plane and its settled plane:
 *       [y plane | settled_y | z plane | settled_z]     rows = sy * sz * count, wpr = ceil(sx / 32)
 *       run-start plane   wpr words per row (y, z), bit x % 32 of word x / 32: a y-run (z-run) starts
 *                         at the voxel -- y == 0 or its label differs from row y - 1's (z within its
 *                         own volume: z == 0 or its label differs from slice z - 1's); 0 past sx
 *       settled plane     one word per row: bit s set when every voxel of x-segment s (32 voxels, padding
 *                         voxels past sx counting as settled) ends the pass at f <= w_y^2 (w_z^2)
 *     passes 1: the X pass.  passes 2: then the Y pass as a transform on predicted label noise plans it
 *     (reading its plane, skipping settled tiles and refreshing settled_z where it does), so that f and
 *     the planes are what the Z pass would find.  flags: 0 or EDTB200_SQRT (its sqrt applies in the Y
 *     pass of a 2-D transform).  nchunks: y-chunks per slice of the pass's march, 1..sy (0: the
 *     transform's own rule); ctas: its grid, 1..items, only with nchunks given (0: one persistent wave).
 *     info (10 ints): label bytes, K (128-voxel blocks per row), Plain, planes written (1 or 2), the
 *     march's nchunks, items and grid, and for passes 2 whether the Y pass read its plane, skipped
 *     settled tiles and refreshed settled_z.  edtb200_last_later_launch reports the Y launch.  Refused
 *     (EDTB200_EINVAL, before any device is touched) is every call a transform never sends down this
 *     path: labels of 1 or 2 bytes, ndim 1, EDTB200_SIGNED or another flag, rows longer than 512 or not
 *     a multiple of 4, more than 2^31 - 1 slices or 2^30 - 1 rows, nchunks or ctas out of range, and
 *     pointers not aligned for vector access; passes 2 also where the transform would take no planes
 *     (EDTB200_EINVAL after the probe).  Checks, in order: label width and sizes, label width >= 4,
 *     ndim, count, weights, flags, passes, sx, counters, nchunks, ctas, emptiness, pointers, alignment,
 *     then the device. */
int edtb200_noise_planes(const void *labels_dev, int label_bytes, int ndim,
                         int64_t sx, int64_t sy, int64_t sz, int64_t count,
                         float wx, float wy, float wz, int black_border, int flags,
                         int passes, int nchunks, int ctas,
                         float *f_dev, uint32_t *planes_dev, int *info,
                         int device, void *stream);

/* Z-slab decomposition across GPUs (DESIGN.md section 8): a rank runs edtb200_pass_later(axis=2)
 * on its slab with the interior faces open (border flags 0 there) and then folds the
 * neighbouring slabs in with these two calls, which replace what the reference gets for free
 * from having the whole z-line in one address space (src/edt.hpp:465-475).
 *
 * edtb200_slab_face_runs : for every (x,y) line, the length m (1..halo) of the run of equal
 *     labels that touches the low (high_face=0) or high (high_face=1) face of this slab;
 *     m = halo+1 means "longer than the halo, or spanning the whole slab".  *overflow_dev (device
 *     int, zeroed by the caller) is raised when that happens for a foreground run (any run with
 *     EDTB200_SIGNED): a hint that the fix-up's verdict below matters for this volume.
 * edtb200_slab_face_fixup : after the third-axis pass (same flags: EDTB200_SQRT / SIGNED),
 *     min-combines every row of the face-touching runs with the neighbour's sites:
 *     nb_label_dev = the neighbour's face plane of labels, nb_m_dev = its face_runs output,
 *     nb_f_dev = `halo` planes of the neighbour's distances taken after ITS second-axis pass,
 *     in the neighbour's z order (its last `halo` planes for our low face, its first for our
 *     high face).  Requires sz > halo on both sides.  Runs that go on behind the halo are exact
 *     as long as the distances at the face stay within the halo's reach (value <= (w*halo)^2);
 *     *inexact_dev (device int, zeroed by the caller, may be NULL) is raised when they do not,
 *     and the caller must then repeat with a deeper halo or an exact method.
 */
int edtb200_slab_face_runs(const void *labels_dev, int label_bytes,
                           int64_t sx, int64_t sy, int64_t sz, int high_face, int halo, int flags,
                           unsigned char *m_dev, int *overflow_dev, int device, void *stream);

int edtb200_slab_face_fixup(const void *labels_dev, int label_bytes,
                            int64_t sx, int64_t sy, int64_t sz, int high_face, int halo, float wz,
                            int flags, const void *nb_label_dev, const unsigned char *nb_m_dev,
                            const float *nb_f_dev, float *f_dev, int *inexact_dev,
                            int device, void *stream);

/* Exact fallback of the Z-slab decomposition (runs deeper than any halo): the ranks re-partition
 * the volume from Z slabs to Y slabs, run the third-axis pass on whole z-lines and re-partition
 * back.  edtb200_slab_pack moves a device-resident slab (zc, sy, row_bytes) -- distances or
 * labels, the row is opaque bytes -- into the exchange layout in ONE launch: the slab is cut
 * along y into `parts` pieces (piece i = rows y_start[i] .. y_start[i+1], y_start[0] = 0,
 * y_start[parts] = sy; HOST array of parts + 1 entries, parts <= 64), and piece i becomes one
 * contiguous block (zc, c_i, row_bytes), the blocks in piece order -- block i is the single
 * message for rank i.  unpack != 0 applies the inverse map (blocks -> slab) for the way back.
 * Replaces what the reference gets from having the whole volume in one address space
 * (src/edt.hpp:450-475).
 */
int edtb200_slab_pack(const void *src_dev, void *dst_dev, int64_t zc, int64_t sy, int64_t row_bytes,
                      int parts, const int64_t *y_start, int unpack, int device, void *stream);

/* One whole step of the Z-slab decomposition on this rank, device-resident, asynchronous on
 * `stream`: X pass, Y pass, publication of this slab's faces to the neighbours, Z pass (interior
 * faces open) and the fix-up that folds the neighbours' rows in -- five launches from ONE call, no
 * host synchronisation, no collective.  The ranks meet only through flag words in a staging buffer
 * that every rank allocates in CUDA symmetric memory (peer-mapped over NVLink):
 *   sym_self        this rank's buffer, edtb200_slab_stage_bytes(sx, sy, label_bytes, halo) bytes,
 *                   ZERO-FILLED once before the first step (all ranks, then a barrier)
 *   sym_lo, sym_hi  the lower / upper neighbour's buffer as mapped into this process (NULL where
 *                   has_lo / has_hi is 0)
 *   step            1, 2, 3, ... the same on every rank; staging sets alternate by its parity
 *   status_dev      device int, OR-ed with 1 when the halo was too shallow for this volume (a run
 *                   goes on behind the neighbour's `halo` rows and the distances at the face exceed
 *                   the halo's reach: repeat with a deeper halo or an exact method), and with 2
 *                   when a neighbour never published the step (time-out)
 * flags: EDTB200_SQRT / EDTB200_SIGNED as for edtb200_transform; black_border applies to the real
 * volume faces only (z low face on the rank with has_lo == 0, z high face where has_hi == 0).
 * This is what replaces the reference's single-address-space Z loop (src/edt.hpp:465-475) when
 * the volume is spread over several GPUs. */
int64_t edtb200_slab_stage_bytes(int64_t sx, int64_t sy, int label_bytes, int halo);

int edtb200_slab_step(const void *labels_dev, int label_bytes, int64_t sx, int64_t sy, int64_t sz,
                      float wx, float wy, float wz, int black_border, int has_lo, int has_hi, int flags,
                      float *f_dev, int halo, void *sym_self, void *sym_lo, void *sym_hi,
                      unsigned long long step, int *status_dev, int device, void *stream);

/* Per-label views of a finished transform, on the device: the reference's `edt.each`
 * (src/edt.pyx:951-994: one masked distance image per label, built from run lists,
 * src/edt_voxel_graph.hpp:238-310) for labels and distances that are already resident on the GPU.
 *
 * edtb200_label_stats : ONE pass over (labels, dt) fills an open-addressing table of `capacity`
 *     slots (a power of two, at least twice the number of distinct labels): keys_dev[s] = label
 *     (0 = empty slot; label 0 is background and skipped), count_dev[s] = its voxels,
 *     max_dev[s] = its largest distance, argmax_dev[s] = the smallest linear index (x fastest)
 *     where that maximum is attained, box_dev[6*s..] = bounding box x0 y0 z0 x1 y1 z1 (inclusive).
 *     A label's key is its raw bits zero-extended to 64 bits (signed labels are never sign-extended);
 *     distances may be negative or infinite (not NaN).  Only each axis has to fit an int: a plane
 *     sx * sy of more than 2^31 voxels is supported.
 *     *overflow_dev is raised when the table was too small (repeat with a larger capacity).  While it
 *     is 0 the table is complete, even with every slot filled; once it is 1 the call still returns
 *     0 and the only guarantee is that every filled slot holds a label of the volume, each label at
 *     most once -- its statistics may be partial and other labels are missing.
 * edtb200_label_extract : out = (labels == key) ? dt : 0 inside `box` (6 host ints as above, NULL =
 *     whole volume), nothing outside it is touched -- the equivalent of transfer_run_voxels on a
 *     blank image; erase != 0 zeroes the box instead (the reference's erase()).
 * All pointers except `box` are device pointers on `device`; asynchronous on `stream`. */
int edtb200_label_stats(const void *labels_dev, int label_bytes, const float *dt_dev,
                        int64_t sx, int64_t sy, int64_t sz, int capacity,
                        unsigned long long *keys_dev, unsigned long long *count_dev, float *max_dev,
                        long long *argmax_dev, int *box_dev, int *overflow_dev, int device, void *stream);

int edtb200_label_extract(const void *labels_dev, int label_bytes, const float *dt_dev,
                          int64_t sx, int64_t sy, int64_t sz, unsigned long long key, const int *box,
                          int erase, float *out_dev, int device, void *stream);

/* Page-locked host memory for result arrays (cudaHostAlloc, portable): a transform whose `out` lies
 * in such a block is copied back by one DMA at PCIe rate, with no staging copy and no page faults.
 * The Python front door keeps a small pool of these blocks behind the arrays it returns.
 * edtb200_host_alloc returns NULL when no device / no memory is available. */
void *edtb200_host_alloc(size_t bytes);
void edtb200_host_free(void *p);

/* Measurement hooks (used by bench.py): with profiling enabled on the calling thread, every
 * edtb200_transform records CUDA events around its axis passes on the transform's stream into a
 * ring of 256 slots -- nothing synchronises inside a timed loop.  edtb200_pass_ms(k, ms) waits
 * for the transform issued k calls ago (0 = the latest) and returns the device time of its
 * first, second and third axis pass in milliseconds (0 for passes that did not run). */
int edtb200_profile_passes(int enable);
int edtb200_pass_ms(int steps_back, float *ms3);

/* Which kernel variant the last later-axis (Y or Z) pass launched by the calling thread used, so
 * that tests can tell which code paths they reached.  Read-only: it changes no launch.  Fills
 * info[0..9): kernel (0 = shared-memory tile, 1 = long-line, 2 = the bounded transforms' window
 * kernel, with its radius in place of the tile width), tile width TX, TMA staging, wide
 * CTA, CTAs per SM the tile kernel is compiled for, integer hull tests, epilogue (sqrt / sign in
 * the store), every candidate formed in double, tiles left settled by the X pass skipped.
 * EDTB200_EINVAL before any such launch. */
int edtb200_last_later_launch(int *info);

/* Free every cached device buffer / stream this library holds on all devices. */
int edtb200_release(void);

#ifdef __cplusplus
}
#endif
#endif /* EDT_B200_H */
