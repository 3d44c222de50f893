/*
 * mrx.h -- C ABI of the H100 (sm_90a) Mask R-CNN serving hot path.
 *
 * The reference (huyhoang17/matterport-maskrcnn-with-tensorflow-serving) has NO
 * FFI / plugin interface: its boundary is three plain Python call sites in
 * serve.py.  Each entry point below names the Python call it stands behind:
 *
 *   mrx_anchors            <- api_utils.get_anchors(image_shape)          serve.py:105
 *   mrx_unmold_prepare     <- api_utils.unmold_detections(...) steps 1-6  serve.py:147-154
 *                             and mrcnn_mask[arange(N),:,:,class_ids]     (same call)
 *   mrx_mask_expand        <- per-instance unmold_mask + np.stack(axis=-1)(same call)
 *   mrx_mask_expand_values    (parity instrumentation of the kernel above)
 *   mrx_cv2_resize_u8c3[_batch] <- cv2.resize(img, (S, S))                serve.py:88-89
 *   mrx_mold_image[_batch] <- resize_image + mold_image                   serve.py:91-98
 *   mrx_composite_masks    <- visualize.display_instances (mask overlay)  serve.py:160-169
 *   mrx_pack_masks         (extension: bit-packed transport of the masks of serve.py:147)
 *   mrx_mask_expand_packed (extension: the expand step writing that packed layout directly)
 *   mrx_rle_count / _write (extension: the same masks as COCO run-length encodings)
 *   mrx_rle_strings        (extension: those encodings as COCO compressed RLE strings)
 *   mrx_contours_count / _write <- visualize.display_instances (contour polygons) serve.py:160-169
 *   mrx_annotate_draw / _resolve <- visualize.display_instances (boxes, outlines, captions) serve.py:160-169
 *   mrx_mask_extents / _overlaps / _matches (extension: mrcnn.utils.compute_overlaps_masks and
 *                             compute_matches, scoring the masks against ground truth)
 *   mrx_rle_parse / _decode (extension: ground truth given as COCO RLE, decoded to packed planes)
 *   mrx_coco_ranks / _ious / _box_ious / _match[_f64area] (extension: pycocotools' COCOeval for
 *                             "segm" and "bbox", the per-image half)
 *   mrx_mask_boundary / mrx_coco_boundary_ious (extension: the same for "boundary", Boundary AP)
 *   mrx_lvis_ranks         (extension: lvis-api's LVISEval, the per-image cut and federated filter)
 *   mrx_jpeg_coefficients / _pixels <- api_utils.load_img (cv2.imread)   serve.py:85-86
 *                             (extension: JPEG request bytes decoded on the device, as cv2.imdecode;
 *                             mrx_jpeg_progressive_coefficients for progressive files)
 *   mrx_png_decode         <- api_utils.load_img (cv2.imread)   serve.py:85-86
 *                             (extension: PNG request bytes decoded on the device, as cv2.imdecode)
 *   mrx_png_encode        <- cv2.imwrite of the overlay PNG                 serve.py:168
 *   mrx_jpeg_encode       <- cv2.imwrite of the overlay                     serve.py:168
 *                             (extension: the overlay as a JPEG file, as cv2.imencode('.jpg'))
 *   mrx_peer_*             (multi-GPU: the final gather of the masks to rank 0, SURVEY.md 8e)
 *   mrx_device_alloc/_free (the canvas allocation: compressible device memory where offered)
 *
 * Conventions
 *   - every pointer named d_* is DEVICE memory owned by the caller (the Python
 *     side holds them as torch tensors and passes data_ptr()); nothing here
 *     allocates, frees or synchronises -- all work is ordered on `stream`
 *     (a cudaStream_t passed as void*; NULL = legacy default stream).
 *   - return value: MRX_OK (0) or a negative MRX_E_* code; mrx_last_error()
 *     returns a thread-local description of the last failure.
 *   - dtype codes: MRX_F32 = 0, MRX_F64 = 1.
 *   - there is no CPU fallback behind any of these calls.
 */
#ifndef MRX_H_
#define MRX_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MRX_ABI_VERSION 17

#define MRX_OK              0
#define MRX_E_INVALID      -1   /* bad argument (null pointer, size out of range) */
#define MRX_E_UNSUPPORTED  -2   /* shape outside what the kernels are built for   */
#define MRX_E_CUDA         -3   /* a CUDA runtime call failed                      */

#define MRX_F32 0
#define MRX_F64 1

/* per-image status bits written by mrx_unmold_prepare into d_status[b] */
#define MRX_ST_CLASS_RANGE  1   /* class id outside [-C, C) or NaN: numpy would raise IndexError */
/* kept box outside the canvas: numpy's paste would raise, or wrap a box that lies entirely at
 * negative coordinates to the far edge; we raise for both */
#define MRX_ST_BOX_RANGE    2

/* limits (compile-time properties of the kernels) */
#define MRX_MAX_LEVELS   8
#define MRX_MAX_RATIOS   8
#define MRX_MAX_BATCH    4096    /* images per mrx_mask_expand launch */
#define MRX_MAX_MASK_DIM 64      /* mask tile side (28 upstream); width must be a multiple of 4 */
#define MRX_MAX_LANE_MASK_W 30   /* tile width of the lane kernels: mw + 2 lanes per warp */

int         mrx_abi_version(void);
const char *mrx_last_error(void);

/* Device properties the host-side planner needs (SM count, opt-in smem per block). */
int mrx_device_props(int device, int *sm_count, int *cc_major, int *cc_minor,
                     int *max_smem_optin);

/* ---------------------------------------------------------------- anchors (a5) */
/* Number of anchors for an image of img_h x img_w:  R * sum_l ceil(ceil(H/s_l)/as) * ceil(ceil(W/s_l)/as). */
int mrx_anchor_count(int img_h, int img_w, const int *strides, int n_levels,
                     int n_ratios, int anchor_stride, long long *count);

/* d_out: [A,4] float32 (y1,x1,y2,x2) normalised by norm_boxes; level-major, then
 * y, x, ratio innermost.  scales[n_levels], ratios[n_ratios] are HOST arrays.
 * Arithmetic is fp64 with numpy's operation order, rounded once to fp32. */
int mrx_anchors(float *d_out, int img_h, int img_w,
                const double *scales, const double *ratios, const int *strides,
                int n_levels, int n_ratios, int anchor_stride, void *stream);

/* ---------------------------------------------------------------- unmold (a1-a4) */
/* Geometry per image, 8 x int32:
 *   [0] orig_h [1] orig_w   original image (canvas) size
 *   [2] img_h  [3] img_w    molded image size
 *   [4..7]  window y1,x1,y2,x2 in molded pixels                                  */
#define MRX_GEOM_INTS 8

/* Scheduler scratch of the expand kernels: MRX_SCHED_WORDS x uint32 of device memory that the
 * caller zeroes ONCE after allocating it; every launch hands out its work through it and leaves
 * it zeroed (no memset between launches).  One scratch per stream of launches. */
#define MRX_SCHED_WORDS 4

/* Steps 1-6 of unmold_detections and the class-tile gather for a batch of B images, in ONE
 * launch.  Steps 1-6, one CTA per image: trim at the first class_id==0 row, class ids, window
 * normalisation (float32), box affine + denorm (float64, round-half-even), zero-area drop with
 * order-preserving compaction.
 *   d_detections [B,R,6] det_dtype      d_mrcnn_mask [B,R,mh,mw,C] mask_dtype   d_geom [B,8] int32
 *   d_boxes [B,R,4] int32   d_class_ids [B,R] int32   d_scores [B,R] det_dtype
 *   d_src_index [B,R] int32 (kept row -> original row)
 *   d_counts [B] int32 (N per image)    d_status [B] int32 (MRX_ST_* bits)
 * C = number of classes in mrcnn_mask's last axis (for the class-range check).
 * d_sched (may be NULL): the scheduler words of the expand kernels (MRX_SCHED_WORDS x uint32),
 * zeroed here as well.  The class tiles are stored by ORIGINAL detection row,
 *   d_tiles[b][t] = float32(mrcnn_mask[b, t, :, :, class_id of row t])
 *   (rows whose class_id is exactly 0: untouched; 0.5 truncates to class 0 and is gathered)
 * which needs nothing from steps 1-6, so both run side by side in the same grid.  The expand
 * entry points then take d_tile_index = d_src_index (kept instance k -> its row). */
int mrx_unmold_prepare(const void *d_detections, int det_dtype, const void *d_mrcnn_mask,
                       int mask_dtype, int B, int R, int mh, int mw, int C,
                       const int *d_geom, int *d_boxes, int *d_class_ids, void *d_scores,
                       int *d_src_index, int *d_counts, int *d_status,
                       float *d_tiles, unsigned int *d_sched, void *stream);

/* Tile batch: the inputs of every entry point that reads the class tiles (mrx_mask_expand,
 * mrx_mask_expand_values, mrx_mask_expand_packed, mrx_rle_count, mrx_rle_write), as
 * mrx_unmold_prepare leaves them:
 *   d_tiles [B,R,mh,mw] float32   d_boxes [B,R,4] int32   d_counts [B] int32   d_geom [B,8] int32
 *   d_tile_index [B,R] int32, required: kept instance k of image b resizes
 *   d_tiles[b][d_tile_index[b][k]] (d_src_index for the layout mrx_unmold_prepare writes).
 * Each of them checks these first, in this order, before anything reaches the device:
 *   - d_tiles, d_boxes, d_counts or d_geom null: MRX_E_INVALID;
 *   - B outside [0, MRX_MAX_BATCH] or R outside [1, 65534]: MRX_E_INVALID;
 *   - mh outside [2, MRX_MAX_MASK_DIM], or mw outside [4, max_mw] or not a multiple of 4:
 *     MRX_E_UNSUPPORTED.  max_mw is MRX_MAX_MASK_DIM for mrx_mask_expand and MRX_MAX_LANE_MASK_W
 *     for the others, the lane kernels, which keep a tile row in one warp's lanes;
 *   - d_tile_index null: MRX_E_INVALID.
 * Then it checks its own arguments, and B = 0 returns MRX_OK without launching anything. */

/* Output slots: where the masks of a planned batch live (engine.BatchLayout states the same on
 * the host), for every entry point that writes or reads them (mrx_mask_expand,
 * mrx_mask_expand_values, mrx_mask_expand_packed, mrx_pack_masks, mrx_composite_masks,
 * mrx_contours_count, mrx_contours_write, mrx_mask_extents, mrx_mask_overlaps, mrx_rle_decode,
 * mrx_mask_boundary, mrx_coco_boundary_ious).
 * N_b = d_counts[b], H_b, W_b = d_geom[b][0], [1].
 *   Canvas slots: image b's bool masks [H_b, W_b, N_b] (N innermost, 1 byte per element, values
 *     0/1) at d_canvas + d_canvas_off[b] (int64, each a multiple of 16).  Slot b holds at least
 *     round_up(H_b*W_b*N_b, 16) bytes; bytes past H_b*W_b*N_b may be read, and written by the
 *     expand kernels.
 *   Packed slots: image b's planes uint8 [N_b, H_b, ceil(W_b/8)] at d_packed + d_packed_off[b]
 *     (int64), packed[n, y, :] = np.packbits(masks[y, :, n]) (most significant bit first); slot b
 *     holds R*H_b*ceil(W_b/8) bytes.  Planes n >= N_b are not written.
 *   Extents for grid sizing: max_h, max_w and max_pixels are the largest H_b, W_b and H_b*W_b of
 *     the batch (or more).  mrx_pack_masks and mrx_composite_masks take 0 as "no image has a
 *     pixel" and return MRX_OK without launching; mrx_mask_expand_packed and mrx_contours_* need
 *     at least 1 (contours writes its offsets even when there is nothing to trace).
 * Each of them checks, in this order, before anything reaches the device (right after the tile
 * batch, for the three that read one):
 *   - the slot base (d_canvas or d_packed), its offsets, d_counts or d_geom null: MRX_E_INVALID;
 *   - B outside [0, MRX_MAX_BATCH] or R outside [1, 65534]: MRX_E_INVALID;
 *   - then its own extents and arguments, and B = 0 returns MRX_OK without launching anything.
 * Every message of mrx_last_error() starts with the name of the function called. */

/* The hot kernel.  For every image b writes its canvas slot (see "Output slots"): zero fill,
 * zero-border half-pixel bilinear resize of each tile to its box, >= 0.5 threshold and paste,
 * fused so each output byte is written once.  Inputs: a tile batch.
 *   chunk_bytes: upper bound, in bytes, of the canvas tile a team of warps builds in
 *   shared memory and stores with one bulk copy per tile row (a tile is P pixels x
 *   10 rows x N instances; it is raised to the minimum that holds 16 pixels of R
 *   instances per row); multiple of 16, >= 1024; 0 = as large as fits (library default).
 *   ctas_per_sm: used by the generic kernel only (R too large for the tile buffers, or
 *   mask tiles wider than MRX_MAX_LANE_MASK_W); 0 = as many as fit. */
int mrx_mask_expand(const float *d_tiles, const int *d_tile_index, const int *d_boxes,
                    const int *d_counts, const int *d_geom, const long long *d_canvas_off,
                    unsigned char *d_canvas, int B, int R, int mh, int mw,
                    int chunk_bytes, int ctas_per_sm,
                    unsigned int *d_sched, void *stream);

/* Parity instrumentation: the SAME kernel template as mrx_mask_expand (same culling, source
 * coordinates, interpolation and row walk -- a second instantiation of it), which in addition
 * stores every pre-threshold sample it evaluates: d_values is float32, indexed exactly like
 * d_canvas (element d_canvas_off[b] + (y*W_b + x)*N_b + n); only elements inside box n are
 * written.  The canvas slots are written as usual.  Tests compare these values with the float64
 * oracle (|diff| <= 1e-6).  Inputs: a tile batch, as a lane kernel.  R whose tile row no longer
 * fits a team's buffer returns MRX_E_UNSUPPORTED before launching anything (on an H100, R > 213
 * at B = 1; the limit drops slowly for large batches, whose scheduler table takes shared memory
 * from the buffers). */
int mrx_mask_expand_values(const float *d_tiles, const int *d_tile_index, const int *d_boxes,
                           const int *d_counts, const int *d_geom, const long long *d_canvas_off,
                           unsigned char *d_canvas, float *d_values, int B, int R, int mh, int mw,
                           unsigned int *d_sched, void *stream);

/* ---------------------------------------------------------------- mold (a6) */
/* cv2.resize(src, (dst_w, dst_h)) for uint8 HxWx3, default INTER_LINEAR
 * (OpenCV's 11-bit fixed-point path, incl. its exact-2x INTER_AREA shortcut). */
int mrx_cv2_resize_u8c3(const unsigned char *d_src, int src_h, int src_w,
                        unsigned char *d_dst, int dst_h, int dst_w, void *stream);

/* The same for a batch in ONE launch (the reference resizes every request image to
 * (IMAGE_SIZE, IMAGE_SIZE), serve.py:88-89, 114): sources of any sizes, image b at
 * d_src + d_src_off[b] (int64 byte offsets) with (h, w) = d_src_hw[2b], d_src_hw[2b+1];
 * destinations densely packed [B, dst_h, dst_w, 3]. */
int mrx_cv2_resize_u8c3_batch(const unsigned char *d_src, const long long *d_src_off,
                              const int *d_src_hw, unsigned char *d_dst, int B,
                              int dst_h, int dst_w, void *stream);

/* resize_image(mode square/pad64/none geometry precomputed by the host) fused
 * with mold_image: scale src (uint8 HxWx3) to new_h x new_w with the zero-border
 * bilinear of a4 in fp64, truncate to uint8, place at (top,left) in an
 * out_h x out_w canvas of zeros, subtract mean_pixel.
 *   out_dtype MRX_F32: float32( float64(u8) - mean )   (what serve.py:117 sends)
 *   out_dtype MRX_F64: float64(u8) - mean              (what preprocess_input returns)
 *   d_molded_u8 (optional, may be NULL): the uint8 image before mean subtraction. */
int mrx_mold_image(const unsigned char *d_src, int src_h, int src_w,
                   int new_h, int new_w, int top, int left, int out_h, int out_w,
                   const double *mean_pixel /* host, 3 */, int out_dtype,
                   void *d_out, unsigned char *d_molded_u8, void *stream);

/* The same for B equally sized images in ONE launch: d_src [B,src_h,src_w,3] ->
 * d_out [B,out_h,out_w,3] (and d_molded_u8 likewise). */
int mrx_mold_image_batch(const unsigned char *d_src, int B, int src_h, int src_w,
                         int new_h, int new_w, int top, int left, int out_h, int out_w,
                         const double *mean_pixel /* host, 3 */, int out_dtype,
                         void *d_out, unsigned char *d_molded_u8, void *stream);

/* ---------------------------------------------------------------- compositing (8f) */
/* Mask part of visualize.display_instances(img, boxes, masks, ...) (serve.py:160-169), on
 * the canvas slots mrx_mask_expand wrote: for every image b, per instance i in order (skipped when
 * its box is all zeros), per channel c,
 *     v = uint32( float64(v) * one_minus_alpha + blend[b][i][c] )      where mask[.,.,i] == 1
 * starting from the uint8 image and ending with astype(uint8).
 *   d_images / d_out: uint8 H_b x W_b x 3 images of the batch, image b at byte offset
 *   d_image_off[b] (int64) in both;  d_blend [B,R,3] float64 = alpha * color[c] * 255,
 *   evaluated by the caller in float64 in that order;  d_boxes [B,R,4] as written by
 *   mrx_unmold_prepare;  max_pixels: the extent of "Output slots", below 2^31 - 257. */
int mrx_composite_masks(const unsigned char *d_canvas, const long long *d_canvas_off,
                        const int *d_counts, const int *d_geom, const int *d_boxes,
                        const unsigned char *d_images, const long long *d_image_off,
                        const double *d_blend, double one_minus_alpha,
                        unsigned char *d_out, int B, int R, long long max_pixels,
                        void *stream);

/* ---------------------------------------------------------------- packed masks (8f) */
/* EXTENSION (not the reference layout): bit-packed copy of the canvas slots into the packed
 * slots, for transport (see "Output slots"): np.unpackbits(packed, axis=-1,
 * count=W).transpose(1, 2, 0) is the bool [H,W,N] array unmold_detections returns.  max_h,
 * max_w: the extents of "Output slots"; max_h above 65535: MRX_E_UNSUPPORTED.  R too large for
 * the kernels' shared memory returns MRX_E_UNSUPPORTED before launching anything (on an H100,
 * R > 907). */
int mrx_pack_masks(const unsigned char *d_canvas, const long long *d_canvas_off,
                   const int *d_counts, const int *d_geom, unsigned char *d_packed,
                   const long long *d_packed_off, int B, int R, int max_h, int max_w,
                   void *stream);

/* EXTENSION: the expand step with bit-packed output, without ever writing the byte canvas
 * (expand_bits.cu).  Inputs: a tile batch, as a lane kernel (wider tiles take mrx_mask_expand +
 * mrx_pack_masks).  Output: the packed slots (see "Output slots"), exactly as mrx_pack_masks
 * writes them.  The samples are computed with the same arithmetic as mrx_mask_expand, so
 * packed == np.packbits(canvas)  bit for bit.  d_packed may be memory of ANOTHER GPU mapped with
 * mrx_peer_open (fused compute + gather).  max_w: the extent of "Output slots". */
int mrx_mask_expand_packed(const float *d_tiles, const int *d_tile_index, const int *d_boxes,
                           const int *d_counts,
                           const int *d_geom, const long long *d_packed_off,
                           unsigned char *d_packed, int B, int R, int mh, int mw, int max_w,
                           unsigned int *d_sched, void *stream);

/* EXTENSION: COCO run-length masks (pycocotools' "uncompressed RLE": the mask in COLUMN-major
 * order as alternating run lengths of zeros and ones, starting with zeros), computed from the
 * tiles with the arithmetic of mrx_mask_expand -- decoding them gives that kernel's masks bit
 * for bit -- without materialising any mask (rle.cu).  Two calls around one host read:
 *   mrx_rle_count:  d_col_count [B,R,max_w] int32 scratch; d_inst_off [B*R+1] int64: on return
 *                   (stream-ordered) d_inst_off[i] = number of value changes of all instances
 *                   before i = b*R + k, d_inst_off[B*R] = their total T.  The caller reads T and
 *                   allocates d_positions [T] and d_run_lengths [T + B*R] (uint32).
 *   mrx_rle_write:  instance i's runs are d_run_lengths[d_inst_off[i] + i ...], one more than
 *                   its value changes (d_inst_off[i+1] - d_inst_off[i] + 1); they sum to H*W.
 * Inputs: a tile batch, as a lane kernel; max_w as for mrx_mask_expand_packed. */
int mrx_rle_count(const float *d_tiles, const int *d_tile_index, const int *d_boxes,
                  const int *d_counts, const int *d_geom, int *d_col_count,
                  long long *d_inst_off, int B, int R, int mh, int mw, int max_w, void *stream);
int mrx_rle_write(const float *d_tiles, const int *d_tile_index, const int *d_boxes,
                  const int *d_counts, const int *d_geom, int *d_col_count,
                  long long *d_inst_off, unsigned int *d_positions, unsigned int *d_run_lengths,
                  int B, int R, int mh, int mw, int max_w, void *stream);

/* EXTENSION: pycocotools' compressed RLE ("counts" string of mask.encode) of every kept instance,
 * from the output of mrx_rle_write (d_run_lengths, d_inst_off as written there; d_counts and R as
 * given there).  d_str_off [B*R+1] int64: exclusive byte offsets of the instances' strings, total
 * at [B*R] (instances k >= counts[b] get empty strings).  d_str: at least
 * MRX_RLE_STRING_BOUND(T, B*R) bytes, T = d_inst_off[B*R] (every count takes at most 7
 * characters).  Strings are not NUL-terminated.  Run j of an instance is written as
 * x = cnts[j] - cnts[j-2] (cnts[j] for j <= 2) in little-endian 5-bit groups, character
 * '0' + group, 0x20 added to every group but the last, whose bit 0x10 is the sign.  Checks: null
 * pointers, B outside [0, MRX_MAX_BATCH] or R outside [1, 65534]: MRX_E_INVALID; B = 0 returns
 * MRX_OK without launching anything. */
#define MRX_RLE_STRING_BOUND(T, n) (7LL * ((T) + (n)))
int mrx_rle_strings(const unsigned int *d_run_lengths, const long long *d_inst_off,
                    const int *d_counts, int B, int R, long long *d_str_off,
                    unsigned char *d_str, void *stream);

/* EXTENSION: mask outlines as polygons, the contour loop of visualize.display_instances
 * (serve.py:160-169): for each instance, skimage.measure.find_contours(padded, 0.5) of the mask
 * padded with one pixel of zeros on every side (fully_connected and positive_orientation 'low'),
 * vertices as (x, y) image coordinates = np.fliplr(v) - 1 (contours.cu).  Input: the packed slots
 * (see "Output slots") as mrx_pack_masks / mrx_mask_expand_packed write them; max_h: the extent
 * of "Output slots", below 2^30.  d_regions [B,R,4] int32 (y1, x1, y2, x2), required: instance k is traced
 * only inside that pixel rectangle (clamped to the image; pixels outside it count as 0; an empty
 * rectangle gives no contour), e.g. the d_boxes of mrx_unmold_prepare, outside which the plane is
 * zero.  Two calls around one host read:
 *   mrx_contours_count:  d_row_off [B,R,max_h+1] int32 scratch; d_inst_off [B*R+1] int64: on
 *                        return (stream-ordered) d_inst_off[i] = number of segments of all
 *                        instances before i = b*R + k, d_inst_off[B*R] = their total S.  The
 *                        caller reads them and allocates, from S alone:
 *                          d_scratch          MRX_CONTOUR_SCRATCH_BYTES(S) bytes
 *                          d_vertices         float64 [S + S/4, 2]   (every contour has >= 4 segments)
 *                          d_contour_off      int64 [S/4 + 1]
 *                          d_inst_contour_off int64 [B*R + 1]
 *   mrx_contours_write:  total_segments = S, max_inst_segments = the largest d_inst_off[i+1] -
 *                        d_inst_off[i] (it sets the number of pointer-jumping rounds).  Instance i's
 *                        contours are c in [d_inst_contour_off[i], d_inst_contour_off[i+1]), in
 *                        find_contours' order; contour c's vertices are
 *                        d_vertices[d_contour_off[c] .. d_contour_off[c+1]) as (x, y) pairs, the
 *                        first repeated at the end.  The values are exact (integers and halves,
 *                        float64 for every side below 2^30; float32 would round halves past 2^23).
 * S above MRX_MAX_CONTOUR_SEGMENTS: MRX_E_UNSUPPORTED (split the batch). */
#define MRX_MAX_CONTOUR_SEGMENTS (1 << 30)
#define MRX_CONTOUR_SCRATCH_BYTES(S) (48LL * (S) + 256)
int mrx_contours_count(const unsigned char *d_packed, const long long *d_packed_off,
                       const int *d_counts, const int *d_geom, const int *d_regions,
                       int *d_row_off, long long *d_inst_off, int B, int R, int max_h,
                       void *stream);
int mrx_contours_write(const unsigned char *d_packed, const long long *d_packed_off,
                       const int *d_counts, const int *d_geom, const int *d_regions,
                       const int *d_row_off, const long long *d_inst_off, long long total_segments,
                       long long max_inst_segments, void *d_scratch, double *d_vertices,
                       long long *d_contour_off, long long *d_inst_contour_off, int B, int R,
                       int max_h, void *stream);

/* EXTENSION: the boxes, contour outlines and captions visualize.display_instances draws over the
 * overlay (serve.py:160-169), as these OpenCV calls draw them at the image's own resolution
 * (annotate.cu; DESIGN.md section 3.25): for every kept instance k whose box is not all zeros, in
 * order, cv2.rectangle(img, (x1, y1), (x2, y2), col_k, 1, LINE_8) when show_bbox, and
 * cv2.polylines(img, [int32(2 v)], False, col_k, 1, LINE_8, shift=1) for each of its contours v;
 * then every caption, cv2.putText in white.  Two calls:
 *   mrx_annotate_draw:    d_keys: int32 key planes, image b's [H_b, W_b] at d_keys + d_key_off[b]
 *                         (int64, in elements); they are zeroed, then every pixel instance k draws
 *                         does atomicMax(key, k + 1), so a later instance wins.  Box edges are
 *                         clipped to the image.  A contour segment sets its two end points rounded
 *                         half up, ((2x + 1) >> 1, (2y + 1) >> 1), where they lie in the image (what
 *                         LINE_8 with shift=1 draws for every step between edge midpoints).  d_boxes
 *                         [B,R,4] int32 (y1, x1, y2, x2); the contours as mrx_contours_write leaves
 *                         them: d_vertices float64 [n_vertices, 2], d_contour_off, d_inst_contour_off
 *                         [B*R + 1] (instance i = b*R + k); n_vertices = 0 draws no outline (the
 *                         three pointers may then be NULL).
 *   mrx_annotate_resolve: the uint8 [H_b, W_b, 3] images at d_images + d_image_off[b] (int64 bytes)
 *                         in place: a pixel with key k + 1 becomes d_rgb8[b][k] (uint8 [B,R,3]);
 *                         then the P caption patches are set to 255 where their stencil bit is
 *                         set: record p is d_patches[6p .. 6p+5] = (image, y0, x0, h, w, byte
 *                         offset) int64, and patch pixel (y, x) is bit 7 - (j & 7) of
 *                         d_stencils[offset + (j >> 3)], j = y*w + x.  Patch pixels outside their
 *                         image, and records of an image outside [0, B), are not written.
 * max_pixels: the extent of "Output slots".  Checks: null pointers, B outside [0, MRX_MAX_BATCH], R
 * outside [1, 65534], max_pixels outside [0, 2^31 - 1), n_vertices or P below 0: MRX_E_INVALID.
 * B = 0 or max_pixels = 0 returns MRX_OK without launching anything. */
int mrx_annotate_draw(const int *d_counts, const int *d_geom, const int *d_boxes,
                      const double *d_vertices, const long long *d_contour_off,
                      const long long *d_inst_contour_off, long long n_vertices, int show_bbox,
                      int *d_keys, const long long *d_key_off, int B, int R, long long max_pixels,
                      void *stream);
int mrx_annotate_resolve(const int *d_geom, const int *d_keys, const long long *d_key_off,
                         const unsigned char *d_rgb8, unsigned char *d_images,
                         const long long *d_image_off, const unsigned char *d_stencils,
                         const long long *d_patches, int P, int B, int R, long long max_pixels,
                         void *stream);

/* ---------------------------------------------------------------- mask IoU and matches */
/* EXTENSION: upstream mrcnn.utils.compute_overlaps_masks and the matching loop of compute_matches
 * on the packed slots (see "Output slots"), so that scoring predictions against ground truth
 * needs no mask on the host (overlaps.cu).
 *
 * mrx_mask_extents: for every plane k < N_b, d_areas[b][k] (int64) = its set pixels and
 *   d_extents[b][k] (int32 y1, x1, y2, x2, exclusive ends; all 0 for an empty plane) = their tight
 *   bounding box, counted only inside d_regions[b][k] (int32 [B,R,4] y1, x1, y2, x2, required;
 *   clamped to the image, pixels outside count as 0), e.g. the d_boxes of mrx_unmold_prepare,
 *   outside which an expanded plane is zero, or (0, 0, H_b, W_b).
 * mrx_mask_overlaps: two slot sets of one batch (R1 and R2 planes per slot) sharing d_geom, with
 *   their areas and extents from mrx_mask_extents: d_overlaps [B,R1,R2] float32, element (b, i, j)
 *   for i < N1_b, j < N2_b = IoU of plane i of set 1 and plane j of set 2 in NumPy's float32
 *   order, i = f32(inter), u = (f32(a1) + f32(a2)) - i, i / u (NaN when both are empty); other
 *   elements are not written.  d_packed1 and d_packed2 must be 4-byte aligned.
 * mrx_mask_matches: per image b, its N_b = d_pred_counts[b] predictions (d_pred_class_ids [B,R1]
 *   int32, d_scores [B,R1] of score_dtype) and M_b = d_gt_counts[b] ground-truth instances
 *   (d_gt_class_ids [B,R2] int32), d_overlaps as above.  thresholds[T] (HOST, 1 <= T <=
 *   MRX_MAX_IOU_THRESHOLDS) and score_threshold are compared with (double)IoU.  Writes
 *     d_order [B,R1] int32: rank -> prediction, by score descending, NaN first, ties larger
 *                           index first;
 *     d_pred_match [T,B,R1] int32 by rank: the matched ground-truth index or -1;
 *     d_gt_match   [T,B,R2] int32: the rank of the prediction that matched it or -1.
 *   The prediction of rank r takes, among the ground truth still unmatched and of its class whose
 *   IoU is NaN or >= both thresholds, the one with the largest IoU (NaN above every number, ties
 *   the larger index): what compute_matches' loop picks.
 * Checks: those of "Output slots" for each slot set (mrx_mask_extents, mrx_mask_overlaps), then
 * null pointers; for mrx_mask_matches null pointers, B outside [0, MRX_MAX_BATCH], R1 or R2
 * outside [1, 65534], T outside [1, MRX_MAX_IOU_THRESHOLDS] or a bad score_dtype: MRX_E_INVALID.
 * B = 0 returns MRX_OK without launching anything. */
#define MRX_MAX_IOU_THRESHOLDS 64
int mrx_mask_extents(const unsigned char *d_packed, const long long *d_packed_off,
                     const int *d_counts, const int *d_geom, const int *d_regions,
                     long long *d_areas, int *d_extents, int B, int R, void *stream);
int mrx_mask_overlaps(const unsigned char *d_packed1, const long long *d_packed_off1,
                      const int *d_counts1, const long long *d_areas1, const int *d_extents1,
                      int R1, const unsigned char *d_packed2, const long long *d_packed_off2,
                      const int *d_counts2, const long long *d_areas2, const int *d_extents2,
                      int R2, const int *d_geom, float *d_overlaps, int B, void *stream);
int mrx_mask_matches(const float *d_overlaps, const int *d_pred_counts,
                     const int *d_pred_class_ids, const void *d_scores, int score_dtype,
                     const int *d_gt_counts, const int *d_gt_class_ids, const double *thresholds,
                     int T, double score_threshold, int *d_order, int *d_pred_match,
                     int *d_gt_match, int B, int R1, int R2, void *stream);

/* ---------------------------------------------------------------- COCO mask and box evaluation */
/* EXTENSION: the per-image half of pycocotools' COCOeval for iouType "segm" (computeIoU with
 * maskApi.c's rleIou on the packed slots, see "Output slots") and "bbox" (computeIoU with
 * maskApi.c's bbIou), and the matching loop of evaluateImg for both; the host accumulates the
 * per-detection flags (cocoeval.cu).  Categories are dense indices >= 0; -1 is a category that
 * is not evaluated.
 *
 * mrx_coco_ranks: per image b, its N_b = d_counts[b] predictions (d_class_ids [B,R] int32,
 *   d_scores [B,R] of score_dtype), d_class_map [C] int32 (class id -> dense category or -1; a
 *   class id outside [0, C) is -1).  Writes, for k < N_b,
 *     d_cat  [B,R] int32: the dense category;
 *     d_rank [B,R] int32: the rank within (image, category) in np.argsort(-score,
 *                         kind="mergesort") order: descending, equal scores by smaller index,
 *                         NaN after every number;
 *     d_keep [B,R] uint8: d_cat >= 0 and d_rank < max_det (maxDets[-1]);
 *     d_walk [B,R] int32: rank -> prediction in that order across categories.
 * mrx_coco_ious: two slot sets of one batch sharing d_geom, with areas and extents from
 *   mrx_mask_extents; d_pred_cat / d_pred_keep from mrx_coco_ranks, d_gt_cat [B,R2] int32 and
 *   d_gt_crowd [B,R2] uint8 (iscrowd).  d_iou [B,R1,R2] float64: element (b, i, j) for a kept
 *   i < N1_b and j < N2_b of the same category is (double)inter / (double)u rounded once, 0 when
 *   inter = 0, u = area(i) for a crowd j and area(i) + area(j) - inter otherwise; other elements
 *   are not written.  d_packed1 and d_packed2 must be 4-byte aligned.
 * mrx_coco_box_ious: the same d_iou for boxes.  d_pred_boxes [B,R1,4] is, by box_form,
 *   MRX_BOX_YXYX_I32: int32 (y1, x1, y2, x2), e.g. the d_boxes of mrx_unmold_prepare, taken as
 *     [x1, y1, x2 - x1, y2 - y1] (build_coco_results' `bbox`, exact in double), or
 *   MRX_BOX_XYWH_F64: float64 [x, y, w, h], a result's `bbox`;
 *   d_pred_counts [B], d_pred_cat / d_pred_keep from mrx_coco_ranks; d_gt_boxes [B,R2,4] float64
 *   [x, y, w, h], d_gt_counts [B], d_gt_cat [B,R2] int32, d_gt_crowd [B,R2] uint8.  Element
 *   (b, i, j) for a kept i < N1_b and j < N2_b of the same category is bbIou's, every operation
 *   rounded on its own (no FMA): w = fmin(D[2]+D[0], G[2]+G[0]) - fmax(D[0], G[0]), 0 when
 *   w <= 0, h the same in y, i = w*h, u = D[2]*D[3] for a crowd j and (D[2]*D[3] + G[2]*G[3]) - i
 *   otherwise, i / u.  Also writes d_pred_area [B,R1] float64 = D[2]*D[3] for kept i (loadRes'
 *   `area` of a bbox result).  Other elements are not written.
 * mrx_coco_match: d_iou as above, the ranks' d_pred_cat, d_pred_keep and d_walk, d_pred_area
 *   [B,R1] int64 (mask pixels; mrx_coco_match_f64area: float64, the box areas of
 *   mrx_coco_box_ious), d_gt_counts [B], d_gt_cat, d_gt_crowd, d_gt_area [B,R2] float64
 *   (the annotation's area).  thresholds[T] (HOST, compared as IoU >= t: the caller caps them at
 *   1 - 1e-10 as evaluateImg does) and area_rng[A][2] (HOST, lo and hi, both inclusive).  For
 *   area range a and threshold t, ground-truth j is ignored when crowd or its area is outside
 *   [lo, hi]; predictions go in walk order, each kept one takes, among the instances of its
 *   category that are unmatched or crowd with IoU >= t, the non-ignored one with the largest IoU,
 *   else the ignored one with the largest IoU, ties the larger index.  Writes, for kept i,
 *     d_dt_match  [A,T,B,R1] int32: the matched ground-truth index or -1;
 *     d_dt_ignore [A,T,B,R1] uint8: the matched instance's ignore flag, or for an unmatched
 *                                   prediction whether its area is outside [lo, hi].
 *   Other elements are not written.
 * Checks: mrx_coco_ious: those of "Output slots" for each slot set, then null pointers and the
 * alignment; the others: null pointers, B outside [0, MRX_MAX_BATCH], R (R1, R2) outside
 * [1, 65534], for mrx_coco_ranks C or max_det below 1 or a bad score_dtype, for
 * mrx_coco_box_ious a bad box_form, for mrx_coco_match[_f64area] T outside
 * [1, MRX_MAX_IOU_THRESHOLDS] or A outside [1, MRX_MAX_AREA_RANGES]: MRX_E_INVALID.
 * B = 0 returns MRX_OK without launching anything. */
#define MRX_MAX_AREA_RANGES 16
#define MRX_BOX_YXYX_I32 0
#define MRX_BOX_XYWH_F64 1
int mrx_coco_ranks(const int *d_class_ids, const void *d_scores, int score_dtype,
                   const int *d_counts, const int *d_class_map, int C, int max_det, int *d_cat,
                   int *d_rank, unsigned char *d_keep, int *d_walk, int B, int R, void *stream);

/* mrx_lvis_ranks: the rank step of lvis-api's LVISEval (LVISResults.limit_dets_per_image and the
 *   federated filter of LVISEval._prepare); the IoUs and matches that follow are
 *   mrx_coco_[box_]ious and mrx_coco_match[_f64area] with all-zero crowd flags.  Arguments as for
 *   mrx_coco_ranks, plus d_status [B,K] uint8: bit MRX_LVIS_POSITIVE when image b has ground truth
 *   of dense category k, MRX_LVIS_NEGATIVE when k is in its neg_category_ids (and
 *   MRX_LVIS_NOT_EXHAUSTIVE, for the host, when k is in its not_exhaustive_category_ids; not read
 *   here).  d_cat, d_rank and d_walk are mrx_coco_ranks's; d_keep [B,R] uint8 is d_cat in
 *   [0, K), the walk position (the number of the image's predictions before it, whatever their
 *   category) below max_det, and d_status[b][d_cat] & MRX_LVIS_EVALUATED.  Checks: those of
 *   mrx_coco_ranks, and K below 1: MRX_E_INVALID. */
#define MRX_LVIS_POSITIVE 1
#define MRX_LVIS_NEGATIVE 2
#define MRX_LVIS_EVALUATED 3
#define MRX_LVIS_NOT_EXHAUSTIVE 4
int mrx_lvis_ranks(const int *d_class_ids, const void *d_scores, int score_dtype,
                   const int *d_counts, const int *d_class_map, int C, const unsigned char *d_status,
                   int K, int max_det, int *d_cat, int *d_rank, unsigned char *d_keep, int *d_walk,
                   int B, int R, void *stream);
int mrx_coco_ious(const unsigned char *d_packed1, const long long *d_packed_off1,
                  const int *d_counts1, const long long *d_areas1, const int *d_extents1,
                  const int *d_pred_cat, const unsigned char *d_pred_keep, int R1,
                  const unsigned char *d_packed2, const long long *d_packed_off2,
                  const int *d_counts2, const long long *d_areas2, const int *d_extents2,
                  const int *d_gt_cat, const unsigned char *d_gt_crowd, int R2, const int *d_geom,
                  double *d_iou, int B, void *stream);
int mrx_coco_match(const double *d_iou, const int *d_pred_counts, const int *d_pred_cat,
                   const unsigned char *d_pred_keep, const int *d_walk,
                   const long long *d_pred_area, const int *d_gt_counts, const int *d_gt_cat,
                   const unsigned char *d_gt_crowd, const double *d_gt_area,
                   const double *thresholds, int T, const double *area_rng, int A,
                   int *d_dt_match, unsigned char *d_dt_ignore, int B, int R1, int R2,
                   void *stream);
int mrx_coco_match_f64area(const double *d_iou, const int *d_pred_counts, const int *d_pred_cat,
                           const unsigned char *d_pred_keep, const int *d_walk,
                           const double *d_pred_area, const int *d_gt_counts, const int *d_gt_cat,
                           const unsigned char *d_gt_crowd, const double *d_gt_area,
                           const double *thresholds, int T, const double *area_rng, int A,
                           int *d_dt_match, unsigned char *d_dt_ignore, int B, int R1, int R2,
                           void *stream);
int mrx_coco_box_ious(const void *d_pred_boxes, int box_form, const int *d_pred_counts,
                      const int *d_pred_cat, const unsigned char *d_pred_keep, int R1,
                      const double *d_gt_boxes, const int *d_gt_counts, const int *d_gt_cat,
                      const unsigned char *d_gt_crowd, int R2, double *d_pred_area, double *d_iou,
                      int B, void *stream);

/* ---------------------------------------------------------------- Boundary IoU evaluation */
/* EXTENSION: COCOeval for iouType "boundary" (Cheng et al., "Boundary IoU", CVPR 2021; the
 * boundary_iou_api restatement of pycocotools), whose computeIoU takes the smaller of the mask IoU
 * and the IoU of the masks' boundaries; ranks and matches are mrx_coco_ranks and mrx_coco_match.
 *
 * mrx_mask_boundary: for every plane k < N_b of the packed slots (see "Output slots"), its
 *   boundary plane into d_boundary at the same slot offsets (d_packed_off): mask AND NOT the mask
 *   eroded by a (2d+1) x (2d+1) square, d = d_dilation[b] (int32 [B], the caller's
 *   max(1, round(ratio * sqrt(H_b^2 + W_b^2))); a d below 1 is taken as 1), counting every pixel
 *   outside d_regions[b][k] (int32 [B,R,4] y1, x1, y2, x2, required, clamped to the image) as 0:
 *   boundary_iou_api's mask_to_boundary (cv2.erode of the mask padded with one zero pixel, d
 *   iterations of a 3 x 3 kernel) when the plane is zero outside its region, e.g. an expanded
 *   plane and its d_boxes of mrx_unmold_prepare, or any plane and (0, 0, H_b, W_b).  A d at or
 *   above the region's height or width erodes everything: the boundary is the mask.  Written:
 *   every byte of the plane that holds a pixel of the region, its bits outside the region 0;
 *   other bytes are not written, and readers that stay inside the region (mrx_mask_extents with
 *   the same regions, the pair walk of mrx_coco_boundary_ious) never see them.  The boundary of a
 *   mask has the mask's tight extents.  d_boundary must not overlap d_packed.  max_w: the extent
 *   of "Output slots", at least 1; rows wider than the device's shared memory holds return
 *   MRX_E_UNSUPPORTED (on an H100, max_w above 116 224).  Areas: mrx_mask_extents over
 *   d_boundary with the same regions.
 * mrx_coco_boundary_ious: mrx_coco_ious's arguments plus each side's boundary planes (d_boundary1,
 *   d_boundary2, in the slots of d_packed1, d_packed2; 4-byte aligned) and their areas
 *   (d_boundary_areas1, d_boundary_areas2 [B,R] int64); the extents are the masks'.  Element
 *   (b, i, j) for a kept i < N1_b and j < N2_b of the same category is fmin(mask IoU, boundary
 *   IoU), each as mrx_coco_ious computes it (exact counts, one rounding, 0 when the intersection
 *   is 0, the crowd union = the detection's area: its boundary area for the boundary IoU).  Other
 *   elements are not written.
 * Checks: those of "Output slots" (for mrx_coco_boundary_ious, for each slot set), then
 * mrx_mask_boundary: a null d_regions, a null d_dilation or d_boundary, max_w below 1;
 * mrx_coco_boundary_ious: null areas or extents, null pointers, the alignment of the packed and
 * then of the boundary bases: MRX_E_INVALID.  B = 0 returns MRX_OK without launching anything. */
int mrx_mask_boundary(const unsigned char *d_packed, const long long *d_packed_off,
                      const int *d_counts, const int *d_geom, const int *d_regions,
                      const int *d_dilation, unsigned char *d_boundary, int B, int R, int max_w,
                      void *stream);
int mrx_coco_boundary_ious(const unsigned char *d_packed1, const long long *d_packed_off1,
                           const int *d_counts1, const long long *d_areas1, const int *d_extents1,
                           const unsigned char *d_boundary1, const long long *d_boundary_areas1,
                           const int *d_pred_cat, const unsigned char *d_pred_keep, int R1,
                           const unsigned char *d_packed2, const long long *d_packed_off2,
                           const int *d_counts2, const long long *d_areas2, const int *d_extents2,
                           const unsigned char *d_boundary2, const long long *d_boundary_areas2,
                           const int *d_gt_cat, const unsigned char *d_gt_crowd, int R2,
                           const int *d_geom, double *d_iou, int B, void *stream);

/* ---------------------------------------------------------------- COCO RLE to packed planes */
/* EXTENSION: the inverse of mrx_rle_strings / mrx_rle_write, for ground truth held as COCO RLE
 * (pycocotools' compressed strings or uncompressed count lists; rle_decode.cu).  Instance
 * i = b*R + k for k < N_b = d_counts[b]; others are not read or written.
 *
 * mrx_rle_parse: the "counts" strings of mask.encode, instance i's at
 *   d_str[d_str_off[i] .. d_str_off[i+1]) (d_str_off [B*R+1] int64), in the format of
 *   mrx_rle_strings.  A string of L characters holds at most L runs: they go to
 *   d_runs + d_str_off[i] (uint32), their number to d_run_count[i], and the instance's status
 *   word (MRX_RLE_ST_* bits of CHAR, TRUNC, RANGE) to d_status[i].  An instance with an empty
 *   string is left alone (its runs, count and status are the caller's: how a batch mixes strings
 *   with uploaded count lists).
 * mrx_rle_decode: instance i's d_run_count[i] runs (column-major, starting with zeros) at
 *   d_runs + d_run_off[i] (d_run_off [B*R] int64) into the packed slots (see "Output slots"):
 *   every byte of planes k < N_b, pad bits included, is written, so no memset is needed.
 *   d_run_end: int64 scratch indexed like d_runs (the run ends).  d_status [B*R]: as
 *   mrx_rle_parse left it (or zeroed by the caller); MRX_RLE_ST_SUM is added when the runs do not
 *   sum to H_b*W_b.  The plane of an instance with any status bit is unspecified; whatever its
 *   runs say, nothing outside that plane is written.  max_h, max_w: the extents of
 *   "Output slots", at least 1.
 * Checks: mrx_rle_parse: null pointers, B outside [0, MRX_MAX_BATCH] or R outside [1, 65534]:
 * MRX_E_INVALID.  mrx_rle_decode: those of "Output slots", then null pointers and the extents.
 * B = 0 returns MRX_OK without launching anything.  Areas and extents: mrx_mask_extents with the
 * whole image as region.  The plane of an instance whose status word has any bit is not written;
 * a batch that mixes RLE with another path (mrx_poly_decode) sets MRX_RLE_ST_SKIP in the status
 * of that path's instances (empty strings, no runs) before the decode, and ignores their status
 * afterwards. */
#define MRX_RLE_ST_CHAR   1   /* a character outside '0' .. '0' + 63 */
#define MRX_RLE_ST_TRUNC  2   /* the string ends inside a value */
#define MRX_RLE_ST_RANGE  4   /* a count negative or above 2^32 - 1 (or a value of > 7 groups) */
#define MRX_RLE_ST_SUM    8   /* the counts do not sum to H*W */
#define MRX_RLE_ST_SKIP  16   /* set by the caller: another path writes the plane */
int mrx_rle_parse(const unsigned char *d_str, const long long *d_str_off, const int *d_counts,
                  unsigned int *d_runs, int *d_run_count, int *d_status, int B, int R,
                  void *stream);
int mrx_rle_decode(const unsigned int *d_runs, const long long *d_run_off, const int *d_run_count,
                   long long *d_run_end, int *d_status, const int *d_counts, const int *d_geom,
                   const long long *d_packed_off, unsigned char *d_packed, int B, int R,
                   int max_h, int max_w, void *stream);

/* ---------------------------------------------------------------- COCO polygons to packed planes */
/* EXTENSION: pycocotools' annToRLE of a polygon annotation (frPyObjects: rleFrPoly per part, then
 * rleMerge with intersect = 0, the union of the parts) decoded, into the packed slots (see
 * "Output slots"; polygons.cu).  Instance i = b*R + k for k < N_b = d_counts[b].
 *
 * d_vert [V, 2] int32: the vertices (x, y) of every part, each coordinate rleFrPoly's
 *   (int)(5.0 * c + .5) (the caller scales and rounds them, and checks that they and the
 *   differences of consecutive vertices fit in int); part p's nv_p >= 1 vertices at
 *   d_part_vert[p] .. d_part_vert[p+1] (d_part_vert [P+1] int64), closed from the last to the
 *   first.  d_part_inst [P] int32: the instance i of part p.  d_inst_part [B*R+1] int32: instance
 *   i's parts are d_inst_part[i] .. d_inst_part[i+1], an instance's parts consecutive.
 * Scratch: d_col_start [C] int64 and d_carry [C] uint8, part p's W_b + 1 entries from
 *   d_part_col[p] (d_part_col [P] int64); d_tog int32, part p's toggle rows at d_part_tog[p] ..
 *   d_part_tog[p+1] (d_part_tog [P+1] int64), at least sum over its edges of
 *   min(W_b, (|dx| + 2) / 5 + 1) + 1 entries (dx: the edge's scaled x difference).
 * Every byte of the plane k < N_b of an instance with parts, pad bits included, is written, so no
 * memset is needed; the planes of instances without parts are not touched.  Positions are int64
 * (pycocotools' int positions overflow once H*W >= 2^31).  max_h, max_w: the extents of "Output
 * slots", at least 1.
 * Checks: those of "Output slots", then null pointers, P below 0 and the extents: MRX_E_INVALID.
 * B = 0 or P = 0 returns MRX_OK without launching anything.  Areas and extents: mrx_mask_extents
 * with the whole image as region. */
int mrx_poly_decode(const int *d_vert, const long long *d_part_vert, const int *d_part_inst,
                    const long long *d_part_col, const long long *d_part_tog, int P,
                    const int *d_inst_part, int *d_tog, long long *d_col_start,
                    unsigned char *d_carry, const int *d_counts, const int *d_geom,
                    const long long *d_packed_off, unsigned char *d_packed, int B, int R,
                    int max_h, int max_w, void *stream);

/* ---------------------------------------------------------------- JPEG decode (load_img) */
/* Baseline JPEG files decoded bit for bit as cv2.imdecode(buf, IMREAD_COLOR) then BGR2RGB
 * (libjpeg-turbo: JDCT_ISLOW, fancy upsampling, EXIF orientation; csrc/jpeg.cu).  The host
 * (jpeg.Plan) parses the headers and lays the batch out: the files at d_files + desc[b][0],
 * desc [B, 80] int64 words per image (geometry and every buffer offset, jpeg.py's D_* indices),
 * d_tabs [B, 9312] bytes (per component: quant int32[64] in natural order, DC and AC Huffman
 * lookups), d_unit_img [U] int32 (the image of each of the batch's U restart units).
 *
 * mrx_jpeg_coefficients: unstuffs each scan into d_unst, splits it at RSTn into units, decodes the
 *   Huffman data by self-synchronisation over subsequences of S bits (scratch in d_work) and
 *   writes the quantised coefficients, int16 [blocks, 64] in natural order and decode (MCU) order,
 *   DC after the prediction (JCOEF), into d_coef (zeroed here first; coef_blocks of them) at
 *   desc's block offsets.  d_status [B] int32 (zeroed here first) gets MRX_JPEG_ST_* bits for
 *   corrupt entropy-coded data; libjpeg-turbo warns and substitutes zeros instead (a stated
 *   difference).  max_subs: the largest per-image subsequence count desc plans, which is the S
 *   desc was planned with.
 * mrx_jpeg_pixels: the islow IDCT of every block into the component planes (d_planes, at their
 *   full padded block size), then upsampling, colour conversion and orientation into uint8 RGB
 *   [H', W', 3] at d_out + d_out_off[b] -- the source slots mrx_cv2_resize_u8c3_batch reads.
 *   Images whose status word has a bit are not written.  max_blocks, max_pixels: the largest
 *   per-image block and pixel counts.
 * Checks: null pointers, B outside [0, MRX_MAX_BATCH], S not a multiple of 32 in [32, 65536],
 * U below B, a max extent below 1: MRX_E_INVALID.  B = 0 returns MRX_OK without launching
 * anything. */
#define MRX_JPEG_ST_CODE   1   /* a bad Huffman code */
#define MRX_JPEG_ST_TRUNC  2   /* the data ends before the last MCU */
#define MRX_JPEG_ST_RST    4   /* a missing or out-of-order RSTn */
#define MRX_JPEG_ST_DC     8   /* a DC value outside int32 */
#define MRX_JPEG_ST_MARKER 16  /* a marker other than EOI ends the scan (a second scan) */
int mrx_jpeg_coefficients(const unsigned char *d_files, const long long *d_desc,
                          const unsigned char *d_tabs, const int *d_unit_img, int B, int U, int S,
                          int max_subs, unsigned char *d_unst, int *d_work, short *d_coef,
                          long long coef_blocks, int *d_status, void *stream);
int mrx_jpeg_pixels(const long long *d_desc, const unsigned char *d_tabs, const short *d_coef,
                    const int *d_status, int B, int max_blocks, long long max_pixels,
                    unsigned char *d_planes, unsigned char *d_out, const long long *d_out_off,
                    void *stream);

/* Progressive (SOF2) files, decoded into the same coefficient buffer (jpeg.ProgressivePlan lays the
 * batch out; csrc/jpeg.cu).  d_desc and the quantisation part of d_tabs are the image descriptors
 * mrx_jpeg_pixels reads; d_scans [n_scans, 32] int64 words per scan (jpeg.py's S_* indices: image,
 * Ss, Se, Ah, Al, components, the byte range of its entropy-coded data in d_files, restart
 * interval, block grid and the offset of its part of every buffer), scans ordered by round, a
 * scan's round being its dependency level in its file (jpeg.scan_levels); d_scan_tabs [n_scans, 4272] bytes (the Huffman lookup of each
 * component of the scan); d_unit_scan: the scan of each restart unit, units grouped by round;
 * d_round_off [rounds + 1] int32: each round's first unit.
 * mrx_jpeg_progressive_coefficients: unstuffs every scan into d_unst and splits it at RSTn (unit
 *   start bits in d_unit_bit), then decodes round after round, one warp per restart unit, as
 *   jdphuff.c does (DC first, DC refinement, AC first with EOB runs, AC refinement with its
 *   correction bits), into d_coef (zeroed here first).  d_status as for mrx_jpeg_coefficients;
 *   an image with a status bit is skipped by the later rounds.  max_round_units: the most units of
 *   one round.
 * Checks: null pointers, B outside [0, MRX_MAX_BATCH], n_scans outside [B, B * MRX_JPEG_MAX_SCANS],
 * rounds outside [1, MRX_JPEG_MAX_SCANS], a max extent below 1: MRX_E_INVALID.  B = 0
 * returns MRX_OK without launching anything. */
#define MRX_JPEG_MAX_SCANS 256  /* scans of one progressive file */
int mrx_jpeg_progressive_coefficients(const unsigned char *d_files, const long long *d_desc,
                                      const long long *d_scans, const unsigned char *d_scan_tabs,
                                      const int *d_unit_scan, const int *d_round_off, int B,
                                      int n_scans, int rounds, int max_round_units,
                                      unsigned char *d_unst, int *d_unit_bit, short *d_coef,
                                      long long coef_blocks, int *d_status, void *stream);

/* ---------------------------------------------------------------- PNG encode (cv2.imwrite) */
/* uint8 RGB images encoded byte for byte as cv2.imwrite(path, rgb[..., ::-1]) writes them
 * (libpng: Sub filter, or none when the width is 1; zlib level 1, Z_RLE, memLevel 8; 8192-byte
 * IDAT chunks; csrc/png.cu, tests/png_oracle.py).  The host (png.Plan) lays the batch out:
 * d_desc [B, 20] int64 words per image (png.py's D_* indices: the address of the image's
 * contiguous H x W x 3 bytes, H, W, the filtered stream length n = H * (3W + 1), and the offset of
 * the image's part of every buffer below).  Buffers, each sized by png.Plan from H and W alone:
 *   d_stream  uint8 [n] per image (the filtered rows)      d_sym  int16 [n] per image
 *   d_stretch int32 [2 * cap] per image                    d_tiles int64 [2 * (total_tiles + 1)]
 *   d_blk_pos int32 [max blocks + 1] per image             d_blk_tab int32 [blocks, 654]
 *   d_blk_info int64 [blocks, 8] (MRX_PNG_BLK_*)           d_img_info int64 [B, 8] (MRX_PNG_IMG_*)
 *   d_zbuf    uint32 [zbuf_words] (zeroed here; each image's deflate bits at its offset)
 *   d_out     uint8: image b's file at its offset, at most png.png_bound(n) bytes
 *   d_sizes   int64 [B]: the byte count of each file.
 * max_n, max_blocks, max_chunks: the largest n, block count bound and IDAT count bound of the
 * batch.  Checks: null pointers, B outside [0, MRX_MAX_BATCH], max_n outside
 * [4, MRX_PNG_MAX_STREAM], a max extent below 1: MRX_E_INVALID.  B = 0 returns MRX_OK without
 * launching anything. */
#define MRX_PNG_MAX_STREAM (1 << 30)   /* filtered bytes per image: positions stay in int32 */
#define MRX_PNG_BLK_TYPE      0   /* 0 stored, 1 static, 2 dynamic */
#define MRX_PNG_BLK_LAST      1
#define MRX_PNG_BLK_HDR_BITS  2   /* the dynamic tree description */
#define MRX_PNG_BLK_DATA_BITS 3   /* the symbols' codes, extra bits included, end-of-block excluded */
#define MRX_PNG_BLK_EOB       4   /* end-of-block code | length << 16 */
#define MRX_PNG_BLK_BIT       5   /* the block's first bit in the deflate stream */
#define MRX_PNG_BLK_PBASE     6
#define MRX_PNG_BLK_BITS      7   /* the block's bits, stored padding included */
#define MRX_PNG_IMG_NSYM      0
#define MRX_PNG_IMG_NBLK      1
#define MRX_PNG_IMG_BITS      4   /* deflate stream bits */
#define MRX_PNG_IMG_ZLEN      5   /* zlib stream bytes */
#define MRX_PNG_IMG_CHUNKS    6
#define MRX_PNG_IMG_FILE      7
int mrx_png_encode(const long long *d_desc, int B, long long max_n, int max_blocks,
                   long long max_chunks, long long total_tiles, long long zbuf_words,
                   unsigned char *d_stream, short *d_sym, int *d_stretch, long long *d_tiles,
                   int *d_blk_pos, int *d_blk_tab, long long *d_blk_info, unsigned int *d_zbuf,
                   long long *d_img_info, unsigned char *d_out, long long *d_sizes, void *stream);

/* ---------------------------------------------------------------- JPEG encode (cv2.imwrite) */
/* uint8 RGB images encoded byte for byte as cv2.imencode('.jpg', rgb[..., ::-1],
 * [IMWRITE_JPEG_QUALITY, quality, IMWRITE_JPEG_OPTIMIZE, optimize]) writes them (libjpeg-turbo:
 * JFIF 1.01, jpeg_set_quality(quality, force_baseline), YCbCr 4:2:0, ISLOW FDCT, one interleaved
 * baseline scan with the Annex K tables, or with optimize the K.2 optimal tables of the image, no
 * restart markers; csrc/jpeg_encode.cu, tests/jpeg_encode_oracle.py).  The host
 * (jpeg_encode.EncodePlan) lays the batch out: d_desc [B, 16] int64 words per image
 * (jpeg_encode.py's D_* indices: the address of the image's contiguous H x W x 3 bytes, H, W, the
 * MCU grid, the scan's block count nblk = 6 * MCUs, and the offset of the image's part of every
 * buffer below).  Buffers, each sized by jpeg_encode.EncodePlan from H and W alone:
 *   d_huff    uint8 [B, 4, 272]: bits[16] and vals of the tables DC0, AC0, DC1, AC1
 *   d_codes   int32 [B, 4, 256]: code | length << 16 per symbol     d_hist int32 [B, 4, 256]
 *   d_coef    int16 [blocks, 64]: each block's quantised coefficients in zigzag order, MCU order
 *   d_blk_bit int32 [blocks]: each block's first bit within its tile of 256 blocks
 *   d_tiles   int64 [blk_tiles + 1 + byte_tiles + 1]
 *   d_words   uint32 [word_count] (zeroed here): each image's entropy-coded bits, big-endian
 *   d_info    int64 [B, 8] (MRX_JPEG_ENC_*)
 *   d_out     uint8: image b's file at its offset, at most jpeg_encode.file_bound(nblk) bytes
 *   d_sizes   int64 [B]: the byte count of each file.
 * min_side / max_side: the smallest and largest H or W of the batch; max_blocks, max_bytes: the
 * largest nblk and entropy-coded byte bound.  Checks: null pointers, B outside [0, MRX_MAX_BATCH],
 * quality outside [0, 100], optimize not 0 or 1, a max extent below 1: MRX_E_INVALID; a side
 * outside [1, MRX_JPEG_ENC_MAX_SIDE]: MRX_E_UNSUPPORTED.  B = 0 returns MRX_OK without launching
 * anything. */
#define MRX_JPEG_ENC_MAX_SIDE 65535   /* the largest side a baseline frame header holds */
#define MRX_JPEG_ENC_BITS     0   /* entropy-coded bits, padding excluded */
#define MRX_JPEG_ENC_BYTES    1   /* entropy-coded bytes before stuffing */
#define MRX_JPEG_ENC_FF       2   /* 0x00 bytes stuffed after 0xFF */
#define MRX_JPEG_ENC_HDR      3   /* bytes from SOI to the end of SOS */
#define MRX_JPEG_ENC_FILE     4
#define MRX_JPEG_ENC_BLOCKS   5   /* blocks of the scan, dummy blocks included */
#define MRX_JPEG_ENC_INFO_WORDS 8
int mrx_jpeg_encode(const long long *d_desc, int B, int quality, int optimize, int min_side,
                    int max_side, int max_blocks, long long max_bytes, long long blk_tiles,
                    long long byte_tiles, long long word_count, unsigned char *d_huff,
                    int *d_codes, int *d_hist, short *d_coef, int *d_blk_bit, long long *d_tiles,
                    unsigned int *d_words, long long *d_info, unsigned char *d_out,
                    long long *d_sizes, void *stream);

/* ---------------------------------------------------------------- PNG decode (load_img) */
/* PNG files decoded bit for bit as cv2.imdecode(buf, IMREAD_COLOR) then BGR2RGB (libpng:
 * strip_16, gray 1/2/4 expanded by bit replication, palette to RGB with indices past PLTE giving
 * 0,0,0, gray to RGB, alpha dropped, Adam7; EXIF orientation; csrc/png_decode.cu).  The host
 * (png.DecodePlan) parses every chunk but the image data and lays the batch out: the files at
 * d_files, d_desc [B, 16] int64 words per image (png.py's DD_* indices: the image's zlib stream
 * and filtered stream offsets and lengths, geometry, colour type, bit depth, interlace,
 * orientation, palette length, block-list offset and capacity, window size, candidate tiles),
 * d_chunks [n_chunks, 4] int64 words per IDAT chunk (image, file offset of its type, data
 * length, offset in the image's zlib stream), d_plte [B, 768] (each image's palette).  Buffers,
 * each sized by png.DecodePlan from the headers and file lengths alone:
 *   d_z        uint8: each image's IDAT payloads, concatenated (its zlib stream)
 *   d_tile_cnt int32 [total_tiles]: candidate block starts found per tile of
 *              MRX_PNG_DEC_TILE_BITS stream bits (zeroed here first)
 *   d_cand     int64 [total_tiles, K]: their bit positions (the first K of each tile)
 *   d_meas     int64 [total_tiles, K, 4]: each candidate's end bit, bytes, reach before the
 *              block, valid | BFINAL << 1
 *   d_cells    int32: per filtered byte, a value or a reference to an earlier byte
 *   d_filt     uint8: each image's filtered rows, exactly n = sum over passes of rows x (1 + row
 *              bytes), unfiltered in place
 *   d_blocks   int64 [blocks, 2]: per image, the first bit (in its zlib stream) and the output
 *              offset of each block, up to the image's capacity (past it the image is expanded
 *              by one warp, in order)
 *   d_info     int64 [B, MRX_PNG_DEC_INFO_WORDS] (MRX_PNG_DEC_*), zeroed here first
 *   d_status   int32 [B] (zeroed here first): MRX_PNG_ST_* bits; an image with a bit is not written
 *   d_out      uint8 RGB [H', W', 3] at d_out + d_out_off[b]: the slots mrx_jpeg_pixels writes.
 * K: candidate slots per tile, 0 to measure every block in the chain.  An error in the deflate
 * stream is refused when libpng meets it before it has every row (a distance too far back:
 * before it needs a byte past the rows); later ones end the stream, as libpng only warns there.
 * The Adler-32 trailer is checked when the stream holds exactly the image's rows.  max_n,
 * max_pixels, max_zlen, max_tiles, max_blocks: the batch's largest filtered length, pixel count,
 * zlib length, tile count and block capacity.  Checks: null pointers, B outside
 * [0, MRX_MAX_BATCH], n_chunks outside [B, 2^31], max_n outside [2, MRX_PNG_DEC_MAX_FILTERED],
 * max_pixels outside [1, 2^30], max_zlen outside [2, MRX_PNG_DEC_MAX_FILE], K outside
 * [0, MRX_PNG_DEC_MAX_SLOTS], a tile or block extent below 1: MRX_E_INVALID.  B = 0 returns MRX_OK
 * without launching anything. */
#define MRX_PNG_DEC_MAX_FILE     (1 << 27)   /* bytes per file: bit positions stay in int32 */
#define MRX_PNG_DEC_MAX_FILTERED (1 << 30)   /* filtered bytes per image: positions in int32 */
#define MRX_PNG_DEC_TILE_BITS    1024        /* stream bits per candidate tile */
#define MRX_PNG_DEC_MAX_SLOTS    32          /* candidate slots per tile */
#define MRX_PNG_ST_CRC    1    /* an IDAT chunk's CRC-32 */
#define MRX_PNG_ST_TRUNC  2    /* the stream ends before the image's last row or its trailer */
#define MRX_PNG_ST_CODE   4    /* an invalid block type, code set, code or stored length */
#define MRX_PNG_ST_DIST   8    /* a distance past the stream start or the window */
#define MRX_PNG_ST_ADLER  16   /* the Adler-32 trailer of a stream of exactly the image's rows */
#define MRX_PNG_ST_FILTER 32   /* a filter type above 4 */
#define MRX_PNG_DEC_NBLK    0   /* deflate blocks chained */
#define MRX_PNG_DEC_SEQ     1   /* of them, measured by the chain itself */
#define MRX_PNG_DEC_OUT     2   /* bytes the chained blocks describe */
#define MRX_PNG_DEC_ADLER   3   /* the trailer when checked, else -1 */
#define MRX_PNG_DEC_ADLER_A 4
#define MRX_PNG_DEC_ADLER_B 5
#define MRX_PNG_DEC_CAND    6   /* candidate block starts found */
#define MRX_PNG_DEC_INFO_WORDS 8
int mrx_png_decode(const unsigned char *d_files, const long long *d_desc,
                   const long long *d_chunks, const unsigned char *d_plte, int B,
                   long long n_chunks, long long max_n, long long max_pixels, long long max_zlen,
                   long long max_tiles, long long total_tiles, long long max_blocks, int K,
                   unsigned char *d_z, long long *d_cand, int *d_tile_cnt, long long *d_meas,
                   int *d_cells, unsigned char *d_filt, long long *d_blocks, long long *d_info,
                   int *d_status, unsigned char *d_out, const long long *d_out_off, void *stream);

/* ---------------------------------------------------------------- multi-GPU gather (8e) */
/* Peer-memory plumbing for the final gather of the canvases to rank 0 (one process per GPU).
 * Rank 0: mrx_peer_alloc a receive buffer + mrx_peer_export its 64-byte handle; other ranks:
 * mrx_peer_open the handle and pass the mapped address as the OUTPUT pointer of
 * mrx_mask_expand / mrx_mask_expand_packed -- the kernels store over NVLink straight into
 * rank 0's HBM.  mrx_peer_signal(flag, v, stream): after everything queued on `stream` so far,
 * store v to *flag (system scope, release).  mrx_peer_wait(flags, n, v, stream): `stream`
 * proceeds once flags[0..n) are all >= v (acquire).  Flags live in peer-allocated memory. */
#define MRX_PEER_HANDLE_BYTES 64
int mrx_peer_alloc(unsigned long long bytes, void **d_ptr);
int mrx_peer_free(void *d_ptr);
int mrx_peer_export(void *d_ptr, unsigned char *handle64);
int mrx_peer_open(const unsigned char *handle64, void **d_ptr);
int mrx_peer_close(void *d_ptr);
int mrx_peer_signal(unsigned int *d_flag, unsigned int value, void *stream);
int mrx_peer_wait(const unsigned int *d_flags, int n_flags, unsigned int value, void *stream);

/* ---------------------------------------------------------------- canvas memory */
/* Device memory on the current device for the mask canvas, requested as compressible (Hopper's
 * compute data compression: mostly-zero lines take fewer DRAM bytes, reads and writes are
 * unchanged) when the device reports CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, plain
 * otherwise or when the compressible request is refused.  The size is rounded up to the
 * allocation granularity.  *compressed = 1 when the driver granted compression, else 0.
 * mrx_device_free takes the pointer and the byte count given to mrx_device_alloc; it synchronises
 * the device first (as cudaFree does). */
int mrx_device_alloc(unsigned long long bytes, void **d_ptr, int *compressed);
int mrx_device_free(void *d_ptr, unsigned long long bytes);

#ifdef __cplusplus
}
#endif
#endif /* MRX_H_ */
