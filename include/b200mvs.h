/*
 * b200mvs - H100-native (sm_90a) dense multi-view-stereo depth-map engine behind the
 * interface of simonfuhrmann/mve's libs/dmrecon.
 *
 * This is the drop-in boundary: a plain C ABI (no C++/torch types) exported by
 * mve_b200/libb200mvs.so.  The reference has no FFI layer of its own for this path - its
 * boundary is the C++ class mvs::DMRecon in a static library (libs/dmrecon/dmrecon.h:40-68)
 * - so each entry point below names the reference interface it replaces; INTEGRATION.md
 * shows the header-identical mvs::DMRecon shim a maintainer links instead of
 * libmve_dmrecon.a.  All citations are relative to the reference tree.
 *
 * Conventions: every function returns 0 on success or a negative B200MVS_ERR_* code;
 * b200mvs_last_error() gives the message.  No exception crosses this boundary; the C++ shim
 * re-throws the exception types the reference throws (SURVEY.md §8b "Errors").
 * There is NO CPU fallback: b200mvs_create fails when no CUDA device is usable.
 */
#ifndef B200MVS_H
#define B200MVS_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200MVS_OK               0
#define B200MVS_ERR_INVALID_ARG (-1)  /* std::invalid_argument in the reference (dmrecon.cc:37-75)        */
#define B200MVS_ERR_CUDA        (-2)  /* CUDA runtime failure -> std::runtime_error in the shim           */
#define B200MVS_ERR_GLOBAL_VS   (-3)  /* "Global View Selection failed" (dmrecon.cc:222-223)               */
#define B200MVS_ERR_CANCELLED   (-4)  /* progress.cancelled was set (dmrecon.cc:100-104, RECON_CANCELLED) */
#define B200MVS_ERR_OVERFLOW    (-5)  /* frontier buffer capacity exceeded                                 */
#define B200MVS_ERR_UNSUPPORTED (-6)  /* setting outside the range the kernels implement (see below)       */
#define B200MVS_ERR_NO_MEMORY   (-7)  /* one reference view does not fit the device budget on its own      */

#define B200MVS_MAX_GLOBAL_VIEWS 32   /* settings.global_vs_max must be <= 32 (reference default 20)      */
#define B200MVS_MAX_LOCAL_VIEWS  4    /* settings.nr_recon_neighbors must be 1..4 (reference default 4)   */

typedef struct b200mvs_ctx b200mvs_ctx;

/* POD part of mvs::Settings (libs/dmrecon/settings.h:22-52), field for field.
 * filter_width must be 5: the reference hard-codes patchPoints[12] (patch_sampler.cc:96). */
typedef struct b200mvs_settings {
    uint32_t filter_width;        /* settings.h:31  = 5     */
    float    min_ncc;             /* settings.h:32  = 0.3   */
    float    min_parallax;        /* settings.h:33  = 10    */
    float    accept_ncc;          /* settings.h:34  = 0.6   */
    float    min_refine_diff;     /* settings.h:35  = 0.001 */
    uint32_t max_iterations;      /* settings.h:36  = 20    */
    uint32_t nr_recon_neighbors;  /* settings.h:37  = 4     */
    uint32_t global_vs_max;       /* settings.h:38  = 20    */
    int32_t  scale;               /* settings.h:39  = 0     */
    int32_t  use_color_scale;     /* settings.h:40  = 1     */
    float    aabb_min[3];         /* settings.h:44          */
    float    aabb_max[3];         /* settings.h:45          */
    /* Engine knobs (no reference counterpart; DESIGN.md "Frontier schedule").  The reference pops strictly by
     * descending confidence (dmrecon.h:72-76); the GPU advances a whole frontier per round.  Both knobs restrict a
     * round to the most confident queued entries of each view so that the order approaches the reference's:
     *   frontier_band  > 0: only entries within this confidence distance of the view's most confident entry run;
     *   frontier_topk  > 0: only about the K most confident entries of each view run (confidence resolution 1/8192).
     * 0 / 0 (default): every queued entry runs each round (fastest). */
    float    frontier_band;
    uint32_t frontier_topk;
} b200mvs_settings;

/* Fills the defaults of settings.h:22-52. */
void b200mvs_default_settings(b200mvs_settings* s);

/* mvs::Progress (libs/dmrecon/progress.h:27-43); read/written without locks like the reference
 * (fancy_progress_printer.cc:84-91, apps/umve/viewinspect/imageoperations.cc:177-184). */
typedef struct b200mvs_progress {
    volatile int32_t  status;     /* ReconStatus: 0 idle, 1 globalvs, 2 features, 3 queue, 4 saving, 5 cancelled */
    volatile int32_t  cancelled;  /* set from outside (any thread) to cancel THIS view; relayed to the running kernel within
                                     ~0.2 ms, its queue is dropped at the next frontier round, status ends as 5 and its maps
                                     are not written; the other views of the batch go on.  The call returns
                                     B200MVS_ERR_CANCELLED only when every view of the batch was cancelled */
    volatile uint64_t filled;
    volatile uint64_t queue_size;
    volatile uint64_t start_time;
} b200mvs_progress;

/* Result maps of one reference view, caller-owned HOST buffers of width*height pixels at pyramid
 * level settings.scale, row-major - the images DMRecon::start attaches to the view
 * (dmrecon.cc:119-145): depth (1 ch), conf (1 ch), dz (2 ch), plus normal (3 ch, computed but never
 * saved by the reference, single_view.cc:78-81) and the per-pixel local view ids (4 x int32, -1
 * padded, ascending) of the optimisation that wrote the pixel.  Any pointer except depth may be
 * NULL.  width/height are outputs. */
typedef struct b200mvs_maps {
    float*   depth;
    float*   conf;
    float*   dz;
    float*   normal;
    int32_t* view_ids;
    int32_t  width, height;
} b200mvs_maps;

/* One mvs::PatchOptimization (patch_optimization.cc:21-30): inputs and results. */
typedef struct b200mvs_patch_in {
    int32_t x, y;
    float   depth, dz_i, dz_j;
    int32_t n_local;              /* propagated local view ids (0 = run the full local view selection) */
    int32_t local_ids[4];
} b200mvs_patch_in;

typedef struct b200mvs_patch_out {
    float   conf;                 /* computeConfidence() (patch_optimization.cc:114-142) */
    float   depth, dz_i, dz_j;
    float   normal[3];
    int32_t n_local;
    int32_t local_ids[4];         /* ascending view ids, -1 padded */
    int32_t iterations;           /* status.iterationCount */
    int32_t converged;
    int32_t opti_success;
} b200mvs_patch_out;

/* Device-side work counters of one call (DESIGN.md "Measurement"). */
typedef struct b200mvs_stats {
    uint64_t n_opt;               /* patch optimisations executed                               */
    uint64_t n_sample_sets;       /* fused colour+derivative 5x5 sample sets drawn              */
    uint64_t n_rounds;            /* frontier rounds                                            */
    uint64_t n_filled;            /* pixels with conf > 0 (progress.filled)                     */
    uint64_t n_seeds_processed;   /* "Processed N features" (dmrecon.cc:286)                    */
    uint64_t n_seeds_success;     /* "... from which N succeeded optimization" (dmrecon.cc:301) */
    uint64_t n_entries_peak;      /* peak frontier size                                         */
    double   ms_patch_kernel;     /* CUDA-event time of the kernel that runs the patch optimisations (reconstruct: the
                                     persistent frontier kernel, seeds + all rounds in one launch) */
    double   ms_total_device;     /* CUDA-event time first launch -> last launch of the call    */
    uint64_t n_patch_launches;    /* launches of the kernel that runs the patch optimisations   */
    uint64_t n_kernel_launches;   /* all kernel launches of the call                            */
    double   ms_optimise_phases;  /* part of ms_patch_kernel spent in the optimise phases (rest: queue bookkeeping + barriers) */
    uint64_t n_grid_barriers;     /* grid-wide barriers executed by the persistent kernel       */
    double   ms_optimise_thread_phases; /* part of ms_optimise_phases in rounds run one thread per patch       */
    double   ms_sort_phases;      /* grouping the winners of large rounds by tile               */
} b200mvs_stats;

/* ---- lifecycle (mvs::DMRecon ctor/dtor, dmrecon.cc:30-87; ImagePyramidCache, image_pyramid.cc:99-160) ---- */
/* device >= 0: a CUDA device (fails loudly when there is none).  B200MVS_DEVICE_NONE creates a PLANNING context without a
 * GPU: b200mvs_set_view_camera, b200mvs_set_features and b200mvs_global_view_selection work (they are host logic in the
 * reference too); every entry point that computes on images fails with B200MVS_ERR_CUDA - there is no CPU fallback. */
#define B200MVS_DEVICE_NONE (-1)
int  b200mvs_create(int device, int n_views, b200mvs_ctx** out);
void b200mvs_destroy(b200mvs_ctx* ctx);
const char* b200mvs_last_error(const b200mvs_ctx* ctx);   /* the message of the calling thread's last failing call, whichever
                                                              context it was made on (ctx is not used and may be NULL): read
                                                              it from the thread that got the error code */
const char* b200mvs_version(void);

/* ---- inputs ---- */
/* Replaces SingleView::create + SingleView::loadColorImage for one mve::View (single_view.cc:24-66,
 * image_pyramid.cc:56-95): takes the `undistorted` uint8 image (1, 2, 3 or 4 channels; alpha dropped,
 * grey expanded as image_pyramid.cc:65-73) and the mve::CameraInfo fields (camera.h:23-170), builds the
 * Gaussian pyramid on the device.  rgb is a HOST pointer, h x w x channels, row-major. */
int b200mvs_upload_view(b200mvs_ctx* ctx, int view_id, const uint8_t* rgb, int w, int h, int channels,
                        float flen, float paspect, const float ppoint[2],
                        const float rot[9], const float trans[3]);
/* Same with a DEVICE pointer (3 channels) on the ctx's device; `cuda_stream` is a cudaStream_t or NULL.
 * Used for HBM-resident inputs and after an NCCL all-gather of the images (DESIGN.md "Multi-GPU"). */
int b200mvs_upload_view_device(b200mvs_ctx* ctx, int view_id, const uint8_t* rgb_dev, int w, int h,
                               float flen, float paspect, const float ppoint[2],
                               const float rot[9], const float trans[3], void* cuda_stream);
/* Camera and image size only - SingleView::create (single_view.cc:24-53).  The reference creates a SingleView for every
 * valid view but loads colour images only for the master view and its selected neighbours (dmrecon.cc:78,238-240); a
 * caller that wants the same economy registers all cameras, asks b200mvs_global_view_selection which views are needed
 * and uploads only those images - or installs an image source (b200mvs_set_image_source), which loads them on demand.
 * Without a source b200mvs_reconstruct fails with B200MVS_ERR_INVALID_ARG ("color image of view N is not loaded") when a
 * needed image is missing. */
int b200mvs_set_view_camera(b200mvs_ctx* ctx, int view_id, int w, int h, float flen, float paspect,
                            const float ppoint[2], const float rot[9], const float trans[3]);
/* Radial distortion of the images this view is given, as sfmrecon undistorts a view's `original` photo into its
 * `undistorted` image (apps/sfmrecon/sfmrecon.cc:425-437): k2, k4 are CameraInfo::dist[0], dist[1] (camera.h:161-162,
 * meta.ini camera.radial_distortion).  Every later b200mvs_upload_view, b200mvs_upload_view_device and image-source fetch
 * of the view then takes the distorted photo, and level 0 of its pyramid is byte for byte
 * mve::image::image_undistort_k2k4<uint8_t>(photo, flen, k2, k4) (image_tools.h:1731-1769) with the flen the view is
 * registered with.  k2 == k4 == 0 (the default) imports the image unchanged, as the reference's duplicate() does.
 * Changing the values drops a resident pyramid: with an image source the view is fetched again when a call needs it;
 * without one a reconstruction fails with "color image of view N is not loaded" until the view is uploaded again.
 * Cameras and prepared plans are untouched (the geometry stays pinhole, as for the `undistorted` image), no memory is
 * allocated, and it works in a planning context, where it only stores the values.  Non-finite values or a bad view id:
 * B200MVS_ERR_INVALID_ARG. */
int b200mvs_set_view_distortion(b200mvs_ctx* ctx, int view_id, float k2, float k4);
/* Reconstruction mask of a reference view: w x h bytes, row-major, 0 = background (the convention of scene2pset -m).
 * When the view is reconstructed at level `scale` (maps W x H), its pixel (x, y) is background when mask pixel
 * (floor((2x+1) w / 2W), floor((2y+1) h / 2H)) is 0, in integer arithmetic: a mask of the map's size maps one to one, a
 * mask of the photo's size gives the photo pixel under the level pixel's centre.  A feature seed on a background pixel is
 * dropped before the launch (it counts in neither n_seeds_processed nor n_seeds_success), no queue entry is ever made for
 * a background pixel, and background pixels end as unfilled ones do: depth, conf, dz and normal 0, view ids -1; they are
 * not counted in progress.filled or n_filled, and no point of b200mvs_pset_add_reconstruction comes from one.  Foreground
 * pixels follow the unmasked rules.  b200mvs_reconstruct, b200mvs_reconstruct_device and b200mvs_pset_add_reconstruction
 * apply it, with or without a budget.  Masks leave view selection, plans, b200mvs_working_set, b200mvs_plan_batches,
 * b200mvs_optimize_patches and the sampling of neighbour views as they are, and add no device bytes (the mask travels
 * in the batch's own map arrays).  It is not the clip of b200mvs_pset_clip_masks, which deletes points afterwards.
 * The mask is copied to the host; NULL clears it (w and h are then ignored).  A view has one mask: this call replaces a
 * mask of b200mvs_set_view_mask_device and frees its device block.  Plans and pyramids are kept, and it works in a
 * planning context, where it only stores the mask.  A bad view id, or w or h < 1 with a mask: B200MVS_ERR_INVALID_ARG. */
int b200mvs_set_view_mask(b200mvs_ctx* ctx, int view_id, const uint8_t* mask_or_null, int w, int h);
/* The same mask read from DEVICE memory on the context's device: row y of the w x h bytes starts at
 * mask_dev + y * row_pitch (row_pitch >= w).  Every reconstruction gives exactly what b200mvs_set_view_mask gives for the
 * same bytes: the same maps, seeds, counters and points on every route, with or without a budget.
 *   - The bytes are copied into a packed w x h block of the view in device memory, after an event recorded on cuda_stream
 *     (NULL = the legacy default stream); the call returns when the copy is done, so the source may then be reused.
 *   - The block is taken from the context's budget and counted in b200mvs_memory.fixed (and resident) until the mask is
 *     cleared or replaced, or the context is destroyed.  A mask that does not fit gives B200MVS_ERR_NO_MEMORY and leaves
 *     the view's previous mask in place.
 *   - A launch resamples the mask into the batch's map arrays on the device: no host loop and no upload.
 *   - It replaces a host mask of b200mvs_set_view_mask; NULL clears either kind (w, h and row_pitch are then ignored).
 *   - B200MVS_ERR_INVALID_ARG, naming the function and the field, before anything is copied: a bad view id, w or h < 1,
 *     row_pitch < w, a planning context, and a mask_dev in host memory (pinned or pageable) or on another device. */
int b200mvs_set_view_mask_device(b200mvs_ctx* ctx, int view_id, const uint8_t* mask_dev_or_null, int w, int h,
                                 int64_t row_pitch, void* cuda_stream);
/* Prior depth map of a reference view: region growing starts from it as well as from the SfM features.  depth is w x h
 * floats, row-major, in MVE's convention: the distance from the camera centre along the pixel's unit ray, as in a
 * depth-L<s> embedding.  That value does not depend on the level, so it is never rescaled.
 *   - Which pixels seed: an entry that reconstructs the view at level `scale` with a W x H map has the candidate pixels
 *     x = 2 + stride i <= W - 3 and y = 2 + stride k <= H - 3 (a pixel nearer the edge always fails in the PatchSampler
 *     ctor): nx = W >= 5 ? (W - 5) / stride + 1 : 0 columns and, by the same rule, ny rows.  Candidate (x, y) reads prior
 *     pixel (floor((2x+1) w / 2W), floor((2y+1) h / 2H)), the pixel rule of b200mvs_set_view_mask, and is a seed when
 *     that value is finite and > 0 and the pixel is not background under the view's mask.
 *   - A prior seed is what a feature seed is: no local views, conf 0, the prior depth and dz 0, so the seed round runs
 *     the full local view selection for it (b200mvs_set_view_prior_state also carries dz and local views).  Prior seeds come after every feature seed of the launch; per pixel the
 *     most confident seed wins and the earlier one wins a tie, so a feature seed beats a prior seed of equal confidence.
 *     n_seeds_processed and n_seeds_success count the prior seeds that were made.
 *   - Every reconstruction entry point applies it: b200mvs_reconstruct[_levels][_device] and
 *     b200mvs_pset_add_reconstruction[_levels].  b200mvs_optimize_patches does not.
 *   - b200mvs_working_set[_levels] and b200mvs_plan_batches[_levels] count an entry's candidate bound nx x ny as seeds,
 *     as they count feature seeds; a view without a prior gives what it gives without this call.  A launch group whose
 *     feature seeds and candidate bounds exceed 2^31 - 1 fails with B200MVS_ERR_INVALID_ARG before anything runs
 *     (failed_view receives one of its views).
 *   - The prior is copied into a packed w x h float block of the view in device memory, taken from the context's budget
 *     and counted in b200mvs_memory.fixed (and resident) until it is cleared or replaced, or the context is destroyed.
 *     A prior that does not fit gives B200MVS_ERR_NO_MEMORY and leaves the previous one in place.  A new prior replaces
 *     the old one and frees its block; NULL clears it (w, h and stride are then ignored).  Plans and pyramids are kept.
 *   - B200MVS_ERR_INVALID_ARG, naming the function and the field, before anything is copied: a bad view id, w or h < 1,
 *     stride outside 1..65535, and a planning context (the prior lives on the device). */
int b200mvs_set_view_prior(b200mvs_ctx* ctx, int view_id, const float* depth_or_null, int w, int h, int stride);
/* The same prior read from DEVICE memory on the context's device: row y of the w x h floats starts at
 * depth_dev + y * row_pitch bytes.  Every reconstruction gives exactly what b200mvs_set_view_prior gives for the same
 * values.  The copy runs after an event recorded on cuda_stream (NULL = the legacy default stream), and the call returns
 * when it is done, so the source may then be reused.  Its checks, plus row_pitch < 4 w or not a multiple of 4, and a
 * depth_dev in host memory (pinned or pageable), on another device or not 4-byte aligned. */
int b200mvs_set_view_prior_device(b200mvs_ctx* ctx, int view_id, const float* depth_dev_or_null, int w, int h,
                                  int64_t row_pitch, int stride, void* cuda_stream);
/* A prior with the rest of a queue entry's state (QueueData, dmrecon.h:28-38): next to the w x h depth map, an optional
 * w x h x 2 float dz map and an optional w x h x 4 int32 view-id map, as the dz and view_ids maps of an earlier
 * reconstruction hold them.  b200mvs_set_view_prior(d) is this call with dz and view_ids NULL.
 *   - Which candidates seed is the rule of b200mvs_set_view_prior, unchanged.  Candidate (x, y) of an entry with a W x H
 *     map reads the prior pixel (px, py) of that rule.
 *   - dz: the seed's dz is the prior's, scaled to the entry's pixel size in float32: dz_i = dz[py][px][0] * ((float)w /
 *     (float)W) and dz_j = dz[py][px][1] * ((float)h / (float)H) (a dz is a depth change per map pixel, and one prior
 *     pixel spans W / w map pixels).  If either is not finite, or there is no dz map, the seed's dz is (0, 0).
 *   - Local views: the distinct ids >= 0 among the four at (px, py) that are in the entry's global view selection.  If
 *     exactly nr_recon_neighbors (N) remain, the seed carries them as its local views, so the seed round skips the local
 *     view selection for it, as b200mvs_optimize_patches does with n_local = N.  Otherwise, or without an id map, it
 *     carries none and runs the full selection.  (The reference propagates 0 or N local views, never a part of a set.)
 *   - A dz map of zeros and an id map of -1 give what no map gives: the same maps, counters and b200mvs_memory_stats
 *     apart from the blocks' bytes.  b200mvs_working_set and b200mvs_plan_batches are unchanged: the bound is the same.
 *   - A view has one prior.  Depth, dz and ids are copied into packed blocks of 4, 8 and 16 B per prior pixel, a block
 *     only for a plane that is given, taken from the budget and counted in b200mvs_memory.fixed (and resident).  Any
 *     prior call replaces every plane; one that does not fit gives B200MVS_ERR_NO_MEMORY and leaves the previous prior
 *     whole.  NULL depth (with NULL dz and view_ids) clears the prior and frees every block.
 *   - B200MVS_ERR_INVALID_ARG, naming the function and the field, before anything is copied: the checks of
 *     b200mvs_set_view_prior, and dz or view_ids given with a NULL depth. */
int b200mvs_set_view_prior_state(b200mvs_ctx* ctx, int view_id, const float* depth_or_null, const float* dz_or_null,
                                 const int32_t* view_ids_or_null, int w, int h, int stride);
/* The same from DEVICE memory on the context's device: row y of each plane starts at y * <plane>_pitch bytes.  Every
 * reconstruction gives exactly what b200mvs_set_view_prior_state gives for the same values.  The stream and the return
 * are those of b200mvs_set_view_prior_device.  Its checks, plus depth_pitch < 4 w, dz_pitch < 8 w, ids_pitch < 16 w or a
 * given plane's pitch not a multiple of 4, and a given plane in host memory, on another device or not 4-byte aligned. */
int b200mvs_set_view_prior_state_device(b200mvs_ctx* ctx, int view_id, const float* depth_dev_or_null,
                                        const float* dz_dev_or_null, const int32_t* view_ids_dev_or_null, int w, int h,
                                        int64_t depth_pitch, int64_t dz_pitch, int64_t ids_pitch, int stride,
                                        void* cuda_stream);
/* What a relative prior's values are (b200mvs_set_view_prior_relative): z is planar depth, d a value of the map. */
enum { B200MVS_PRIOR_DISPARITY = 0,      /* 1/z = s d + t  (relative inverse-depth models)  */
       B200MVS_PRIOR_DEPTH = 1,          /*   z = s d + t  (affine-invariant depth models)  */
       B200MVS_PRIOR_DEPTH_SCALE = 2 };  /*   z = s d      (metric models, SfM scale unknown) */
typedef struct b200mvs_prior_fit {
    double   scale, shift;               /* s, t as installed (shift 0 for DEPTH_SCALE)         */
    uint32_t n_obs, n_inliers;           /* usable feature observations, final inliers           */
    double   median_rel_err;             /* lower median of |z_fit - z| / z over the inliers     */
} b200mvs_prior_fit;
/* A prior from a map known only up to a transform, such as a monocular network's disparity or depth: the view's
 * registered features fix s and t on the device, and the map, turned into depth in MVE's convention, is installed as
 * b200mvs_set_view_prior would install it.  values is w x h floats, row-major; kind is a B200MVS_PRIOR_* above.
 *   - Observations: every registered feature X (b200mvs_set_features) whose refs contain the view.  Xc = R X + t with the
 *     view's float rot and trans widened to double, z = Xc.z, which must be > 0.  u = ax Xc.x / z + cx and
 *     v = ay Xc.y / z + cy, with ax, ay, cx, cy the float level-0 calibration of the view (fill_calibration of its
 *     registered W0 x H0) widened to double; each expression is evaluated left to right.  The prior pixel
 *     (floor(u w / W0), floor(v h / H0)) must lie inside the w x h map, and its value d must be finite and > 0.  The
 *     observation is (d, y) with y = 1/z for DISPARITY and y = z for the two depth kinds.
 *   - Fit, in double.  med is the lower median, element floor((n - 1) / 2) in ascending order, by exact selection.
 *     Fewer than 16 observations fail.  Start: DEPTH_SCALE s = med(y/d), t = 0; the other kinds s = MAD(y) / MAD(d) and
 *     t = med(y) - s med(d), with MAD(v) = med(|v - med v|); MAD(d) = 0 fails.  Then 3 rounds: r = y - (s d + t),
 *     sigma = 1.4826 med(|r|) over all observations, the inliers are those with |r| <= 3 sigma (fewer than 16 fail), and
 *     s, t are refit by least squares over them: s = sum(d y) / sum(d^2) for DEPTH_SCALE, else the centred solution
 *     s = sum((d - dm)(y - ym)) / sum((d - dm)^2), t = ym - s dm; a zero denominator fails.  The inliers are then counted
 *     once more with the final s and t by the same rule.  s <= 0, or s or t not finite, fails.  These constants are fixed.
 *   - median_rel_err: z = 1/y for DISPARITY, else y; z_fit = 1/(s d + t) for DISPARITY, else s d + t.
 *   - Apply: prior pixel (px, py) with a finite d > 0 gets z = s d + t (1/(s d + t) for DISPARITY),
 *     a = ((px + 0.5) W0 / w - cx) / ax, b = ((py + 0.5) H0 / h - cy) / ay and depth = (float)(z sqrt(a a + b b + 1)),
 *     each product and sum rounded on its own (no fused multiply-add).  Every other pixel, and every pixel whose z is not
 *     finite or is <= 0, is 0.
 *   - The depth map is installed as b200mvs_set_view_prior(view, depth, w, h, stride) installs it: the same candidates
 *     and seeds, the same block in b200mvs_memory.fixed and resident.  It replaces any earlier prior of the view, with its
 *     dz and ids.  A later b200mvs_set_features does not refit.
 *   - fit_out (may be NULL) receives the fit.  A failed fit gives B200MVS_ERR_INVALID_ARG with a message that names the
 *     function and the reason; fit_out then holds n_obs, its other fields are 0, and the view's previous prior stays.
 *   - The observations, the fit and the apply run on the context's stream; their scratch (28 B per feature of the view,
 *     its position and its observation, and a 64 B fit record) comes from the budget and is freed before the call returns.  A prior block or
 *     scratch that does not fit gives B200MVS_ERR_NO_MEMORY and leaves the previous prior in place.
 *   - B200MVS_ERR_INVALID_ARG, naming the function and the field, before anything is copied: the checks of
 *     b200mvs_set_view_prior, a NULL values, a kind outside 0..2, a view without a camera, a context without features,
 *     and a planning context. */
int b200mvs_set_view_prior_relative(b200mvs_ctx* ctx, int view_id, const float* values, int w, int h, int stride,
                                    int kind, b200mvs_prior_fit* fit_out);
/* The same from DEVICE memory on the context's device: row y of the w x h floats starts at values_dev + y * row_pitch
 * bytes.  It gives exactly what b200mvs_set_view_prior_relative gives for the same values: the same fit and the same
 * prior, which the apply writes straight into the view's block.  The work runs after an event recorded on cuda_stream
 * (NULL = the legacy default stream), and the call returns when the prior is installed.  Its checks, plus row_pitch < 4 w
 * or not a multiple of 4, and a values_dev in host memory, on another device or not 4-byte aligned. */
int b200mvs_set_view_prior_relative_device(b200mvs_ctx* ctx, int view_id, const float* values_dev, int w, int h,
                                           int64_t row_pitch, int stride, int kind, void* cuda_stream,
                                           b200mvs_prior_fit* fit_out);
/* mve::Bundle::Features (bundle.h:51-60) as position + CSR list of referencing view ids. */
int b200mvs_set_features(b200mvs_ctx* ctx, int n_features, const float* pos,
                         const int32_t* ref_offsets, const int32_t* ref_view_ids);

/* ---- inspection (parity of the pyramid, image_tools.h:617-694) ---- */
int b200mvs_num_levels(b200mvs_ctx* ctx, int view_id);
/* With an image source installed, an evicted view is fetched again (its pyramid is rebuilt bit for bit). */
int b200mvs_get_level(b200mvs_ctx* ctx, int view_id, int level, int* w, int* h, uint8_t* rgb_host_or_null);
/* The same into DEVICE memory: rgb_dev_or_null receives the h x w x 3 bytes b200mvs_get_level writes (NULL: sizes only).  The
 * buffer is checked as b200mvs_reconstruct_device checks its maps (any alignment) and the stream rule is the same. */
int b200mvs_get_level_device(b200mvs_ctx* ctx, int view_id, int level, int* w, int* h, uint8_t* rgb_dev_or_null,
                             void* cuda_stream);

/* ---- DMRecon::analyzeFeatures + globalViewSelection (dmrecon.cc:179-241, global_view_selection.cc) ---- */
/* Returns the number of selected views (ids ascending in ids_out) or a negative error. */
int b200mvs_global_view_selection(b200mvs_ctx* ctx, const b200mvs_settings* s, int ref_view,
                                  int32_t* ids_out, int cap);

/* Engine knob (no reference counterpart): which of the two device implementations of PatchOptimization runs.
 * mode (b200mvs_optimize_patches): 0 = by batch size, 1 = one warp per patch (low latency), 2 = one thread per patch
 * (throughput).  thread_min (b200mvs_reconstruct): in a frontier round, a VIEW with at least this many patches runs them one
 * thread per patch, a view with fewer one warp per patch (the rule looks at the view alone, so a view's maps do not depend on
 * which other views share the batch); -1 = built-in default, 0 = always, a huge value = never.  Both implementations are
 * checked against the oracle. */
int b200mvs_set_patch_mode(b200mvs_ctx* ctx, int mode, int64_t thread_min);

/* Engine knob (no reference counterpart): the initial frontier capacity of a b200mvs_reconstruct launch,
 * max(ceil(entries_per_px x reference pixels), seeds, min_entries) entries of 169 device bytes each (default 2.0, 65536).
 * A smaller capacity shrinks b200mvs_working_set, so
 * b200mvs_plan_batches fits more views per launch; when a frontier round may not fit, the kernel stops before the round's
 * pushes, the library grows the frontier arrays to max(2 x capacity, what the round may need) entries (fewer when the budget
 * allows fewer, never fewer than needed) and resumes the launch where it stopped.  Maps and counters do not depend on the
 * capacity (n_patch_launches, n_kernel_launches and the times count the resumed launches too).  When the budget cannot hold
 * what the round needs, the call fails with B200MVS_ERR_OVERFLOW and a message naming both entry counts; the context stays
 * usable.  entries_per_px in [0, 64]; min_entries at most 2^40 and not 0 together with entries_per_px = 0; else
 * B200MVS_ERR_INVALID_ARG.  Works in a planning context. */
int b200mvs_set_frontier_capacity(b200mvs_ctx* ctx, double entries_per_px, uint64_t min_entries);
/* The frontier of the last b200mvs_reconstruct: initial and final capacity in entries (the largest over its launch groups)
 * and the number of resumes (summed over its groups).  Any pointer may be NULL. */
int b200mvs_frontier_info(b200mvs_ctx* ctx, uint64_t* initial_entries, uint64_t* final_entries, uint64_t* n_resumes);

/* Prepares, on host threads, what DMRecon::start computes before its queue runs - analyzeFeatures, globalViewSelection and
 * the seed list of processFeatures (dmrecon.cc:179-292) - for the given reference views, so that a LATER
 * b200mvs_reconstruct of these views (same settings) starts its kernel at once.  May be called from another thread WHILE a
 * b200mvs_reconstruct of a previous batch is running (the reference overlaps them the same way: its OpenMP threads are in
 * different stages of different views, apps/dmrecon/dmrecon.cc:285); cameras and features must not change meanwhile
 * (re-uploading the image of a view with an UNCHANGED camera is allowed).  b200mvs_global_view_selection of a planned view
 * returns the plan's selection; b200mvs_reconstruct uses a plan once and drops it; changing a camera or the features drops
 * all plans.  Host threads: up to hardware_concurrency(), or the value of the environment variable B200MVS_HOST_THREADS
 * (several processes sharing one box, one per GPU).  Settings and views are checked as b200mvs_reconstruct checks them,
 * with the same codes and messages. */
int b200mvs_plan_views(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* ref_views);

/* How the last b200mvs_reconstruct, b200mvs_reconstruct_device or b200mvs_pset_add_reconstruction planned its views
 * (analyzeFeatures, globalViewSelection and the seed list).  A view with a plan from b200mvs_plan_views uses it; the others
 * are planned on the device, one CTA per view and one launch per chunk of views that fits the budget, with selections and
 * seeds equal to the host planner's.  A view is planned on host threads instead when its planning workspace does not fit
 * the budget on its own, or when min_parallax is above about 41 degrees (the device's table of parallax factors would
 * exceed 2^22 entries).  The planning allocations go through the budget and are freed before the first launch group, so
 * they never add to b200mvs_memory.fixed. */
typedef struct b200mvs_plan_info {
    uint64_t n_prepared;     /* views taken from b200mvs_plan_views plans */
    uint64_t n_device;       /* views planned on the device               */
    uint64_t n_host;         /* views planned on host threads             */
    double   ms_plan;        /* wall time of the call's planning phase    */
    double   ms_device;      /* CUDA-event time of the planning kernels   */
    uint64_t peak_bytes;     /* largest planning allocation               */
} b200mvs_plan_info;
/* The b200mvs_plan_info of the last reconstruction (all zero before the first one).  The struct and the function cannot share
 * one name in C, so the query is named like b200mvs_memory_stats. */
int b200mvs_plan_stats(b200mvs_ctx* ctx, b200mvs_plan_info* out);

/* ---- batch of independent PatchOptimization runs: ctor + doAutoOptimization + computeConfidence
 *      (patch_optimization.cc:21-242); the patch-level parity entry ---- */
int b200mvs_optimize_patches(b200mvs_ctx* ctx, const b200mvs_settings* s, int ref_view,
                             const int32_t* global_ids, int n_global,
                             const b200mvs_patch_in* in, int n, b200mvs_patch_out* out,
                             b200mvs_stats* stats_or_null);

/* ---- DMRecon::start (dmrecon.cc:90-172) for a batch of reference views ----
 * Runs analyzeFeatures, globalViewSelection, processFeatures and processQueue for every view in
 * ref_views; all of them advance together, one frontier round per kernel sequence.  Views without a b200mvs_plan_views
 * plan are planned on the device before the first group (b200mvs_plan_info).
 * maps: array of n_refs entries, or NULL to leave the results on the device (HBM-resident timing);
 * progress: array of n_refs entries or NULL; stats: one aggregate or NULL.
 * A view whose global view selection is empty makes the call fail with B200MVS_ERR_GLOBAL_VS
 * (failed_view_or_null receives its id).
 * The batch is split into groups that fit the device budget (b200mvs_plan_batches with available = budget - fixed bytes;
 * without an image source there is no budget and the batch is one group); each group evicts the pyramids it does not need
 * (least recently used first), fetches the images it lacks through the source and runs its own frontier launch.  A view's
 * maps do not depend on which views share its launch, so they are bit-identical to one launch of the whole batch.
 * Without a source, a needed image that is not loaded fails the call before anything runs.  Across groups `stats` sums
 * counts and times, takes the maximum of n_entries_peak and counts one patch launch per group; a view cancelled before
 * its group starts never runs; B200MVS_ERR_CANCELLED is returned only when every view was cancelled; maps == NULL with
 * more than one group fails with B200MVS_ERR_INVALID_ARG (the results of a group do not stay on the device); a view that
 * does not fit on its own fails the call with B200MVS_ERR_NO_MEMORY (failed_view_or_null receives its id).  At most 4000
 * views per group (per call without a source). */
int b200mvs_reconstruct(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* ref_views,
                        b200mvs_maps* maps, b200mvs_progress* progress, b200mvs_stats* stats,
                        int32_t* failed_view_or_null);

/* b200mvs_reconstruct with the maps written into DEVICE memory: every non-NULL pointer of maps_dev[j] is device (or managed)
 * memory on the context's device, in the layouts of b200mvs_maps; depth is required, the others may be NULL; width/height
 * are written into the host structs.  Settings and view checks, codes and messages, progress, cancellation (a cancelled
 * view's buffers are left untouched), stats, groups, planning on the device (b200mvs_plan_info), the image source and the
 * budget are b200mvs_reconstruct's, and each
 * group's maps are written right after its launch.
 *   - Before anything runs, each buffer is checked with cudaPointerGetAttributes: host memory (pinned or pageable), memory
 *     of another device, a pointer that is not 4-byte aligned and a NULL depth give B200MVS_ERR_INVALID_ARG with a message
 *     naming the view and the field.  A NULL context, settings or maps_dev is B200MVS_ERR_INVALID_ARG; a planning context
 *     B200MVS_ERR_CUDA.
 *   - Streams: the library's work waits for an event recorded on cuda_stream (a cudaStream_t; NULL = the legacy default
 *     stream) at entry, so the caller may produce or reuse the buffers on its stream just before the call.  The call
 *     returns when the writes are complete.
 *   - The buffers are the caller's memory: they are not counted in the context's budget. */
int b200mvs_reconstruct_device(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* ref_views,
                               b200mvs_maps* maps_dev, void* cuda_stream, b200mvs_progress* progress, b200mvs_stats* stats,
                               int32_t* failed_view_or_null);

/* ---- per-entry pyramid levels: views of different sizes (apps/dmrecon --max-pixels, dmrecon.cc:89-111,299-302) or one
 *      view at several levels (scene2pset -F2, -F3) in one call ----
 * The *_levels forms of b200mvs_reconstruct, b200mvs_reconstruct_device, b200mvs_pset_add_reconstruction,
 * b200mvs_working_set and b200mvs_plan_batches take levels[j] (n_refs entries) next to ref_views[j]:
 *   - Levels.  Entry j reconstructs ref_views[j] at pyramid level levels[j]; s->scale is not read.  Every other rule is
 *     that of the call without levels: settings checks, codes and messages, progress and cancellation per entry, stats
 *     summed over entries, groups, the budget, the image source, the sink and the stream rule.  A call with every
 *     levels[j] == s->scale is the call without levels.
 *   - Maps.  An entry's maps (depth, conf, dz, normal, view_ids) are bit for bit those of a single-level call of that view
 *     at that level, whatever the other entries and levels of the call; b200mvs_maps.width/height are those of the
 *     entry's level.  Masks are per view and resampled to each entry's map size by the rule of b200mvs_set_view_mask.
 *   - Checks.  levels == NULL, a level < 0 or past the view's pyramid ("Invalid scale factor", failed_view_or_null
 *     receives the view) give B200MVS_ERR_INVALID_ARG; the 65535-pixels-per-side limit applies to each entry's level.
 *   - Repeated views.  A view may appear at several levels, but a (view, level) pair only once: a repeat gives
 *     B200MVS_ERR_INVALID_ARG with a message naming the view and the level before anything runs.  All entries of a view
 *     share its one pyramid: it is counted once in the working set, pinned once per group and fetched once when its
 *     group needs it.
 *   - Plans.  Prepared plans (b200mvs_plan_views) stay stored one per view with their settings; an entry uses one when
 *     the plan's settings equal s with scale = levels[j], and the other entries are planned in the call, once per
 *     distinct level with that level's calibration, so selections and seeds are those of a single-level call.
 *     b200mvs_plan_info counts entries.
 *   - Groups.  Working set and groups work per entry, at the entry's pixel and seed counts; the 4000-views-per-group
 *     limit counts entries. */
int b200mvs_reconstruct_levels(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* ref_views,
                               const int32_t* levels, b200mvs_maps* maps, b200mvs_progress* progress, b200mvs_stats* stats,
                               int32_t* failed_view_or_null);
int b200mvs_reconstruct_levels_device(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* ref_views,
                                      const int32_t* levels, b200mvs_maps* maps_dev, void* cuda_stream,
                                      b200mvs_progress* progress, b200mvs_stats* stats, int32_t* failed_view_or_null);

/* ---- device memory budget: images loaded on demand (ImagePyramidCache::cleanup, image_pyramid.cc:134-155) ----
 * Without a source (the default) the context has no budget: no pyramid is evicted, so every one stays resident until the
 * context is destroyed, and b200mvs_reconstruct runs a batch of up to 4000 views in one launch. */
typedef struct b200mvs_image {
    const uint8_t* rgb;           /* HOST pointer, h x w x channels, row-major; valid until the release callback */
    int32_t w, h, channels;       /* must equal the size registered for the view; channels 1..4                  */
} b200mvs_image;
/* Returns 0 and fills *out with the `undistorted` image of view_id, or non-zero when it cannot be loaded. */
typedef int  (*b200mvs_fetch_fn)(void* user, int32_t view_id, b200mvs_image* out);
/* Called once per successful fetch, after the image was copied; the pointer may be freed. */
typedef void (*b200mvs_release_fn)(void* user, int32_t view_id);
/* Installs (fetch != NULL) or removes (fetch == NULL) the image source of the context and sets its device budget.
 * budget_bytes = 0: 90 % of the free bytes cudaMemGetInfo reports at this call.  The budget bounds every device allocation
 * of the context (accounted in requested bytes); installing it evicts pyramids and drops idle workspace until the resident
 * bytes fit.  With a source, a view whose pyramid is needed and not resident (b200mvs_reconstruct, b200mvs_get_level,
 * b200mvs_optimize_patches) is fetched and uploaded, and pyramids - also those the caller uploaded - may be evicted.
 * The callbacks run on the calling thread WITH THE CONTEXT LOCK HELD: they must not call into this context. */
int b200mvs_set_image_source(b200mvs_ctx* ctx, b200mvs_fetch_fn fetch, b200mvs_release_fn release, void* user,
                             uint64_t budget_bytes);

/* An image source whose images are in DEVICE memory, e.g. decoded on the GPU or held as CUDA tensors.  Texel (x, y),
 * channel c lies at data + y * row_pitch + x * channels + c when plane_pitch == 0 (interleaved, HWC) and at
 * data + c * plane_pitch + y * row_pitch + x when plane_pitch > 0 (planar, CHW). */
typedef struct b200mvs_device_image {
    const uint8_t* data;          /* DEVICE pointer on the context's device; valid until the release callback             */
    int32_t w, h, channels;       /* must equal the registered size; channels 1..4 (grey expanded, alpha dropped)        */
    int64_t row_pitch;            /* bytes between rows; >= w * channels interleaved, >= w planar                        */
    int64_t plane_pitch;          /* 0 = interleaved (HWC); else planar (CHW): bytes between channel planes, >= h * row_pitch */
    void*   cuda_stream;          /* cudaStream_t the image was produced on (NULL = the legacy default stream)             */
} b200mvs_device_image;
/* Returns 0 and fills *out with the `undistorted` image of view_id (or the distorted photo, b200mvs_set_view_distortion),
 * non-zero when it cannot be loaded. */
typedef int (*b200mvs_device_fetch_fn)(void* user, int32_t view_id, b200mvs_device_image* out);
/* Installs (fetch != NULL) or removes (fetch == NULL) a device image source.  A context has one source: installing either
 * kind replaces the other, and removing either removes it.
 *   - As b200mvs_set_image_source: the budget and budget_bytes = 0, which calls fetch and when, LRU eviction, the groups
 *     of b200mvs_reconstruct, the context lock held during the callbacks, and the failure messages and failed_view of a
 *     fetch that fails.
 *   - Accounting: b200mvs_memory is kept as for a host source, so both plan the same groups, evict the same pyramids and
 *     report the same numbers over the same scene.  The pyramid is built straight from the caller's memory, with no
 *     staging copy; the budget is still charged the two staging buffers a host source would allocate (fixed keeps their
 *     bound).  n_loads counts the device fetches and bytes_loaded their w * h * channels.  The caller's image memory is
 *     not in the budget.
 *   - Ordering: when fetch returns, the library records an event on cuda_stream and its kernels wait for it before they
 *     read the image, so fetch may enqueue the decode and return without synchronising.
 *   - Release: release (may be NULL) is called once per successful fetch, after every kernel that reads the image has
 *     completed and before the call that fetched it returns.  The library waits for those kernels once per batch of
 *     loads (one b200mvs_reconstruct group, one b200mvs_get_level, ...), never with cudaDeviceSynchronize.
 *   - Before anything reads the image, the descriptor is checked: data must be device (or managed) memory on the
 *     context's device (cudaPointerGetAttributes, as for the maps of b200mvs_reconstruct_device: host memory, pinned or
 *     pageable, and memory of another device are rejected), w and h the registered size, channels 1..4, row_pitch and
 *     plane_pitch non-negative and within the bounds above (a plane_pitch below h * row_pitch would overlap the rows of
 *     a plane).  A failed check gives B200MVS_ERR_INVALID_ARG with a message naming the view (failed_view as for a
 *     failed fetch); release is still called, nothing is launched, and the context stays usable.  The caller keeps the
 *     whole extent of the image within one allocation. */
int b200mvs_set_image_source_device(b200mvs_ctx* ctx, b200mvs_device_fetch_fn fetch, b200mvs_release_fn release, void* user,
                                    uint64_t budget_bytes);

typedef struct b200mvs_memory {
    uint64_t budget;              /* 0 = no source installed (no limit)                                           */
    uint64_t fixed;               /* bytes that do not depend on the batch: view table, sRGB table, settings and frontier
                                     control block, two upload staging buffers of the largest registered image (bound),
                                     device masks and priors                                                          */
    uint64_t resident;            /* device bytes the context holds now                                          */
    uint64_t peak;                /* maximum of `resident` since creation or since the source was installed        */
    uint64_t n_loads;             /* images fetched through the source                                           */
    uint64_t bytes_loaded;        /* host bytes of those images                                                  */
    uint64_t n_evictions;         /* pyramids evicted                                                            */
    uint64_t n_groups;            /* launches (sub-batches) of the last b200mvs_reconstruct                       */
} b200mvs_memory;
int b200mvs_memory_stats(b200mvs_ctx* ctx, b200mvs_memory* out);

/* Device bytes one b200mvs_reconstruct launch of these reference views needs beyond the fixed bytes: the pyramids of the
 * views and their global selections (every level, 20 bytes per texel at a row pitch of 4 texels), the maps (40 bytes per
 * pixel of level `scale`, + 2 KiB), the frontier arrays (169 bytes per entry, the initial capacity of
 * b200mvs_set_frontier_capacity: max(ceil(2 x pixels), seeds, 65536) entries by default), the tile arrays (12 bytes per
 * 16x16 tile) and the per-view arrays.  b200mvs_reconstruct reserves exactly these sizes before its first launch.  Works
 * in a planning context (cameras and features suffice); prepared plans are read, not consumed. */
int b200mvs_working_set(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* ref_views, uint64_t* bytes);

/* Splits the reference views into groups whose working sets fit `available` bytes; group_of_ref[j] receives the group of
 * ref_views[j]; returns the number of groups.  Deterministic: a group opens with the first unassigned view in the given
 * order, then repeatedly takes the unassigned view that fits and adds the fewest new pyramid bytes (ties: lowest index),
 * until none fits (or the group has 4000 views).  B200MVS_ERR_NO_MEMORY when a view does not fit on its own
 * (failed_view_or_null receives its id). */
int b200mvs_plan_batches(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* ref_views,
                         uint64_t available, int32_t* group_of_ref, int32_t* failed_view_or_null);
/* The two above with one pyramid level per entry (see b200mvs_reconstruct_levels): the maps, tiles and seeds of entry j
 * are those of ref_views[j] at levels[j], and each view's pyramid is counted once however many entries it has.  With every
 * levels[j] == s->scale they return what b200mvs_working_set and b200mvs_plan_batches return. */
int b200mvs_working_set_levels(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* ref_views,
                               const int32_t* levels, uint64_t* bytes);
int b200mvs_plan_batches_levels(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* ref_views,
                                const int32_t* levels, uint64_t available, int32_t* group_of_ref, int32_t* failed_view_or_null);

/* ---- consumers of the depth maps, on the device (SURVEY.md 8f rank 2 and 3).  Stateless: host buffers in, host buffers
 *      out (the *_device forms: device buffers in and out), `device` = CUDA device ordinal.  Errors: negative code, message
 *      from b200mvs_last_error(). ---- */
const char* b200mvs_depthmap_last_error(void);   /* the same message as b200mvs_last_error */
/* mve::image::depthmap_confidence_clean (libs/mve/depthmap.cc:118-131): depth = 0 where conf <= 0, in place. */
int b200mvs_depthmap_confidence_clean(int device, float* depth, const float* conf, int w, int h);
/* mve::image::depthmap_cleanup (depthmap.cc:25-113): 4-connected islands of depth != 0 smaller than thres pixels are erased. */
int b200mvs_depthmap_cleanup(int device, const float* depth, int w, int h, int64_t thres, float* out);
/* The two filters above on n_maps maps of their own sizes (widths[j] x heights[j]) in DEVICE memory on `device`, for GPU
 * callers that hold the maps of b200mvs_reconstruct_device:
 *   - Results: every output map is byte for byte what the host entry point gives for the same map (and threshold),
 *     NaN, +-inf and -0.0 depths and confidences included; a negative threshold is converted to size_t as the reference
 *     does, which erases every island.
 *   - Checks, all before anything is launched or written; a failure is B200MVS_ERR_INVALID_ARG with a message naming the
 *     function, the map index and the field: n_maps < 0; a NULL array, or a NULL map, when n_maps > 0; a width or height
 *     < 1; a map of more than 0xFFFFFFF0 pixels (the host entry point's limit); a buffer that is host memory (pageable or
 *     pinned), memory of another device or not 4-byte aligned (cudaPointerGetAttributes, as b200mvs_reconstruct_device
 *     checks its maps); a written range (depth_dev of confidence_clean, out_dev of cleanup) that overlaps any other range
 *     of the call, except out_dev[j] == depth_dev[j].  n_maps == 0 returns 0 and touches nothing.
 *   - Streams: the work runs on cuda_stream (a cudaStream_t; NULL = the legacy default stream) after what is already
 *     there, and the call returns when the maps are written.
 *   - Memory: the maps are read and written in place in the caller's buffers, with no staging copy.  cleanup takes its
 *     maps in order in chunks, each the longest run of consecutive maps of at most 2^28 pixels in all (a larger map is a
 *     chunk of its own), and allocates once per call a union-find workspace of 8 B per pixel of the largest chunk; both
 *     also hold a table of 56 B per map and 4 B per 256 pixels of a map.  Everything is freed before the call returns. */
/* depthmap_confidence_clean on each map: depth_dev[j] = 0 where conf_dev[j] <= 0, in place. */
int b200mvs_depthmap_confidence_clean_device(int device, int n_maps, float* const* depth_dev, const float* const* conf_dev,
                                             const int32_t* widths, const int32_t* heights, void* cuda_stream);
/* depthmap_cleanup on each map: out_dev[j] = depth_dev[j] with the 4-connected islands of depth != 0 smaller than thres[j]
 * pixels erased.  out_dev[j] == depth_dev[j] cleans in place. */
int b200mvs_depthmap_cleanup_device(int device, int n_maps, const float* const* depth_dev, const int32_t* widths,
                                    const int32_t* heights, const int64_t* thres, float* const* out_dev, void* cuda_stream);
/* mve::geom::depthmap_triangulate (depthmap.cc:196-375, the per-view work of apps/scene2pset/scene2pset.cc:264-328):
 * vertex ids per pixel (0xFFFFFFFF = none), vertices (pixel_3dpos; transformed by the 4x4 row-major cam_to_world when given,
 * like mesh_transform), vertex colours (r, g, b, 1 as floats; NULL colour image = none) and faces, all in the reference's
 * order.  Outputs may be NULL except the counts; capacities in vertices / faces (w*h and 2*(w-1)*(h-1) always suffice). */
int b200mvs_depthmap_triangulate(int device, const float* depth, int w, int h, const float invproj[9], float dd_factor,
                                 const float* cam_to_world_or_null, const uint8_t* color_or_null, int color_channels,
                                 uint32_t* vertex_ids, float* vertices, float* colors, uint32_t* faces,
                                 uint64_t cap_vertices, uint64_t cap_faces, uint64_t* n_vertices, uint64_t* n_faces,
                                 double* device_ms_or_null);

/* The per-view work of apps/scene2pset (scene2pset.cc:264-358) in one call: depthmap_triangulate as above plus, per vertex,
 * the angle-weighted normals of TriangleMesh::recalc_normals (mesh.cc:45-151; normals NULL = skip), the boundary confidences
 * of depthmap_mesh_confidences(mesh, conf_iterations) (depthmap.cc:497-548; the app uses 4; confidences NULL or 0 = skip; any
 * conf_iterations >= 0 is exact, and the ring launches stop once a ring reaches no new vertex) and
 * the scale values (mean distance to the adjacent vertices of MeshInfo times scale_factor, scene2pset.cc:347-357; NULL = skip). */
int b200mvs_depthmap_pointset(int device, const float* depth, int w, int h, const float invproj[9], float dd_factor,
                              const float* cam_to_world_or_null, const uint8_t* color_or_null, int color_channels,
                              uint32_t* vertex_ids, float* vertices, float* colors, uint32_t* faces,
                              float* normals, float* confidences, int conf_iterations, float* scales, float scale_factor,
                              uint64_t cap_vertices, uint64_t cap_faces, uint64_t* n_vertices, uint64_t* n_faces,
                              double* device_ms_or_null);

/* b200mvs_depthmap_pointset (and with the attribute outputs NULL, b200mvs_depthmap_triangulate) on n_maps maps of their
 * own sizes in DEVICE memory on `device`, for GPU callers that hold the maps and level images of
 * b200mvs_reconstruct_device.  One b200mvs_dm_mesh per map: its inputs, its outputs and, on return, its counts.
 *   - Results: each map's outputs are byte for byte what b200mvs_depthmap_pointset gives for that map alone with the same
 *     invproj, cam_to_world, colour image, dd_factor, conf_iterations and scale_factor: vertex ids (0xFFFFFFFF = none),
 *     vertex and face order, and every float, NaN, +-inf and -0.0 depths included.  Vertex ids and face indices start at
 *     0 in every map.  colors are written only with a colour image, confidences only when conf_iterations > 0.
 *   - Counting: a map whose outputs are all NULL is only counted: n_vertices and n_faces are written and its capacities
 *     are not checked, so that two calls give exactly sized buffers.  Otherwise a map whose counts exceed cap_vertices or
 *     cap_faces fails the call with B200MVS_ERR_OVERFLOW and a message naming the first such map; every map's counts are
 *     still written and no output buffer of any map is.
 *   - Checks, all before anything is launched or written; a failure is B200MVS_ERR_INVALID_ARG with a message naming the
 *     function, the map index and the field: n_maps < 0; maps NULL when n_maps > 0; conf_iterations < 0 (the reference's
 *     "Invalid amount of iterations"); a NULL depth_dev; a width or height < 2 or more than 2^31 - 2 pixels (a map's
 *     scan holds up to two faces per pixel in 32 bits); color_channels outside 1..4 with a colour image; an output
 *     whose byte range (capacity x element size, vertex_ids width x height x 4) wraps the address space; a buffer that is host memory, memory of another device, or an output
 *     or depth_dev not 4-byte aligned; a written range that overlaps any other written or read range of the call
 *     (depth_dev and color_dev are read).  n_maps == 0 returns 0 and touches nothing.
 *   - Streams: the work runs on cuda_stream (a cudaStream_t; NULL = the legacy default stream) after what is already
 *     there, and the call returns when every output is written.  The counts are read back once, with one synchronisation;
 *     with confidences, one more every 16 rings of a chunk whose border rings have not yet stopped.
 *   - Memory: the maps go in order in chunks, each the longest run of consecutive maps of at most 2^28 pixels in all (a
 *     larger map is a chunk of its own).  The workspace is allocated once per call and sized to the largest chunk: 17 B
 *     per pixel, plus 4 B when a map with outputs has no vertex_ids, 12 B when one has no vertices (the vertices are
 *     computed for every map with outputs) and 8 B when confidences are computed, plus the scan's temporary storage;
 *     and a table of 224 B per map and 4 B per 256 pixels of a map.  Everything is freed before the call returns. */
typedef struct b200mvs_dm_mesh {
    /* input, read in place */
    const float* depth_dev;           /* width x height floats on `device` */
    int32_t width, height;            /* >= 2 each, width * height <= 2^31 - 2 */
    float invproj[9];                 /* as b200mvs_depthmap_pointset */
    const float* cam_to_world;        /* HOST, 16 floats row-major, or NULL */
    const uint8_t* color_dev;         /* packed height x width x color_channels bytes on `device`, any alignment, or NULL */
    int32_t color_channels;           /* 1..4 when color_dev != NULL */
    /* outputs on `device`, NULL = not wanted */
    uint32_t* vertex_ids;             /* width * height */
    float* vertices;                  /* 3 floats per vertex */
    float* colors;                    /* 4 floats per vertex */
    uint32_t* faces;                  /* 3 per face */
    float* normals;                   /* 3 floats per vertex */
    float* confidences;               /* 1 float per vertex */
    float* scales;                    /* 1 float per vertex */
    uint64_t cap_vertices, cap_faces;
    /* results */
    uint64_t n_vertices, n_faces;
} b200mvs_dm_mesh;
int b200mvs_depthmap_pointset_device(int device, int n_maps, b200mvs_dm_mesh* maps, float dd_factor, int conf_iterations,
                                     float scale_factor, void* cuda_stream);

/* ---- the whole-scene point set of apps/scene2pset (scene2pset.cc:247-464) on the device ---- */
/*

 * A handle collects the point sets of many views: b200mvs_pset_add_view runs the per-view work of
 * b200mvs_depthmap_pointset on one depth map, then the scene-level filters (fill fraction, bounding box, confidence-scaled
 * normals, vertex -> pixel map), and appends the surviving points to a point set kept in HOST memory, in the order the
 * views are added.  b200mvs_pset_clip_masks deletes the points that any silhouette mask marks as background.  The device
 * memory of a handle made by b200mvs_pset_create does not grow with the number of views or points: one view's workspace
 * (kept at the largest view added so far), plus the masks and one chunk of points during clipping.  A handle made by
 * b200mvs_pset_create_on_device keeps its point set in DEVICE memory instead (below).  Errors: negative code,
 * b200mvs_last_error(). */
typedef struct b200mvs_pset b200mvs_pset;
typedef struct b200mvs_pset_options {
    int32_t with_normals;         /* -n: angle-weighted vertex normals                                              */
    int32_t with_conf;            /* -c: boundary confidences with conf_iterations >= 1 rings (scene2pset uses 4)    */
    int32_t with_scale;           /* -s: scale values (mean distance to the adjacent vertices times scale_factor)     */
    int32_t poisson_normals;      /* -p: normal *= confidence; needs with_normals and with_conf                     */
    int32_t correspondence;       /* -C: keep each vertex' pixel; not with use_aabb, and no mask clipping afterwards */
    int32_t use_aabb;             /* -b: keep a point when aabb_min <= p <= aabb_max on every axis (both faces kept) */
    float   aabb_min[3], aabb_max[3];
    float   min_valid_fraction;   /* -f: > 0 skips views whose fill fraction (in the reference's float sums) is lower */
    float   scale_factor;         /* -S, 2.5                                                                        */
    float   dd_factor;            /* mve::geom::DD_FACTOR_DEFAULT = 5                                                */
    int32_t conf_iterations;      /* 4                                                                              */
} b200mvs_pset_options;
/* The fields of mve::CameraInfo a view contributes (libs/mve/camera.h), as b200mvs_set_view_camera takes them. */
typedef struct b200mvs_pset_camera {
    float flen, paspect, ppoint[2], rot[9], trans[3];
} b200mvs_pset_camera;
typedef struct b200mvs_pset_view {
    int32_t  added;               /* 0: skipped by min_valid_fraction                                                */
    float    fraction;            /* the fill fraction as the reference computes it (only when min_valid_fraction > 0) */
    uint64_t n_points;            /* points this view appended (after the bounding box)                              */
    uint64_t first_index;         /* index of its first point in the point set                                       */
} b200mvs_pset_view;
typedef struct b200mvs_pset_info {
    uint64_t n_points;            /* points in the set                                                              */
    uint64_t n_colors;            /* colours in the set: less than n_points when a view had no colour image          */
    uint64_t n_views;             /* views added (not skipped)                                                      */
    uint64_t device_bytes;        /* device bytes the handle holds now (a device-resident set's arrays included)     */
    uint64_t peak_device_bytes;   /* maximum of device_bytes since creation                                         */
    double   ms_pointset;         /* device time of the per-view kernels (triangulation, normals, confidences, scales) */
    double   ms_filter;           /* device time of fill count, bounding box, compaction, normal scaling, pixel map  */
    double   ms_mask;             /* device time of mask clipping: with the transfers of the chunks on a host-resident
                                     set; clip, scan and compaction in place (no transfers) on a device-resident one */
} b200mvs_pset_info;
/* Correspondence metadata of one added view (scene2pset.cc:50-56). */
typedef struct b200mvs_pset_corr_view {
    uint32_t view_id, width, height;
    uint64_t first_index;
} b200mvs_pset_corr_view;

int b200mvs_pset_create(int device, const b200mvs_pset_options* options, b200mvs_pset** out);
/* A handle whose point set is kept in DEVICE memory on `device`; options are checked as b200mvs_pset_create checks them
 * (the same codes and messages, naming this function).  Every b200mvs_pset_* entry point takes it with the same meaning
 * and gives the same arrays, records and counts as for a b200mvs_pset_create handle fed the same inputs:
 *   - views append their points with device-to-device copies; b200mvs_pset_add_reconstruction stages each view on the
 *     device and commits them in ref_views order when the whole call succeeds (on an error, or every view cancelled,
 *     the set is unchanged; its capacity may have grown);
 *   - b200mvs_pset_clip_masks clips and compacts the set in place (the masks are uploaded once);
 *   - b200mvs_pset_read / _read_correspondence copy the set to the host; b200mvs_pset_read_device copies it to device
 *     buffers without a host copy.
 * The set is the caller's memory, like the buffers of b200mvs_reconstruct_device: its arrays grow by doubling through
 * cudaMalloc, are never taken from a context's budget (b200mvs_memory is the same for either kind of handle), and are
 * counted in the handle's device_bytes and peak_device_bytes. */
int b200mvs_pset_create_on_device(int device, const b200mvs_pset_options* options, b200mvs_pset** out);
void b200mvs_pset_destroy(b200mvs_pset* ps);
/* One view (scene2pset.cc:284-399): depth map w x h, colour image of the same size with 1-4 channels or NULL, camera.
 * The view's calibration for the map's size and its camera-to-world matrix are formed as CameraInfo forms them. */
int b200mvs_pset_add_view(b200mvs_pset* ps, int view_id, const float* depth, int w, int h, const uint8_t* color_or_null,
                          int color_channels, const b200mvs_pset_camera* cam, b200mvs_pset_view* out_or_null);
/* The same with the depth map and the colour image in DEVICE memory on the handle's device, checked as
 * b200mvs_reconstruct_device checks its maps (the colour image at any alignment); the work waits for an event recorded on
 * cuda_stream (NULL = the legacy default stream) at entry, and the call returns when it is done. */
int b200mvs_pset_add_view_device(b200mvs_pset* ps, int view_id, const float* depth_dev, int w, int h,
                                 const uint8_t* color_dev_or_null, int color_channels, const b200mvs_pset_camera* cam,
                                 void* cuda_stream, b200mvs_pset_view* out_or_null);
/* Silhouette masks (scene2pset.cc:407-464): n_masks one-channel masks of their own sizes with their cameras.  A point is
 * deleted when, for any mask, it projects inside the mask (0 <= x < w, 0 <= y < h) onto a 0 byte; a projection that is
 * NaN counts as outside.  The result does not depend on the order of the masks; num_filtered receives the number of
 * deleted points.  The per-point lists follow mve::TriangleMesh::delete_vertices: a list is filtered only when it has one
 * entry per point, so a colour list shorter than the point list (a view without a colour image) is left as it is.
 * Callable once per handle; no view can be added afterwards. */
int b200mvs_pset_clip_masks(b200mvs_pset* ps, int n_masks, const uint8_t* const* masks, const int32_t* widths,
                            const int32_t* heights, const b200mvs_pset_camera* cams, uint64_t* num_filtered);
/* The same with the masks in DEVICE memory on the handle's device, read in place: row y of mask m starts at
 * masks_dev[m] + y * row_pitches[m] (row_pitches[m] >= widths[m]).  The point set, num_filtered and the per-list rule are
 * b200mvs_pset_clip_masks' for the same mask bytes, on either kind of handle.  Its checks, plus row_pitches and the
 * device-buffer check of b200mvs_reconstruct_device at any alignment, all run before anything is launched, and a rejected
 * call changes nothing.  The work waits for an event recorded on cuda_stream (NULL = the legacy default stream) at entry,
 * and the call returns when the set is clipped; ms_mask adds the device time of the clip and the compaction.  No device
 * memory beyond the set remains after the call. */
int b200mvs_pset_clip_masks_device(b200mvs_pset* ps, int n_masks, const uint8_t* const* masks_dev, const int32_t* widths,
                                   const int32_t* heights, const int64_t* row_pitches, const b200mvs_pset_camera* cams,
                                   void* cuda_stream, uint64_t* num_filtered);
int b200mvs_pset_get_info(b200mvs_pset* ps, b200mvs_pset_info* out);
/* Copies the point set out; NULL skips an array.  vertices / normals 3 floats, colours 4 floats (n_colors of them),
 * values and confidences 1 float per point.  Normals, values and confidences exist when the options asked for them. */
int b200mvs_pset_read(b200mvs_pset* ps, float* vertices, float* normals, float* colors, float* values, float* confidences);
/* With options.correspondence: pixel (x, y) of every point, and one record per added view (n_views of them). */
int b200mvs_pset_read_correspondence(b200mvs_pset* ps, uint32_t* pixels_xy, b200mvs_pset_corr_view* views);
/* b200mvs_pset_read and the pixel map of b200mvs_pset_read_correspondence into DEVICE buffers on the handle's device, in
 * the same layouts; NULL skips an array, and pixels_xy must be NULL on a handle made without correspondence.  Works on
 * either kind of handle (a host-resident set is copied host to device).  Buffers are checked as b200mvs_reconstruct_device
 * checks its maps (host memory, another device or a pointer not 4-byte aligned: B200MVS_ERR_INVALID_ARG naming the
 * field) before anything is copied; the copies wait for an event recorded on cuda_stream (NULL = the legacy default
 * stream) at entry, and the call returns when they are done. */
int b200mvs_pset_read_device(b200mvs_pset* ps, float* vertices_dev, float* normals_dev, float* colors_dev, float* values_dev,
                             float* confidences_dev, uint32_t* pixels_xy_dev, void* cuda_stream);

/* ---- dmrecon straight into scene2pset: the point sets of a batch of reference views without their maps leaving the device ----
 * Bit-identical to b200mvs_reconstruct(ctx, s, n_refs, ref_views, maps, progress, stats, failed_view_or_null) followed, for
 * each j in ref_views order, by b200mvs_pset_add_view(ps, ref_views[j], depth_j, w, h, level_j, 3, &cam_j, &views_out[j]),
 * where level_j is b200mvs_get_level(ctx, ref_views[j], s->scale, ...) and cam_j the fields the view was registered with
 * (b200mvs_set_view_camera / b200mvs_upload_view): the same arrays from b200mvs_pset_read / _read_correspondence, the same
 * n_points, n_colors and n_views, the same per-view records (views_out_or_null: n_refs of them, views skipped by
 * min_valid_fraction and cancelled views included, both with added = 0).
 *   - Nothing but the surviving points leaves the device: each view's triangulation and filters run on its depth map where
 *     the reconstruction left it, with the colours read in place from its pyramid level `scale`.
 *   - Colours: at scale > 0 the level is what dmrecon saves as undist-L<s> (scene2pset -F<s>).  At scale 0 it is the
 *     `undistorted` image as uploaded, grey (1 or 2 channels) expanded to r = g = b and alpha dropped; for 1, 2, 3 and
 *     4 channels that is exactly what depthmap_triangulate makes of the `undistorted` image itself (depthmap.cc:349-364:
 *     channel 0 is grey below 3 channels, channels 1-2 are green and blue from 3 on, alpha is never read).
 *   - Points are appended in ref_views order, whatever groups the budget makes; nothing depends on group composition.
 *   - Memory: during the call the handle's per-view workspace lives on the context's device in the context's budget; every
 *     group is planned with the workspace of the batch's largest map kept free, so b200mvs_memory.peak stays within the
 *     budget, and a group's maps are consumed before the next group runs.  The workspace is freed when the call returns.
 *   - Argument checks, error codes, progress, cancellation, stats, groups, planning on the device (b200mvs_plan_info) and
 *     the image source are b200mvs_reconstruct's.
 *     A view cancelled on its own adds nothing (added = 0); every view cancelled gives B200MVS_ERR_CANCELLED.
 *   - On any error, and when every view was cancelled, the handle's point set, views and times are unchanged: the points are
 *     committed only when the whole call succeeds.
 *   - B200MVS_ERR_INVALID_ARG for a NULL context, a planning context, a NULL handle, a handle on another device than the
 *     context, and a handle whose masks have been applied (clip masks after this call).
 * Errors: b200mvs_last_error(). */
int b200mvs_pset_add_reconstruction(b200mvs_pset* ps, b200mvs_ctx* ctx, const b200mvs_settings* s,
                                    int n_refs, const int32_t* ref_views,
                                    b200mvs_progress* progress, b200mvs_stats* stats,
                                    int32_t* failed_view_or_null, b200mvs_pset_view* views_out_or_null);
/* The same with one pyramid level per entry (see b200mvs_reconstruct_levels): entry j appends what b200mvs_pset_add_view
 * appends for the depth map of ref_views[j] at levels[j], the view's level image levels[j] (b200mvs_get_level) and its
 * camera, in entry order; views_out_or_null has one record per entry. */
int b200mvs_pset_add_reconstruction_levels(b200mvs_pset* ps, b200mvs_ctx* ctx, const b200mvs_settings* s,
                                           int n_refs, const int32_t* ref_views, const int32_t* levels,
                                           b200mvs_progress* progress, b200mvs_stats* stats,
                                           int32_t* failed_view_or_null, b200mvs_pset_view* views_out_or_null);

#ifdef __cplusplus
}
#endif
#endif /* B200MVS_H */
