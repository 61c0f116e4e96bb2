/*
 * idc_b200.h -- C ABI of the H100-native Local Hints Network forward
 * (interactive deep colorization hot path).
 *
 * The reference has NO native interface: its operator boundary for this path is the
 * Python call
 *     self.net.forward(img_l_mc, input_ab_mc, input_mask_mult, mask_cent)
 *         /root/reference/data/colorize_image.py:263   (ColorizeImageTorch.net_forward)
 *         /root/reference/data/colorize_image.py:308   (ColorizeImageTorchDist.net_forward)
 *     implemented by SIGGRAPHGenerator.forward
 *         /root/reference/models/pytorch/model.py:134-175
 * and, for the Caffe backend, the blob write + net.forward() at
 *         /root/reference/data/colorize_image.py:425-431, 452-463.
 * Every entry point below names the reference statement it replaces.  Plain pointers
 * and sizes only (no torch types); see INTEGRATION.md for the ctypes binding.
 *
 * Conventions
 *   - return value: 0 = IDC_OK, <0 = error (idc_last_error gives the text).
 *   - all image tensors are FP32, NCHW, contiguous (the reference's layout:
 *     model.py:139-141 builds [1,C,H,W] from numpy [C,H,W]).
 *   - idc_forward takes DEVICE pointers and is asynchronous on `stream`;
 *     idc_forward_host takes HOST pointers, copies through pinned staging buffers and
 *     returns after the results are in host memory.
 *   - a ctx is bound to one device, is not thread-safe, and owns packed weights +
 *     activation workspace.  Callers own all I/O buffers.
 *   - H and W must be multiples of 8 (three ::2 subsamplings + three x2 deconvs,
 *     model.py:149-151, :75,:86,:96).
 */
#ifndef IDC_B200_H_
#define IDC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct idc_ctx idc_ctx;

enum {
  IDC_OK = 0,
  IDC_ERR_ARG = -1,          /* bad argument / null pointer / bad shape            */
  IDC_ERR_CUDA = -2,         /* a CUDA call or kernel failed                        */
  IDC_ERR_STATE = -3,        /* wrong call order (e.g. forward before finalize)     */
  IDC_ERR_KEY = -4,          /* unknown / missing state_dict key                    */
  IDC_ERR_UNSUPPORTED = -5,  /* e.g. not an sm_90 device                            */
  IDC_ERR_WATCHDOG = -6,     /* a device-side pipeline wait timed out               */
  IDC_ERR_RANGE = -7         /* an activation reached 65504, FP16's largest value, at its storage exponent
                                (wgmma engine; |v| >= 65488, and values above 65504 saturated).  idc_last_error
                                names the buffers.  idc_forward_host(_q) return it from the forward that saturated;
                                after an idc_forward, the next forward call on the context returns it (before
                                running). */
};

/* idc_create flags */
enum {
  IDC_FLAG_DIST = 1u << 0,        /* also run model_class + softmax (model.py:159-160)           */
  IDC_FLAG_ENGINE_SIMT = 1u << 1, /* FP32 CUDA-core engine (exact FP32, slow); default = wgmma */
  IDC_FLAG_FAST_FP16 = 1u << 2,   /* single-pass FP16 operands (1 MMA / product; measured on an H100:
                                     5.3e-2..1.35e-1 max ab error vs FP64, 2.6e-3 dist, DESIGN §5);
                                     default = 2-term split FP16 (3 MMAs / product, <=1e-3)      */
  IDC_FLAG_GLOBAL_HINTS = 1u << 3,/* global-hints branch (models/global_model/deploy_nodist.prototxt:38-172,501-527) */
  IDC_FLAG_NO_GRAPH = 1u << 4,    /* do not capture the forward into a CUDA graph               */
  IDC_FLAG_KEEP_CONV10 = 1u << 5, /* materialise conv10_2 (debug); default fuses model_out into model10.1 */
  IDC_FLAG_CAFFE313 = 1u << 6     /* Caffe-spec 313-bin hyper-column head (deploy_nopred.prototxt:651-850) */
};

/* dtype codes for idc_load_tensor */
enum { IDC_F32 = 0, IDC_F64 = 1, IDC_I64 = 2 };

/* Library / build info: "idc_b200 <version> sm_90a ..." */
const char* idc_version(void);

/* Replaces `model.SIGGRAPHGenerator(dist=dist)` + `.cuda()` + `.eval()`
 * (data/colorize_image.py:221,230-232).  max_n = largest batch a forward may carry. */
int idc_create(int device, int max_n, int h, int w, unsigned flags, idc_ctx** out);

/* Plan-time options (replace the IDC_* environment switches of round 1; a library embedded in another process
 * must not read process-global state).  Call between idc_create and idc_finalize_weights / idc_adopt_weights;
 * a later call re-plans the launches.  -1 = automatic where it applies.
 *   "halo"          0 / 1 / 3   halo-tile A operand (one TMA tile per 64 input channels serves all 9 taps)
 *   "pairs"         0 / 1 / 2   clusters of two CTAs sharing each weight tile: never (default) / large launches / always
 *   "mt"            1 / 2       128-pixel M-tiles per CTA tile (2 runs the layer with 64-column tiles)
 *   "chunk_kb"      >= 1        k-blocks summed inside the tensor core before the FP32 round-to-nearest add
 *   "split_k"       >= 1        K slices per tile on launches that cannot fill the machine
 *   "conv1_1_umma"  0 / 1       model1.0 on the tensor cores (default 1); 0 = the exact-FP32 CUDA-core kernel
 *   "host_pipe"     0 / 1       idc_forward_host: chunked copy/compute overlap for batches >= 8
 *   "pdl"           0 / 1       programmatic dependent launch between the kernels of one forward
 *   "side_dist"     0 / 1       batches <= 4: run the dist head (class + softmax) on a side stream / graph branch
 *   "tanh_scale"    110 / 100   regression head scale: tanh * 110 (model.py:175) or the Caffe nets' 100
 *                               (models/reference_model/deploy_nodist.prototxt:812-822, SURVEY q4)
 *   "act_exp.<buffer>"  [-24, 24]  wgmma engine: the storage exponent of one activation buffer ("conv4_3", "a8_1", ...;
 *                               idc_act_exponent), replacing the one chosen from the weights.  Only before
 *                               idc_finalize_weights: IDC_ERR_STATE once the weights are packed.
 * Unknown names return IDC_ERR_KEY.  A re-plan that fails returns its error and leaves the context refusing forwards
 * with IDC_ERR_STATE until a later re-plan (idc_set_option or idc_adopt_weights) succeeds. */
int idc_set_option(idc_ctx* ctx, const char* name, int value);

/* Replaces one entry of `self.net.load_state_dict(state_dict)` (data/colorize_image.py:229).
 * key = reference state_dict key ("model1.0.weight", "model1.4.running_var", ...; conv OIHW,
 * deconv IOHW, model.py:13-108).  Extra keys accepted with IDC_FLAG_GLOBAL_HINTS:
 * "glob.{0,1,2,3}.weight/bias" + "glob.{0..3}.bn.*".  data is HOST memory. */
int idc_load_tensor(idc_ctx* ctx, const char* key, const void* data, int dtype, int ndim,
                    const int64_t* dims);

/* Packs every loaded tensor into the device-resident weight arena (K-major FP16 hi/lo
 * tiles for wgmma, FP32 [K][Cout] for the SIMT engine; BatchNorm folded to scale/shift).
 * Fails with IDC_ERR_KEY if a required key is missing. */
int idc_finalize_weights(idc_ctx* ctx);

/* Device pointer + size of the packed arena: rank 0 broadcasts it once over NCCL
 * (SURVEY 8e); ranks != 0 call idc_adopt_weights() after receiving into it. */
int idc_weights_arena(idc_ctx* ctx, void** dev_ptr, size_t* bytes);
int idc_reserve_weights(idc_ctx* ctx);    /* allocate the arena without packing (receiver side) */
int idc_adopt_weights(idc_ctx* ctx);      /* mark a received arena as final                     */
/* The arena does not hold IDC_FLAG_CAFFE313's bin centres: load "caffe.pts_in_hull" [313,2] (idc_load_tensor) before
 * idc_adopt_weights, which fails with IDC_ERR_KEY without it. */

/* Replaces `self.net.forward(img_l_mc, input_ab_mc, input_mask_mult, mask_cent)`
 * (data/colorize_image.py:263 / :308), batched.
 *   L_mc  [n,1,h,w]  L-50 in [-50,50]        ab [n,2,h,w] in [-110,110]
 *   mask  [n,1,h,w]  in [0,1]                maskcent: model.py:142
 *   glob  [n,316] or NULL: [313 ab histogram, 1 indicator, 1 mean saturation, 1 indicator]
 *         (data/colorize_image.py:452-463; deploy_nodist.prototxt:8-18)
 *   out_ab   [n,2,h,w]  tanh*110 (model.py:175).  NOTE the reference's dist=True return is
 *            tanh*110*110 (model.py:166-168, quirk q1); the Python mirror applies that.
 *   out_dist [n,529,h/4,w/4] or NULL: softmax(0.2*model_class(conv8_3)) BEFORE the nearest
 *            x4 upsample (model.py:160); requires IDC_FLAG_DIST.
 *   out_rgb  [n,h,w,3] uint8 or NULL: lab2rgb_transpose(L, out_ab)
 *            (data/colorize_image.py:20-28,264).
 * All pointers are DEVICE memory; asynchronous on `stream` (a cudaStream_t). */
int idc_forward(idc_ctx* ctx, int n, int h, int w, const float* L_mc, const float* ab,
                const float* mask, float maskcent, const float* glob, float* out_ab,
                float* out_dist, uint8_t* out_rgb, void* stream);

/* Same with HOST pointers (synchronous).  This is the call the reference-facing wrapper and bench.py's e2e leg use.
 * Batches <= 4 (the interactive click) replay ONE CUDA graph: a single H2D of the staged inputs, the kernels chained by
 * programmatic dependent launch, a single D2H of the results; batches >= 8 copy straight from / to pinned caller
 * buffers (pageable ones are staged) and overlap the copies with the first / last layer in image chunks.
 * L_mc may be NULL when idc_set_image has made the n L planes resident (then only the hints travel).
 * Results are bit-identical to idc_forward. */
int idc_forward_host(idc_ctx* ctx, int n, int h, int w, const float* L_mc, const float* ab,
                     const float* mask, float maskcent, const float* glob, float* out_ab,
                     float* out_dist, uint8_t* out_rgb);
/* Same + the reference's QUANTISED `self.output_ab` (row a11): out_abq [n,2,h,w] float64 =
 * rgb2lab(out_rgb)[1:] (`_set_out_ab_`, data/colorize_image.py:196-198,267; what the GUI and get_img_fullres read,
 * ui/gui_draw.py:280, :123-131), computed on the device from the just-quantised uint8 pixel, so the wrapper's
 * net_forward is ONE call and one round trip.  out_abq needs out_rgb; NULL = idc_forward_host. */
int idc_forward_host_q(idc_ctx* ctx, int n, int h, int w, const float* L_mc, const float* ab,
                       const float* mask, float maskcent, const float* glob, float* out_ab,
                       float* out_dist, uint8_t* out_rgb, double* out_abq);

/* The reference splits a session into `set_image` / `load_image` (the L plane, once per photo:
 * data/colorize_image.py:68-77, :186-189) and `net_forward(input_ab, input_mask)` (per click, :249).  idc_set_image is
 * the first half: it uploads the n mean-centred L planes [n,1,h,w] once; idc_forward_host(_q) calls with
 * L_mc == NULL and the same n then reuse them, so a click moves only the hints (3/4 of the input bytes).
 * n = 0 or L_mc = NULL forgets the image. */
int idc_set_image(idc_ctx* ctx, int n, int h, int w, const float* L_mc);

/* Hint lists: the GUI's and the notebook's hint IS a rectangle painted with one colour (ui/ui_control.py:52-63
 * PointEdit.updateInput, DemoInteractiveColorization.ipynb put_point), so a click can send the list instead of the
 * dense ab + mask planes.  Raster semantics: pixel (y, x) of image i takes the LAST hint in list order with img == i,
 * y0 <= y <= y1 and x0 <= x <= x1 -> ab = (a, b), mask = 1; no hint -> ab = 0, mask = 0.  Rectangles are inclusive,
 * are clipped to the image, and are empty when y1 < y0 or x1 < x0.  a, b are in the units of the `ab` plane of
 * idc_forward_host, the mask value 1 is what the `mask` plane would hold.
 * idc_set_hints copies the list (HOST memory, 0 <= count <= IDC_MAX_HINTS) into a pinned block of the ctx;
 * idc_forward_host(_q) with ab == NULL && mask == NULL then rasterises that list on the device (hint mode) instead of
 * uploading planes.  Hint mode combines with L_mc == NULL (resident image): a click uploads only the hint block.
 * Errors: IDC_ERR_STATE when idc_set_hints was never called, IDC_ERR_ARG when only one of ab / mask is NULL or a hint's
 * img is outside [0, n) of the forward.  Changing the list never re-captures the click graph (the count travels in the
 * block).  The device-pointer idc_forward has no hint mode. */
typedef struct { int32_t img, y0, x0, y1, x1; float a, b; } idc_hint;
#define IDC_MAX_HINTS 1024
int idc_set_hints(idc_ctx* ctx, int count, const idc_hint* hints);

/* Page-locked host memory for the zero-copy click path: when every buffer handed to idc_forward_host(_q) with
 * n <= 4 comes from idc_host_alloc (or is otherwise pinned), the copy nodes of the click graph read / write the caller's
 * memory directly (no staging copy by the CPU); buffers laid out back to back -- [L | ab | mask (| glob)] and
 * [out_ab | out_rgb | out_abq] -- travel as one copy each way.  The graph is re-captured when the pointers change, so
 * keep the buffers for the lifetime of the session (LhnContext.click_buffers does). */
void* idc_host_alloc(size_t bytes);
int idc_host_free(void* p);

/* Interactive path: keep the 529-bin distribution of the last idc_forward_host on the device instead
 * of copying all of it back (8.7 MB at 256^2) -- the reference only ever reads one pixel of it per click
 * (`self.dist_ab[:, h, w]`, data/colorize_image.py:329).  With resident mode on, idc_forward_host runs the
 * dist head even when out_dist is NULL; idc_fetch_dist then copies dist[img, :, y4, x4] (529 floats) to
 * host memory, or the whole [529, h/4, w/4] plane when y4 < 0. */
int idc_set_dist_resident(idc_ctx* ctx, int on);
int idc_fetch_dist(idc_ctx* ctx, int img, int y4, int x4, float* out_host);

/* The click itself (BASELINE config 5; ui/gui_draw.py:126-142 -> predict_color / suggest_color): tell the context
 * BEFORE the forward which pixel (img, y4, x4) of the (h/4 x w/4) distribution grid the user clicked and how many colour
 * suggestions K (0 = none) the GUI will ask for.  The next idc_forward_host(_q) with n <= 4 and resident mode on then
 * also gathers that pixel's 529-bin pmf and clusters it (idc_ab_reccs with the default 8 restarts / 100 iterations /
 * PyTorch gamut grid) on the dist head's side branch of the click graph -- off the critical path -- and brings the
 * pmf and the picked suggestions (2.6 KB) back with the same graph launch: idc_fetch_dist / idc_ab_reccs for the same
 * pixel (and K) then return from pinned host memory without touching the device.  The coordinates live in mapped host memory and are read when the
 * graph runs, so moving the click never re-captures the graph.  y4 < 0 switches the mode off (one re-capture). */
int idc_set_click(idc_ctx* ctx, int img, int y4, int x4, int K);

/* Colour suggestions at one pixel of the resident distribution (SURVEY row f2; replaces
 * ColorizeImageTorchDist.get_ab_reccs, data/colorize_image.py:322-354: 25 000 inverse-CDF samples of
 * dist_ab[:, h, w] -> sklearn KMeans(K) -> centres ordered by occupancy).  Computed as the sample-size ->
 * infinity limit of that procedure: deterministic weighted k-means over the 529 gamut points with the pmf
 * as weights (seeds: heaviest bin, then argmax w*d^2; FP64 Lloyd iterations until the assignment is stable
 * or max_iter); n_init restarts run side by side (restart v seeds from the bin of weight-rank v) and the one
 * with the lowest inertia wins (sklearn's n_init; 1 <= n_init <= 16).  pts_host: [529][2] ab coordinates of the bins, or NULL for the PyTorch wrapper's grid
 * (bin i = (g[i % 23], g[i / 23]), g = -110..110 step 10, :283).  Outputs (host): centers [K][2], conf [K]
 * (cluster mass, descending; may be NULL), iters_out (Lloyd iterations used; may be NULL).  1 <= K <= 32.  The best
 * restart is picked on the device.  Runs on the legacy default stream in the context scratch of idc_ab_reccs_batch:
 * a batched call still running on another stream must be waited for first. */
int idc_ab_reccs(idc_ctx* ctx, int img, int y4, int x4, int K, int max_iter, int n_init, const float* pts_host,
                 float* centers_host, float* conf_host, int* iters_out);
/* Same clustering for a caller-supplied pmf (host, 529 floats, need not be normalised); no ctx needed. */
int idc_ab_reccs_pmf(int device, const float* pmf_host, int K, int max_iter, int n_init, const float* pts_host,
                     float* centers_host, float* conf_host, int* iters_out);
/* idc_ab_reccs for many pixels of the images of the context's LAST forward (any forward entry point; resident mode is
 * not needed), in one stream-ordered pass: queries_host [q][3] int32 (img, y4, x4) on the (h/4 x w/4) grid.  Each
 * query's pmf is computed from the class logits by the per-pixel routine of the full-map softmax (bit-identical to
 * dist[img, :, y4, x4]), all q x n_init restarts run in one launch, and the best restart of each query is picked on the
 * device by idc_ab_reccs's rule.  Query i's answer equals idc_ab_reccs on the same forward bit for bit, whatever its
 * position in the list, and repeated queries get the same answer.  Outputs (DEVICE memory, float32 / int32):
 * centers_dev [q][K][2], conf_dev [q][K] (may be NULL), iters_dev [q] (may be NULL), pmf_dev [q][529] (may be
 * NULL: each query's pmf, the 529 floats of dist[img, :, y4, x4]).  pts_host: [529][2] HOST, or NULL
 * for the PyTorch wrapper's grid.  Asynchronous on `stream` with no host synchronisation: the queries and the points
 * travel as kernel parameters, so the host arrays may be reused as soon as the call returns.  Scratch (14.7 KB per
 * query) belongs to the context and grows, stream-ordered, only when q exceeds every earlier q; calls on different
 * streams must be ordered by the caller, as must the next forward (it overwrites the logits).  1 <= q <=
 * IDC_MAX_RECCS_QUERIES (the k-means grid has one row per query).  IDC_ERR_STATE without IDC_FLAG_DIST or before any
 * forward; IDC_ERR_ARG for q, K, max_iter, n_init out of range (as idc_ab_reccs), a NULL queries or centers, and a
 * query whose img is outside [0, n) of the last forward or whose pixel is off the grid (idc_last_error names it), all
 * before any device call. */
#define IDC_MAX_RECCS_QUERIES 65535
int idc_ab_reccs_batch(idc_ctx* ctx, int q, const int32_t* queries_host, int K, int max_iter, int n_init,
                       const float* pts_host, float* centers_dev, float* conf_dev, int32_t* iters_dev, float* pmf_dev,
                       void* stream);

/* Caffe-spec 313-bin head (SURVEY row a14; models/reference_model/deploy_nopred.prototxt:651-850, weight
 * injection data/colorize_image.py:405-413).  With IDC_FLAG_CAFFE313 every forward also runs the
 * hyper-column (conv3_pred + conv4..7_pred + conv8_pred, ReLU) and pred_313 (1x1 -> 313 logits at h/4).
 * Extra state_dict keys: "caffe.conv{3..8}_pred.{weight,bias}" (conv3/8: [384,256,3,3]; conv4..7: Caffe
 * Deconvolution [512,384,4,4]), "caffe.pred_313.{weight,bias}" [313,384,1,1], "caffe.pts_in_hull" [313,2].
 *   idc_caffe313_pred_ab:    two grouped bilinear x2 deconvs (kernel [[.25,.5,.25,0],[.5,1,.5,0],[.25,.5,.25,0],0])
 *                            -> softmax(T * logits) -> annealed mean over the 313 bin centres = pred_ab [n,2,h,w]
 *                            (DEVICE pointer; T = 2.6 in the reference, :827-848).
 *   idc_caffe313_dist_pixel: dist_ab_S[:, y, x] = softmax(S * upsampled logits) at ONE full-resolution
 *                            pixel (S = 0.2, :808-820) -> 313 floats in HOST memory.
 *   idc_caffe313_dist_map:   the whole dist_ab_S blob (`self.net.blobs['dist_ab_S'].data`, data/colorize_image.py:499)
 *                            -> out_dist [n,313,h,w] DEVICE memory, asynchronous on `stream`.  Every pixel equals
 *                            idc_caffe313_dist_pixel bit for bit.  IDC_ERR_ARG for n outside [1, max_n] or NULL,
 *                            IDC_ERR_STATE without IDC_FLAG_CAFFE313. */
int idc_caffe313_pred_ab(idc_ctx* ctx, int n, float T, float* out_ab, void* stream);
int idc_caffe313_dist_pixel(idc_ctx* ctx, int img, int y, int x, float S, float* out313_host);
int idc_caffe313_dist_map(idc_ctx* ctx, int n, float S, float* out_dist, void* stream);
/* Colour suggestions of the Caffe distribution model (ColorizeImageCaffeDist.get_ab_reccs, data/colorize_image.py:
 * 515-547) at many pixels of the images of the context's LAST forward, in one stream-ordered pass: idc_ab_reccs_batch
 * with the 313-bin head.  queries_host [q][3] int32 (img, y, x) are FULL-resolution pixels (the head's dist_ab_S is the x4
 * up-sample of the logits).  Each query's pmf is dist_ab_S[img, :, y, x] (the first 313 floats equal
 * idc_caffe313_dist_pixel(img, y, x, S) bit for bit) padded with 216 zeros, the k-means points are the context's
 * caffe.pts_in_hull padded with 216 rows of (0, 0), and each query's answer equals idc_ab_reccs_pmf on that padded pmf and
 * those points bit for bit.  Outputs as idc_ab_reccs_batch (DEVICE memory; pmf_dev [q][529] may be NULL), the same
 * context scratch, no host synchronisation, the same ordering rules.  IDC_ERR_STATE without IDC_FLAG_CAFFE313 or before
 * any forward; IDC_ERR_ARG for q, K, max_iter, n_init out of range (as idc_ab_reccs_batch), a non-finite S, a NULL
 * queries or centers, and a query whose img is outside [0, n) of the last forward or whose pixel is outside h x w
 * (idc_last_error names it), all before any device call. */
int idc_caffe313_reccs_batch(idc_ctx* ctx, int q, const int32_t* queries_host, float S, int K, int max_iter, int n_init,
                             float* centers_dev, float* conf_dev, int32_t* iters_dev, float* pmf_dev, void* stream);

/* Distribution entropy (`compute_entropy`, data/colorize_image.py:356-358 and :545-547:
 * `np.sum(dist_ab * np.log(dist_ab), axis=0)`, the NEGATIVE entropy): out[i, p] = sum_k dist[i, k, p] * logf(dist[i, k, p])
 * in float32, bins summed in order 0 .. bins-1 like numpy's axis-0 sum; a zero bin gives NaN, as in numpy.
 *   idc_negentropy:       dist [n,bins,hw] -> out [n,hw], DEVICE ptrs, asynchronous on `stream` (also serves an
 *                         out_dist of idc_forward or of idc_caffe313_dist_map).
 *   idc_dist_negentropy:  the resident 529-bin distribution of image img (idc_set_dist_resident) -> out [h/4, w/4]
 *                         HOST memory; IDC_ERR_STATE when no resident distribution holds image img. */
int idc_negentropy(int device, int n, int bins, int hw, const float* dist, float* out, void* stream);
int idc_dist_negentropy(idc_ctx* ctx, int img, float* out_host);

/* Stand-alone post-process: lab2rgb_transpose (data/colorize_image.py:20-28).
 * L [n,1,h,w] in [0,100] (NOT mean-centred), ab [n,2,h,w] -> rgb [n,h,w,3] uint8. DEVICE ptrs. */
int idc_lab2rgb_u8(int device, int n, int h, int w, const float* L, const float* ab,
                   uint8_t* rgb, void* stream);

/* f1 (steps either side of the network), float64 like the reference's numpy/skimage/scipy path; DEVICE ptrs.
 * idc_rgb2lab_f64:      skimage color.rgb2lab of uint8 RGB [n,h,w,3] -> Lab planes [n,3,h,w] float64
 *                       (data/colorize_image.py:31-36, :172-178 image prep, :196-198 _set_out_ab_). */
int idc_rgb2lab_f64(int device, int n, int h, int w, const uint8_t* rgb, double* lab, void* stream);
/* f3: global statistics of a reference image (models/global_model/global_stats.prototxt:1-244; NNEncLayer with
 * NN=1, caffe_files/caffe_traininglayers.py:161-196; usage DemoGlobalHistogramTransfer.ipynb:176-182):
 * uint8 RGB [h,w,3] (h,w multiples of 4) + the 313 ab bin centres [313,2] -> out[316] =
 * [313-bin histogram of the 4x4-pooled ab, 1, mean HSV saturation, 1] = the `glob` input of idc_forward. DEVICE ptrs.
 * The histogram is idc_global_stats_batch's bit for bit (the same cell rule); s_avg is summed in another fixed order.
 * The same bytes on every run.  Its scratch is allocated and released stream-ordered (cudaMallocAsync /
 * cudaFreeAsync): the call does not wait for the device. */
int idc_global_stats(int device, int h, int w, const uint8_t* rgb, const float* pts313, float* out316, void* stream);
/* f1, get_img_fullres (:123-131): scipy.ndimage.zoom(order=1) of ab [2,h_in,w_in] float64 to [h,w], then
 * lab2rgb_transpose with the full-resolution L [h,w] -> uint8 [h,w,3].  The same call as
 * idc_render_planes_u8(device, h_in, w_in, ab, 1, 0, NULL, 0, IDC_RENDER_L_PLANE, L_full, h, w, rgb, stream), so the
 * zoom follows scipy's edge rule below; IDC_ERR_ARG also for a NULL ab. */
int idc_zoom_lab2rgb_u8(int device, int h_in, int w_in, const double* ab, int h, int w, const double* L_full,
                        uint8_t* rgb, void* stream);
/* f1, the full-resolution renders of the wrapper (data/colorize_image.py):
 *   get_img_gray_fullres   (:119-121)  lab2rgb_transpose(img_l_fullres, 0)
 *   get_input_img_fullres  (:133-136)  lab2rgb_transpose(img_l_fullres, zoom(input_ab, order=1))
 *   get_img_mask_fullres   (:145-149)  lab2rgb_transpose(100. * (1 - zoom(input_mask, order=0)), 0)
 *   get_sup_fullres        (:154-158)  lab2rgb_transpose(50 * zoom(input_mask, order=0), zoom(input_ab, order=0))
 * -> uint8 rgb [h,w,3].  ab [2,h_in,w_in] (NULL: ab = 0) is zoomed to [h,w] with ab_order 0 or 1 exactly as
 * scipy.ndimage.zoom (1.18) does it, mode 'constant': a sample whose coordinate o * ((n_in-1)/(n_out-1)) lies past the
 * last input reads 0.  ab_f32 = 1 rounds the zoomed ab to float32 (scipy's result for a float32 plane).  L is
 *   IDC_RENDER_L_PLANE  the plane L [h,w]
 *   IDC_RENDER_L_MASK   100 * (1 - m)        m = mask [h_in,w_in] zoomed with order 0 (the same edge rule)
 *   IDC_RENDER_L_SUP    50 * m
 * with mask_f32 = 1 evaluating those statements in float32 (numpy's result for a float32 mask).  float64 otherwise.
 * DEVICE ptrs, asynchronous on `stream`.  IDC_ERR_ARG, before any device call, for h, w, h_in, w_in < 1, ab_order,
 * ab_f32 or mask_f32 outside {0, 1}, an unknown l_mode or a NULL plane that l_mode reads, and a NULL rgb. */
enum { IDC_RENDER_L_PLANE = 0, IDC_RENDER_L_MASK = 1, IDC_RENDER_L_SUP = 2 };
int idc_render_planes_u8(int device, int h_in, int w_in, const double* ab, int ab_order, int ab_f32, const double* mask,
                         int mask_f32, int l_mode, const double* L, int h, int w, uint8_t* rgb, void* stream);

/* f1, image-load side (data/colorize_image.py:52-66): cv2.resize(im, (w_dst, h_dst)) of a uint8 [h,w,3] image with
 * OpenCV's default INTER_LINEAR -- the 8-bit path of OpenCV is fixed-point arithmetic and is restated integer for
 * integer (bit-identical to cv2, incl. the exact-2x shortcut to area averaging).  DEVICE ptrs. */
int idc_resize_u8_linear(int device, int h_src, int w_src, const uint8_t* src, int h_dst, int w_dst, uint8_t* dst,
                         void* stream);
/* f1, GUI display step (ui/gui_draw.py:280-283): cv2.resize(ab [2,h_in,w_in] float64, (w,h), INTER_CUBIC), concatenated
 * with the window-size L [h,w] float64, skimage lab2rgb, clip, x255, truncating cast -> uint8 [h,w,3].  The resize
 * evaluates OpenCV's float32 weights and float64 tap sums in OpenCV's order, so the resized ab equals cv2's bit for
 * bit.  DEVICE ptrs. */
int idc_cubic_lab2rgb_u8(int device, int h_in, int w_in, const double* ab, int h, int w, const double* L, uint8_t* rgb,
                         void* stream);
/* The GUI's gamut map (data/lab_gamut.py:66-78, abGrid(gamut_size, D).update_gamut(L), called on every colour change
 * by ui/gui_gamut.py): for the A x B grid a = -gamut_size + i*D (row i), b = -gamut_size + j*D (column j),
 * A = B = len(np.arange(-gamut_size, gamut_size + D, D)):
 *   rgb  = trunc(255 * clip(lab2rgb(L, a, b), 0, 1))  (uint8)
 *   mask = |(L, a, b) - rgb2lab(rgb)|_2 < 1            (uint8 0 / 1)
 * and rgb = 255 where mask is 0 (`masked_rgb`).  float64 like the reference; rgb [A][B][3], mask [A][B] DEVICE ptrs. */
int idc_gamut_ab(int device, double L, int gamut_size, int D, uint8_t* rgb, uint8_t* mask, void* stream);

/* Batched photos (automatic colorization of many photos; reference: load_image + net_forward + get_img_fullres +
 * get_result_PSNR per photo, data/colorize_image.py:52-66, :98-109, :123-131, :249-267).  A batch is n <= IDC_MAX_PHOTOS
 * photos of any sizes packed back to back in ONE device buffer of uint8 RGB; the table (HOST memory, checked before
 * any device call and passed to the kernels by value) gives each photo's first pixel and size.  Photos must not
 * overlap: off[i] + h[i] * w[i] <= off[i + 1].  X is the network size (a multiple of 8).  DEVICE data pointers,
 * asynchronous on `stream`.  IDC_ERR_ARG, before any device call, for n outside [1, IDC_MAX_PHOTOS], a NULL pointer
 * that is not optional, h or w outside [1, IDC_MAX_PHOTO_SIDE], overlapping photos, X outside [8, IDC_MAX_PHOTO_X] or
 * not a multiple of 8, and a hint count above IDC_MAX_HINTS. */
typedef struct { int64_t off; int32_t h, w; } idc_photo;   /* off = first pixel, in pixels */
#define IDC_MAX_PHOTOS 128
#define IDC_MAX_PHOTO_SIDE 16777216   /* 2^24: pixel and byte indices within one photo row stay in 32 bits */
#define IDC_MAX_PHOTO_X 16384         /* X * X * 3 stays in 32 bits */
/* load_image (:52-66) + the mean-centring of set_image (:68-77, :172-178) for every photo: cv2.resize(photo, (X, X))
 * with OpenCV's 8-bit INTER_LINEAR (the same arithmetic as idc_resize_u8_linear, exact-2x area shortcut included),
 * skimage rgb2lab, L_mc = (float)(L - 50) -> L_mc [n,1,X,X] float32 (idc_forward's input); rgb [n,X,X,3] uint8 = the
 * network-size photo (`img_rgb`), or NULL. */
int idc_photo_prep(int device, int n, const idc_photo* photos, const uint8_t* src, int X, float* L_mc, uint8_t* rgb,
                   void* stream);
/* get_img_fullres (:123-131) for every photo: L of each full-resolution pixel from its own source pixel (skimage
 * rgb2lab, no Lab plane is stored), ab = scipy.ndimage.zoom(order=1) of the photo's quantised output_ab (planes 1-2 of
 * lab [n,3,X,X] float64, as idc_rgb2lab_f64 writes them from idc_forward's out_rgb) with idc_render_planes_u8's edge
 * rule, then lab2rgb_transpose -> out, uint8 RGB in the layout of src.  Each pixel reads only its own source pixel,
 * so out may be src (in place). */
int idc_photo_render(int device, int n, const idc_photo* photos, const uint8_t* src, int X, const double* lab,
                     uint8_t* out, void* stream);
/* The hint raster of idc_set_hints on caller planes: block = [16-byte header {count, 0, 0, 0} | count idc_hint] in
 * DEVICE memory (the kernel reads the count from the header); count (HOST) is the same count, checked against
 * IDC_MAX_HINTS.  Pixel (y, x) of image i in [0, n) takes the last hint with img == i that covers it -> ab [n,2,h,w],
 * mask [n,1,h,w] float32, exactly the planes idc_forward_host's hint mode feeds the network.  n <= 65535 and
 * h * w < 2^31 - 256. */
int idc_hint_raster(int device, int n, int h, int w, int count, const void* block, float* ab, float* mask, void* stream);
/* get_result_PSNR (:98-109) before its float64 tail: sse[i] = sum over the h*w*3 values of image i of (a - b)^2, exact in
 * int64, for uint8 images a, b [n,h,w,3] (img_rgb, output_rgb), n <= 65535.  20 * log10(255 / sqrt(sse / (h*w*3))) on the host then
 * equals numpy's result bit for bit. */
int idc_rgb_sse(int device, int n, int h, int w, const uint8_t* a, const uint8_t* b, int64_t* sse, void* stream);
/* Hints coloured from the ground truth: the notebook's put_point(input_ab, mask, loc, p, val) (DemoInteractive-
 * Colorization.ipynb) with val taken from the photo itself, as a simulated user who reveals points of the true colours.
 * blocks = n_blocks hint blocks in idc_hint_raster's layout, block b at blocks + b * block_stride, DEVICE memory; block
 * b belongs to photo b / levels of lab [*,3,X,X] float64 (as idc_rgb2lab_f64 writes it from idc_photo_prep's rgb).
 * Every hint of a block (its count read from the header on the device, clamped to [0, IDC_MAX_HINTS] and to what
 * block_stride holds) gets (a, b) = the mean of planes 1-2 of that photo over its rectangle clipped to X x X, summed in
 * float64 in row-major order, divided by the pixel count and rounded once to float32; an empty rectangle gets (0, 0).
 * The rectangles and img fields are left as they are; each block is then one idc_hint_raster block.  Deterministic.
 * Asynchronous on `stream`.  IDC_ERR_ARG, before any device call, for n_blocks outside [1, 65535], levels < 1, X
 * outside [1, IDC_MAX_PHOTO_X], NULL lab or blocks, and a block_stride below 16 or blocks / block_stride not a
 * multiple of 4. */
int idc_hint_fill_mean(int device, int n_blocks, int levels, int X, const double* lab, void* blocks, size_t block_stride,
                       void* stream);
/* Global-hints statistics of a batch of network-size images (global_stats.prototxt, as idc_global_stats): rgb [n,h,w,3]
 * uint8 (the layout idc_photo_prep writes img_rgb in), pts313 [313,2] -> out [n,316] float32, row i = [313-bin
 * histogram, 1, s_avg, 1], the `glob` layout of idc_forward.  Per 4x4 cell: the Lab of its 16 pixels (the arithmetic of
 * idc_rgb2lab_f64), a and b summed in float64 in row-major order, / 16, rounded once to float32; the cell's bin is the
 * first minimum of the float32 squared distance with every operation rounded separately (numpy's
 * ((ab - pts)**2).sum(-1)).  hist[k] = float32(count_k / cells) from float64; s_avg = float32 of the float64 mean of
 * skimage's HSV saturation over the h*w pixels, summed in a fixed order.  One CTA per image; a row is identical bit for
 * bit whatever n, wherever the image sits in the batch, and on every run.  Reads no host memory and allocates nothing,
 * so it can be captured in a graph.  DEVICE ptrs, asynchronous on `stream`.  IDC_ERR_ARG, before any device call, for
 * n outside [1, 65535], h or w below 4, not a multiple of 4 or above IDC_MAX_PHOTO_X, and a NULL pointer. */
int idc_global_stats_batch(int device, int n, int h, int w, const uint8_t* rgb, const float* pts313, float* out,
                           void* stream);

/* Colorization by optimization (Levin, Lischinski & Weiss, SIGGRAPH 2004) on a reveal sweep's hint planes: the
 * classical baseline of PhotoColorizer.reveal_sweep(method="levin"); the rule is DESIGN.md §4b's.  DEVICE pointers,
 * asynchronous on `stream`.
 * idc_levin_weights: lab [n,3,h,w] float64 (idc_rgb2lab_f64) -> wts [n,8,h,w] float64.  With Y = L / 100 and N(p) the
 *   3 x 3 window around p without p, clipped to the image: s = max(0.6 * var(Y over N(p) and p), -min_q (Y(q) - Y(p))^2
 *   / ln 0.01, 2e-6), w_pq = exp(-(Y(q) - Y(p))^2 / s) normalised to sum 1 over N(p).  Plane k holds neighbour
 *   (y + dy, x + dx) with (dy, dx) the k-th of (-1,-1) (-1,0) (-1,1) (0,-1) (0,1) (1,-1) (1,0) (1,1); 0 outside the
 *   image.  Each operation rounded on its own.  IDC_ERR_ARG, before any device call, for n outside [1, 65535], h or w
 *   outside [2, IDC_MAX_PHOTO_X] and a NULL pointer. */
int idc_levin_weights(int device, int n, int h, int w, const double* lab, double* wts, void* stream);
/* idc_levin_solve: for each image i of n and each channel c of ab, the u with u_p = ab_hint[i,c,p] where mask[i,0,p] > 0
 *   and u_p - sum_q w_pq u_q = 0 elsewhere, w being photo i / levels of wts -> out_ab [n,2,h,w] float32 (the hints as
 *   they are on hinted pixels).  FP64 BiCGSTAB from u = 0 on the system reduced to the free pixels, one CTA per image,
 *   the iterations on the device.  A channel stops when its true relative residual ||b - A u|| / ||b|| (b = the hinted
 *   columns moved to the right) is at most tol, or after max_iter iterations; iters [n,2] int32 and relres [n,2]
 *   float64 receive each channel's iteration count and the true relative residual it stopped at (0 for b = 0: an image
 *   without hints, or whose hints no free pixel depends on, gets u = 0 exactly).  Free pixels that depend on no hint
 *   through non-zero weights get 0 (DESIGN.md §4b).  relres > tol after the call means "not converged".  Every sum in a
 *   fixed order: an image's result is the same bit for bit whatever n, its position and the other images.  ab_hint
 *   [n,2,h,w] and mask [n,1,h,w] float32 as idc_hint_raster writes them.  workspace: idc_levin_workspace_bytes(n, h, w)
 *   bytes of DEVICE scratch, 8-byte aligned, owned by the caller; nothing is allocated.  IDC_ERR_ARG, before any device
 *   call (idc_levin_check runs the same checks, in this order): n outside [1, 65535], h or w outside
 *   [2, IDC_MAX_PHOTO_X], levels outside [1, n], a NULL wts, ab_hint, mask, out_ab, iters, relres or workspace, tol not
 *   in (0, 1), max_iter outside [1, IDC_LEVIN_MAX_ITER], a workspace not 8-byte aligned, and workspace_bytes below
 *   idc_levin_workspace_bytes(n, h, w).
 * idc_levin_workspace_bytes: the workspace idc_levin_solve needs for n images of h x w; 0 for sizes it rejects.
 * idc_lab2rgb_u8_mc: the render of idc_forward's out_rgb on caller planes, L = (double)L_mc + 50 with L_mc [n,1,h,w]
 *   (idc_forward's mean-centred L input) and ab [n,2,h,w] float32 -> rgb [n,h,w,3] uint8: the network's own ab gives
 *   its out_rgb bit for bit.  IDC_ERR_ARG for n, h or w below 1 and a NULL pointer. */
#define IDC_LEVIN_MAX_ITER 10000000
int idc_levin_solve(int device, int n, int levels, int h, int w, const double* wts, const float* ab_hint,
                    const float* mask, double tol, int max_iter, float* out_ab, int32_t* iters, double* relres,
                    void* workspace, size_t workspace_bytes, void* stream);
size_t idc_levin_workspace_bytes(int n, int h, int w);
int idc_lab2rgb_u8_mc(int device, int n, int h, int w, const float* L_mc, const float* ab, uint8_t* rgb, void* stream);

/* ---- introspection / test hooks (used by tests/, never by the product path) ---- */
/* The host argument checks of idc_ab_reccs_batch, the same code, for a context with (has_head != 0) or without the
 * 529-bin head whose last forward carried n_img images of h x w (n_img = 0: no forward yet) -> the code
 * idc_ab_reccs_batch returns; msg (may be NULL) receives idc_last_error's text.  Touches no device. */
int idc_ab_reccs_batch_check(int has_head, int n_img, int h, int w, int q, const int32_t* queries, int K, int max_iter,
                             int n_init, char* msg, size_t msg_bytes);
/* The same for idc_caffe313_reccs_batch: has_head = the context has IDC_FLAG_CAFFE313; queries on the h x w grid. */
int idc_caffe313_reccs_batch_check(int has_head, int n_img, int h, int w, int q, const int32_t* queries, float S, int K,
                                   int max_iter, int n_init, char* msg, size_t msg_bytes);
/* The host argument checks of idc_levin_solve, the same code -> the code idc_levin_solve returns for these arguments;
 * msg (may be NULL) receives the reason.  The pointers are only tested for NULL and alignment.  Touches no device. */
int idc_levin_check(int n, int levels, int h, int w, const double* wts, const float* ab_hint, const float* mask,
                    double tol, int max_iter, const float* out_ab, const int32_t* iters, const double* relres,
                    const void* workspace, size_t workspace_bytes, char* msg, size_t msg_bytes);
/* wgmma engine: the exponent S with which activation `name` is stored (FP16 hi/lo planes of value * 2^S), chosen per
 * buffer from the weights by idc_finalize_weights (DESIGN.md §3); 0 on the SIMT engine.  IDC_ERR_KEY for an unknown
 * name, IDC_ERR_STATE before the weights are packed. */
int idc_act_exponent(idc_ctx* ctx, const char* name, int* exp_out);
/* The activation buffers this context stores, in plan order (like idc_num_ops / idc_op_name): "a1_1", "conv1_2", ...;
 * "conv10_2" only on the SIMT engine or with IDC_FLAG_KEEP_CONV10, "hyper" only with IDC_FLAG_CAFFE313.  NULL outside
 * [0, idc_num_acts). */
int idc_num_acts(idc_ctx* ctx);
const char* idc_act_name(idc_ctx* ctx, int i);
/* *out_host = the largest |a| over images [0, n) of activation `name` as the last forward / idc_run_op /
 * idc_set_activation left it, i.e. the maximum of what idc_get_activation returns, bit for bit, on both engines (wgmma:
 * |hi + lo| * 2^-S).  A NaN anywhere in the buffer comes back as NaN, an infinity as infinity.  One bandwidth-bound
 * pass over the buffer; synchronises the device.  On the wgmma engine this says how close a checkpoint comes to FP16's
 * limit on an image (stored value = result * 2^S against 65504); on the SIMT engine, whose FP32 planes cannot
 * saturate, it is the measurement idc_set_act_range wants.  IDC_ERR_KEY unknown buffer, IDC_ERR_ARG for n outside
 * [1, max_n] or a NULL argument, IDC_ERR_STATE before the weights are packed. */
int idc_act_absmax(idc_ctx* ctx, const char* name, int n, float* out_host);
/* Calibration: "the largest |a| activation `name` takes on representative inputs is max_abs".  The wgmma engine then
 * stores that buffer with S = 10 - ceil(log2 max_abs), which puts the measured maximum in (512, 1024] and leaves 64x
 * of headroom below 65504 for inputs outside the sample, in place of the exponent estimated from the weights
 * (DESIGN.md §3).  "act_exp.<buffer>" still wins over a range; a buffer without a range keeps the weight-derived
 * exponent, so a partial set of ranges is well defined.  An exponent outside [-24, 24] fails idc_finalize_weights,
 * naming the buffer, as for the estimate.  Same life cycle as "act_exp.<buffer>": only before idc_finalize_weights
 * (IDC_ERR_STATE once the weights are packed); IDC_ERR_KEY unknown buffer; IDC_ERR_ARG unless max_abs is finite and
 * > 0.  No effect on the SIMT engine.  A range stays with the context, like an "act_exp.<buffer>" override: weights
 * loaded and packed again later are packed with it, so a context that moves to another checkpoint needs that
 * checkpoint's ranges set again (or a new context).  The resulting exponents live in the weight arena like any others, so a context
 * that receives the arena (idc_reserve_weights + copy + idc_adopt_weights, ranks != 0) stores its activations exactly
 * as the context that packed it, with no call of its own. */
int idc_set_act_range(idc_ctx* ctx, const char* name, double max_abs);
/* Copy a named activation ("conv1_2", "a8_1", ... see DESIGN.md) of the LAST forward to
 * out [n,C,H,W] FP32 device memory; *c,*h,*w receive its shape. */
int idc_get_activation(idc_ctx* ctx, const char* name, float* out_nchw, size_t out_floats,
                       int* c, int* h, int* w);
/* Overwrite a named activation from [n,C,H,W] FP32 device memory, then run ONE op by name. */
int idc_set_activation(idc_ctx* ctx, const char* name, int n, const float* in_nchw);
int idc_run_op(idc_ctx* ctx, const char* op_name, int n, void* stream);
int idc_num_ops(idc_ctx* ctx);
const char* idc_op_name(idc_ctx* ctx, int i);
/* Per-op device timing (CUDA events on the forward's stream, recorded between the op launches).
 * idc_set_profiling(ctx, 1) starts accumulating over subsequent forwards; idc_get_profile
 * synchronises, writes the MEAN milliseconds per forward of slot i into ms[i] (slot 0 = fused
 * pack+conv1_1, slots 1..num_ops = the ops in idc_op_name order, last slot = heads/post) and resets.
 * Returns the number of slots (num_ops + 2) or <0. */
int idc_set_profiling(idc_ctx* ctx, int enable);
int idc_get_profile(idc_ctx* ctx, float* ms, int max_slots);
/* FLOPs (2*MACs) of op i for ONE image (0 for out-of-range i) */
double idc_op_flops(idc_ctx* ctx, int i);
/* kernels launched by the last forward (gpu_launches in bench.py) */
int idc_last_launch_count(idc_ctx* ctx);
/* click-graph instantiations of this ctx so far (a hint-list click must not add one) */
int idc_graph_captures(idc_ctx* ctx);
/* FLOPs (2*MACs, conv+deconv) of one image at the ctx geometry; includes model_class iff DIST */
double idc_flops_per_image(idc_ctx* ctx);

const char* idc_last_error(idc_ctx* ctx);
int idc_destroy(idc_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* IDC_B200_H_ */
