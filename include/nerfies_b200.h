/* nerfies_b200.h - C ABI of the Hopper-native deformable-NeRF render hot path.
 *
 * The reference (google/nerfies) is pure Python/JAX and has no FFI; the seam a
 * replacement plugs into is the Python call surface listed in SURVEY.md §8(b).
 * Each entry point below names the reference callable it replaces
 * (file:line in /root/reference).  The Python host side
 * (nerfies_b200/models.py, evaluation.py) binds these with ctypes and keeps the
 * reference's names / pytree keys / shapes on top.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer on the current CUDA device unless the
 *    function name ends in _host; tensors are contiguous, row-major, float32;
 *    ids are uint32;
 *  - calls enqueue work on `stream` (a cudaStream_t passed as void*) and return
 *    without synchronising (the *_host variant synchronises before returning);
 *  - the caller owns every input/output buffer and keeps it alive until the
 *    stream has passed the call; the library owns only its workspace, allocated
 *    in nfb_create; nothing is allocated on the hot path;
 *  - return value 0 = success, < 0 = error (message via nfb_last_error());
 *  - the tensor-core kernels never hang or trap on an internal protocol error:
 *    a bounded mbarrier wait raises a process-wide abort flag (mapped host
 *    memory), the kernel drains, and the _host entry point / every later call
 *    returns an error ("a tensor-core kernel aborted ..."); results of that launch
 *    are invalid;
 *  - a handle is not thread-safe: one handle per GPU per process/rank.  Its workspace
 *    is shared by its calls: consecutive calls on one stream are ordered by the
 *    stream; when a call arrives on a different stream than the previous one the
 *    library makes the new stream wait for the previous call's work (one event).
 *    Concurrent launches from one handle on two streams are therefore serialised,
 *    not run in parallel - use one handle per stream for that.
 */
#ifndef NERFIES_B200_H_
#define NERFIES_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nfb_handle nfb_handle;

/* Activation selectors: configs.py:27-32 registers exactly these for gin. */
enum nfb_activation {
  NFB_ACT_NONE = 0, NFB_ACT_RELU = 1, NFB_ACT_ELU = 2, NFB_ACT_LEAKY_RELU = 3,
  NFB_ACT_TANH = 4, NFB_ACT_SIGMOID = 5, NFB_ACT_SOFTPLUS = 6
};
enum nfb_warp_type { NFB_WARP_NONE = 0, NFB_WARP_TRANSLATION = 1, NFB_WARP_SE3 = 2 };
/* warp_metadata_encoder_type (configs.py:103; warping.py:109-123, 250-260):
 * GLO   = GloEncoder on metadata['warp'] ids;
 * TIME  = modules.TimeEncoder (modules.py:297-322) on metadata['time'], annealed by
 *         warp_extra['time_alpha'];
 * BLEND = (1 - time_alpha) * glo(id) + time_alpha * TimeEncoder(float(id)) (warping.py:128-133). */
enum nfb_warp_encoder { NFB_WARP_ENC_GLO = 0, NFB_WARP_ENC_TIME = 1, NFB_WARP_ENC_BLEND = 2 };
/* Arithmetic of the MLP GEMMs.  Everything else is always fp32. */
enum nfb_precision {
  NFB_PREC_FP32 = 0,     /* fp32 FFMA on CUDA cores: general (any width / activation / condition) */
  NFB_PREC_BF16 = 1,     /* bf16 operands, fp32 accumulate, wgmma tensor cores: fastest, ~1e-2  */
  NFB_PREC_FP16X3 = 2    /* fp32 emulated on wgmma by three fp16 MMA chains into one fp32
                          * accumulator (x_hi W_hi + x_lo W_hi + x_hi W_lo, hi = fp16(v),
                          * lo = fp16(v - hi): 22 significant bits per operand): the
                          * tensor-core mode that holds the 1e-4 parity gate.  Activations
                          * beyond fp16's range (|v| > 65504) saturate.  (Round 1 reserved this
                          * value as "bf16x3"; a bf16 split leaves 2^-17 per operand, not enough.) */
};

/* Mirrors the NerfModel attributes that shape the forward pass
 * (nerfies/models.py:76-120; filled from ModelConfig, nerfies/configs.py:37-105). */
typedef struct nfb_config {
  int num_coarse_samples;        /* ModelConfig.num_coarse_samples              */
  int num_fine_samples;          /* ModelConfig.num_fine_samples (0: no fine)   */
  int num_nerf_point_freqs;      /* SinusoidalEncoder F for points (models.py:148) */
  int num_nerf_viewdir_freqs;    /* ... for viewdirs (models.py:151)            */
  int num_warp_freqs;            /* AnnealedSinusoidalEncoder F (warping.py:245) */
  int nerf_trunk_depth, nerf_trunk_width;
  int nerf_rgb_branch_depth, nerf_rgb_branch_width;
  unsigned nerf_skips_mask;      /* bit i set <=> i in nerf_skips (modules.py:47) */
  int alpha_channels, rgb_channels;   /* must be 1 and 3                        */
  int warp_field_type;           /* nfb_warp_type; NONE when use_warp is False  */
  int warp_trunk_depth, warp_trunk_width;   /* SE3Field/TranslationField MLP    */
  unsigned warp_skips_mask;
  int num_warp_features, num_appearance_features, num_camera_features;
  int num_warp_embeddings, num_appearance_embeddings, num_camera_embeddings;
  int use_viewdirs, use_appearance_metadata, use_camera_metadata;
  int use_trunk_condition, use_alpha_condition, use_rgb_condition;
  int activation;                /* hidden activation of NerfMLP (nfb_activation) */
  int sigma_activation;          /* models.py:277                               */
  int use_white_background, use_linear_disparity, use_sample_at_infinity;
  float near_plane, far_plane;   /* NerfModel.near / .far                       */
  int precision;                 /* nfb_precision                               */
  /* warp-field variants (warping.py:84-123, 233-260, 242-243, 339-352) */
  int warp_metadata_encoder;     /* nfb_warp_encoder: glo | time | blend (TranslationField only) */
  int time_encoder_num_freqs;    /* warp_kwargs['metadata_encoder_num_freqs'] (TimeEncoder posenc) */
  int warp_use_pivot;            /* SE3Field(use_pivot=True): branches_p          */
  int warp_use_translation;      /* SE3Field(use_translation=True): branches_t    */
} nfb_config;

/* Flags for the render entry points. */
#define NFB_FLAG_COARSE_ONLY 1u  /* stop after the coarse level                 */
#define NFB_FLAG_NO_WARP     2u  /* use_warp=False call-time override (models.py:321) */
#define NFB_FLAG_METADATA_ENCODED 4u /* metadata_encoded=True (models.py:198-213,251;
                                      * warping.py:186-187): warp_id / app_id / cam_id are
                                      * reinterpreted as const float* per-ray embeddings of
                                      * shape (B, num_warp_features) / (B, num_appearance_features) /
                                      * (B, num_camera_features) and used instead of the GLO
                                      * table rows.  Device entry points only. */

/* Lifetime.  Replaces construct_nerf's model construction (models.py:424-463);
 * max_rays bounds B of every later call (workspace is sized once, here). */
int nfb_create(const nfb_config* cfg, int max_rays, nfb_handle** out);
void nfb_destroy(nfb_handle* h);

/* Parameter interface.  The expected tensors, in order, with their Flax names
 * ("warp_field/trunk/hidden_0/kernel", ... SURVEY.md §8a R12) and (rows, cols);
 * Dense kernels are (in, out), biases (1, out), embeddings (num, features). */
int nfb_param_count(const nfb_handle* h);
int nfb_param_info(const nfb_handle* h, int index, char* name, int name_capacity,
                   long long* rows, long long* cols);
/* Copies/repacks the fp32 tensors (device pointers, order of nfb_param_info)
 * into the library's padded layouts.  Replaces passing {'params': params} to
 * model.apply (models.py:289; eval.py:331). */
int nfb_set_params(nfb_handle* h, const float* const* tensors,
                   const long long* numels, int count, void* stream);

/* NerfModel.__call__ (nerfies/models.py:289-375): coarse level, hierarchical
 * resampling, fine level.
 *   origins, directions, viewdirs : (B,3); viewdirs NULL = directions (:326-329)
 *   warp_id, appearance_id, camera_id : (B) uint32 = metadata[...][:,0]; NULL
 *       allowed when the model does not use that metadata
 *   warp_alpha : warp_extra['alpha'] (model_utils.py:31-33)
 *   t_rand (B,Nc), u_rand (B,Nf) : the uniform draws of the stratified path
 *       (model_utils.py:65,162); NULL = deterministic path (:67-70, :164-165)
 *   out_coarse, out_fine : (B,6) = rgb[3], depth, med_depth, acc
 *   w_coarse (B,Nc), w_fine (B,Nc+Nf), z_fine (B,Nc+Nf) : optional outputs */
int nfb_render_forward(nfb_handle* h, int num_rays, const float* origins,
                       const float* directions, const float* viewdirs,
                       const unsigned* warp_id, const unsigned* appearance_id,
                       const unsigned* camera_id, float warp_alpha,
                       const float* t_rand, const float* u_rand, unsigned flags,
                       float* out_coarse, float* out_fine, float* w_coarse,
                       float* w_fine, float* z_fine, void* stream);

/* warp_extra['time_alpha'] (model_utils.py:31-33; modules.py:317-320) for the
 * TIME / BLEND warp metadata encoders; persists on the handle until changed
 * (default 0).  With NFB_WARP_ENC_TIME the `warp_id` argument of the render / warp
 * entry points is reinterpreted as const float* metadata['time'] (B). */
int nfb_set_time_alpha(nfb_handle* h, float time_alpha);

/* Same call with HOST buffers: stages inputs through pinned memory, H2D,
 * renders, D2H, synchronises.  This is what render_image's model_fn does per
 * chunk in the reference (evaluation.py:85-93: shard -> model_fn -> unshard). */
int nfb_render_forward_host(nfb_handle* h, int num_rays, const float* origins,
                            const float* directions, const float* viewdirs,
                            const unsigned* warp_id,
                            const unsigned* appearance_id,
                            const unsigned* camera_id, float warp_alpha,
                            unsigned flags, float* out_coarse, float* out_fine,
                            void* stream);

/* NerfModel.render_samples (nerfies/models.py:230-287) for one level
 * (0 = coarse MLP, 1 = fine MLP) on caller-supplied z_vals (B,S), points =
 * origins + z * directions.  out (B,6); optional weights (B,S), per-sample
 * sigmoid(rgb)/sigma (B,S,4) and warped_points (B,S,3). */
int nfb_render_samples(nfb_handle* h, int level, int num_rays, int num_samples,
                       const float* z_vals, const float* origins,
                       const float* directions, const float* viewdirs,
                       const unsigned* warp_id, const unsigned* appearance_id,
                       const unsigned* camera_id, float warp_alpha,
                       unsigned flags, float* out, float* weights,
                       float* samples, float* warped_points, void* stream);

/* model_utils.sample_pdf (nerfies/model_utils.py:190-215) with the caller prep
 * of models.py:353-357: bins = midpoints of z_coarse, weights = w_coarse[1:-1];
 * z_fine = sort(concat(z_coarse, inverse-CDF samples)). */
int nfb_sample_pdf(nfb_handle* h, int num_rays, const float* z_coarse,
                   const float* w_coarse, const float* u_rand, float* z_fine,
                   void* stream);

/* model_utils.sample_along_rays z_vals (nerfies/model_utils.py:56-70). */
int nfb_coarse_z_vals(nfb_handle* h, int num_rays, const float* t_rand,
                      float* z_coarse, void* stream);

/* warp_field.apply on free points (nerfies/warping.py:355-389, 160-199; called
 * by training.py:122-131): points (P,3), warp_id (P) -> warped (P,3). */
int nfb_warp_forward(nfb_handle* h, int num_points, const float* points,
                     const unsigned* warp_id, float warp_alpha, unsigned flags,
                     float* warped, void* stream);
/* flags: NFB_FLAG_METADATA_ENCODED = warp_field.apply(..., metadata_encoded=True)
 * (warping.py:186-187, 378): warp_id is (P, num_warp_features) float embeddings. */

/* ---- training tier (SURVEY §8(f) #1) ----------------------------------------------
 * jax.value_and_grad of the photometric loss of training.train_step
 * (training.py:171-175, 214-244, 263-264): loss = mean((rgb_coarse - target)^2) +
 * mean((rgb_fine - target)^2) over the batch, differentiated w.r.t. every model
 * parameter through NerfModel.__call__ (z_fine is a constant: lax.stop_gradient,
 * model_utils.py:211).  fp32, layer-wise with a tape in device memory, hand-written
 * SIMT GEMMs (csrc/train.cuh); uses the parameters of the last nfb_set_params.
 *   rgb_target (B,3); chunk_rays: rays per tape chunk (<= 0: 256);
 *   grads[i]: device tensor of the i-th parameter of nfb_param_info, rows*cols floats,
 *             ACCUMULATED into (+=): zero them first for a plain gradient;
 *   loss_out (device, 2 floats): the coarse and the fine loss.
 * Every warp metadata encoder: with NFB_WARP_ENC_TIME `warp_id` is const float* metadata['time'] (B), as
 * for nfb_render_forward, and the TimeEncoder is annealed by nfb_set_time_alpha; NFB_WARP_ENC_BLEND takes
 * uint32 ids and blends with that time_alpha (a constant of the step, never differentiated).  The
 * TimeEncoder's parameters receive their gradients like every other Dense layer.
 * NFB_FLAG_METADATA_ENCODED is not supported. */
int nfb_train_value_and_grad(nfb_handle* h, int num_rays, const float* origins,
                             const float* directions, const float* viewdirs,
                             const unsigned* warp_id, const unsigned* appearance_id,
                             const unsigned* camera_id, float warp_alpha,
                             const float* t_rand, const float* u_rand, unsigned flags,
                             const float* rgb_target, int chunk_rays, float* const* grads,
                             const long long* numels, int count, float* loss_out, void* stream);

/* Regularisers of training.train_step (training.py:138-147, 71-135, 176-212, 246-257). */
enum { NFB_ELASTIC_LOG_SVALS = 0, NFB_ELASTIC_SVALS = 1, NFB_ELASTIC_JTJ = 2, NFB_ELASTIC_DIV = 3,
       NFB_ELASTIC_DET = 4, NFB_ELASTIC_LOG_DET = 5 };
typedef struct nfb_train_reg {
  int use_elastic_loss;            /* training.py:143; applies to the coarse level (training.py:242-244) */
  int elastic_reduce_method;       /* 0 = 'median' (the median-depth sample of each ray), 1 = 'weight' */
  int elastic_loss_type;           /* NFB_ELASTIC_* = compute_elastic_loss's loss_type ('nr' unsupported) */
  float elastic_loss_weight;       /* ScalarParams.elastic_loss_weight */
  int use_warp_reg_loss;           /* training.py:147, both levels */
  float warp_reg_loss_weight, warp_reg_loss_alpha, warp_reg_loss_scale;
  int use_background_loss;         /* training.py:146 */
  int num_background_points;
  const float* background_points;        /* device (P,3): batch['background_points'] */
  const unsigned* background_warp_ids;   /* device (P): the reference draws random.choice(key, model.warp_ids);
                                            uint32 ids for every encoder (a TimeEncoder reads float(id)) */
  const float* background_noise;         /* device (P,3) or NULL: noise_std * random.normal(key, points.shape) */
  float background_loss_weight;          /* ScalarParams.background_loss_weight */
} nfb_train_reg;

/* nfb_train_value_and_grad plus the regularisers (reg may be NULL).  loss_out: 16 device floats
 *   [0] rgb loss coarse  [1] rgb loss fine  [2] loss/elastic  [3] residual/elastic
 *   [4] metric/jacobian_det  [5] metric/jacobian_div  [6] metric/jacobian_curl (means over the rows whose
 *   Jacobian the loss uses: the reference averages these three over every coarse sample, training.py:214-222)
 *   [7] loss/warp_reg coarse  [8] residual/warp_reg coarse  [9] loss/warp_reg fine  [10] residual fine
 *   [11] background loss (unweighted mean)  [12] mean |warped - x| of the background points.
 * The gradient is that of  rgb_coarse + rgb_fine + elastic_loss_weight * [2] + warp_reg_loss_weight *
 * ([7] + [9]) + background_loss_weight * [11]  (training.py:176-212, 228-259).  Replaces
 * jax.value_and_grad(_loss_fn) (training.py:263-264) with every regulariser of train_step. */
int nfb_train_value_and_grad_reg(nfb_handle* h, int B, const float* origins, const float* directions,
                                 const float* viewdirs, const unsigned* warp_id, const unsigned* app_id,
                                 const unsigned* cam_id, float warp_alpha, const float* t_rand,
                                 const float* u_rand, unsigned flags, const float* rgb_target,
                                 int chunk_rays, const nfb_train_reg* reg, float* const* grads,
                                 const long long* numels, int count, float* loss_out, void* stream);

/* Vector-Jacobian product of one nfb_render_forward call with respect to the parameters: what jax.vjp of
 * NerfModel.__call__ gives for any loss on its outputs (training.py:228-264 is one such loss).
 *   origins ... flags: the forward call's arguments (NFB_FLAG_NO_WARP, NFB_FLAG_COARSE_ONLY and
 *     NFB_FLAG_METADATA_ENCODED as there; with the last, warp_id / appearance_id / camera_id are the (B, G|A|C)
 *     float codes);
 *   z_coarse (B,Nc), z_fine (B,Nc+Nf): the z values the forward used (nfb_coarse_z_vals of its t_rand and the
 *     z_fine output of nfb_render_forward / nfb_sample_pdf).  They are constants (lax.stop_gradient,
 *     model_utils.py:211): nothing is resampled;
 *   cotangents, each nullable (a null one is zero; a level with none is skipped):
 *     d_out_coarse / d_out_fine (B,6) in the forward's out layout (rgb, depth, med_depth, acc; med_depth is
 *     piecewise constant and its column is ignored), d_weights_coarse (B,Nc) / d_weights_fine (B,Nc+Nf),
 *     d_warped_coarse (B,Nc,3) / d_warped_fine (B,Nc+Nf,3) of the warped sample points;
 *   d_warp_code (B,G), d_app_code (B,A), d_cam_code (B,C): with NFB_FLAG_METADATA_ENCODED, nullable, the
 *     gradients of the codes (+=);
 *   chunk_rays, grads, numels, count: as nfb_train_value_and_grad (grads ACCUMULATED into, +=).
 * Per chunk of rays and level, the taped forward of nfb_train_value_and_grad is recomputed at the given z and
 * walked backwards, seeded from the cotangents; it runs in the handle's training precision
 * (nfb_set_train_precision) whatever nfb_config.precision is.  Uses the parameters of the last nfb_set_params
 * and the time_alpha of the last nfb_set_time_alpha. */
int nfb_render_vjp(nfb_handle* h, int num_rays, const float* origins, const float* directions,
                   const float* viewdirs, const unsigned* warp_id, const unsigned* appearance_id,
                   const unsigned* camera_id, float warp_alpha, unsigned flags, const float* z_coarse,
                   const float* z_fine, const float* d_out_coarse, const float* d_out_fine,
                   const float* d_weights_coarse, const float* d_weights_fine, const float* d_warped_coarse,
                   const float* d_warped_fine, float* d_warp_code, float* d_app_code, float* d_cam_code,
                   int chunk_rays, float* const* grads, const long long* numels, int count, void* stream);

/* The same for nfb_warp_forward (warp_field.apply on free points): d_warped (P,3) -> the warp field's parameter
 * gradients (+= into grads, laid out as nfb_train_value_and_grad's) and, with NFB_FLAG_METADATA_ENCODED,
 * d_code (P, num_warp_features), nullable (+=).  Training precision, chunks of max_rays points. */
int nfb_warp_vjp(nfb_handle* h, int num_points, const float* points, const unsigned* warp_id, float warp_alpha,
                 unsigned flags, const float* d_warped, float* d_code, float* const* grads,
                 const long long* numels, int count, void* stream);

/* Jacobian of the warp field at free points: jacobian_out (P,3,3), J[i][j] = d warped_i / d point_j
 * (jax.jacfwd(self.warp, argnums=0), warping.py:196-198, 385-387); warped_out (P,3) nullable.
 * warp_id (P) GLO ids, or with NFB_WARP_ENC_TIME const float* timestamps (P); the metadata embedding is a
 * constant of the Jacobian.  fp32, any precision mode of the handle (layer-wise tape kernels). */
int nfb_warp_jacobian(nfb_handle* h, int P, const float* points, const unsigned* warp_id, float warp_alpha,
                      float* warped_out, float* jacobian_out, void* stream);

/* Per-point outcome of nfb_warp_invert. */
enum { NFB_INVERT_CONVERGED = 0,   /* |W(x) - target| <= tol                                         */
       NFB_INVERT_MAX_ITERS = 1,   /* still improving when the iterations ran out                     */
       NFB_INVERT_SINGULAR = 2,    /* J at the best iterate is singular or not finite                 */
       NFB_INVERT_STALLED = 3,     /* no step down to 2^-10 of the Newton step lowered the residual   */
       NFB_INVERT_NONFINITE = 4 }; /* W at the starting point is not finite                           */

/* Solve W(x) = target for x at free points, where W is the warp field of the frame that warp_id names
 * (nfb_warp_jacobian's W, ids or NFB_WARP_ENC_TIME timestamps; encoded metadata is not supported).
 *   targets (P,3): template points; init (P,3) nullable: starting points (NULL: the targets);
 *   max_iters in [1, 64]; tol > 0 (absolute, in scene units);
 *   points_out (P,3): the best iterate; residual_out (P): |W(points_out) - target|_2;
 *   jacobian_out (P,3,3) nullable: J at points_out; status_out (P) nullable int32 (NFB_INVERT_*).
 * Damped Newton: each of the max_iters iterations evaluates W and J at every point's candidate (the
 * tape kernels of nfb_warp_jacobian) and then, per point in fp64, accepts a candidate whose residual is
 * finite and below the best so far and takes the full Newton step from it (3x3 LU, partial pivoting), or
 * halves the step from the best iterate.  Converged, singular, stalled and non-finite points are frozen.
 * A fixed iteration count and no atomics: the call never synchronises with the host, and a point's
 * results do not depend on the other points.  Chunks of max_rays points; the handle's training precision
 * (fp32 or tf32x3), whatever nfb_config.precision is. */
int nfb_warp_invert(nfb_handle* h, int P, const float* targets, const float* init, const unsigned* warp_id,
                    float warp_alpha, int max_iters, float tol, float* points_out, float* residual_out,
                    float* jacobian_out, int* status_out, void* stream);

/* flax.optim.Adam.apply_gradient (training.py:268; beta1 0.9, beta2 0.999, eps 1e-8, no
 * weight decay are the Flax defaults the reference uses, train.py:219) on flat device
 * vectors of n floats; `step` counts from 1 (bias correction 1 - beta^step).  No handle. */
int nfb_adam_step(float* params, const float* grads, float* m, float* v, long long n,
                  float learning_rate, float beta1, float beta2, float eps, long long step,
                  void* stream);

/* Measurement aid (bench.py's roofline): when enabled, every launch of the field
 * kernel (the dominant kernel) is bracketed by cudaEvents on its launch stream.
 * nfb_field_time_ms synchronises on the events of the most recent launch of
 * `level` (0 coarse, 1 fine) and returns its duration in ms (< 0 on error). */
int nfb_set_profiling(nfb_handle* h, int enabled);
float nfb_field_time_ms(nfb_handle* h, int level);

/* ---- camera -> rays (SURVEY §8(f) row 3) ------------------------------------
 * Mirrors the fields of nerfies.camera.Camera (camera.py:110-137). */
typedef struct nfb_camera {
  float orientation[9];           /* world-to-camera rotation, row-major        */
  float position[3];
  float focal_length;
  float principal_point[2];
  float skew;
  float pixel_aspect_ratio;
  float radial_distortion[3];     /* k1 k2 k3                                   */
  float tangential_distortion[2]; /* p1 p2                                      */
  int image_size[2];              /* (width, height)                            */
} nfb_camera;

/* Replaces datasets/core.py:50-75 camera_to_rays (camera.py:317-321 pixel centres
 * + camera.py:244-269 pixels_to_rays) for the pixels [first_pixel,
 * first_pixel + count) of the frame in row-major order: origins (count,3) =
 * camera position, directions (count,3) unit, pixels (count,2) centres.
 * origins and pixels may be NULL.  Needs no handle. */
int nfb_camera_rays(const nfb_camera* cam, long long first_pixel, long long count,
                    float* origins, float* directions, float* pixels, void* stream);

/* Replaces Camera.pixels_to_rays (camera.py:244-269) for arbitrary float32 pixel
 * positions (n,2) -> unit world-space directions (n,3). */
int nfb_pixels_to_rays(const nfb_camera* cam, const float* pixels, long long n,
                       float* directions, void* stream);

/* ---- preloaded capture -> ray batches (datasets/core.py:392-447) -------------
 * A capture of num_images items, their pixels concatenated image after image in
 * row-major order: ray r of image k is pixel r - pixel_offsets[k] of that image.
 * Every pointer is a device pointer.  pixel_offsets[0] == 0 and
 * pixel_offsets[num_images] == num_rays == the sum of the images' w * h. */
typedef struct nfb_ray_table {
  int num_images;
  const nfb_camera* cameras;         /* (num_images)                                */
  const long long* pixel_offsets;    /* (num_images + 1)                            */
  const unsigned char* rgb;          /* (num_rays, 3) uint8 RGB; nullable           */
  const int* appearance;             /* (num_images) metadata indices; nullable     */
  const int* camera;
  const int* warp;
  const float* time;                 /* (num_images); nullable                      */
  const void* order;                 /* (num_rays) permutation; NULL = identity     */
  int order_is_64;                   /* order is int64 (else int32)                 */
  long long num_rays;
} nfb_ray_table;

/* Output i (0 <= i < count) is ray r = order[(first + i) mod num_rays] of the table:
 * origins (count,3) = its camera position, directions (count,3) unit (as
 * nfb_camera_rays), pixels (count,2) centres, rgb (count,3) = u8 / 255.f, and the
 * image's appearance / camera / warp (count) int32 and time (count) float32.
 * Every output is nullable; an output whose source is NULL in the table is an
 * error.  Needs no handle, allocates nothing, is ordered on `stream`; the outputs
 * do not depend on the launch (no atomics). */
int nfb_gather_rays(const nfb_ray_table* table, long long first, long long count,
                    float* origins, float* directions, float* pixels, float* rgb,
                    int* appearance, int* camera, int* warp, float* time, void* stream);

/* ---- per-frame image metrics of eval.py:process_batch ------------------------
 * Images are (num_images, height, width, channels) float32, channels interleaved (what
 * render_frame returns for 'rgb'), channels in 1..4, height and width >= 161 (MS-SSIM's five
 * scales must each be at least 11x11).  No handle; the caller provides the workspace.
 *
 * Bytes of device workspace nfb_image_metrics needs for this shape (< 0: invalid shape). */
long long nfb_image_metrics_workspace_size(int num_images, int height, int width, int channels);

/* eval.py:process_batch metrics (eval.py:58-62, 120-122, 140) for num_images (h, w, c) images:
 *   ms_ssim (N)   = tf.image.ssim_multiscale(target, image, max_val=1) with TF's defaults (power
 *                   factors 0.0448 0.2856 0.3001 0.2363 0.1333, 11x11 Gaussian of sigma 1.5,
 *                   k1 0.01, k2 0.03);
 *   mse (N)       = mean((image - target)^2);
 *   depth_abs (N) = nanmean(|depth_target - depth|) over (h, w) per image (depth, depth_target
 *                   (N, h, w), nullable together; NaN when every difference is NaN).
 * Output pointers are device pointers and nullable.  workspace: device, 256-byte aligned, at least
 * nfb_image_metrics_workspace_size bytes.  Sums are taken in a fixed order in fp64: two calls on
 * the same input give bit-identical results. */
int nfb_image_metrics(int num_images, int height, int width, int channels,
                      const float* image, const float* target,
                      const float* depth, const float* depth_target,
                      void* workspace, long long workspace_bytes,
                      float* ms_ssim, float* mse, float* depth_abs, void* stream);

/* Float frames -> 8- or 16-bit images, value for value what numpy computes in
 * image_utils.image_to_uint8 / image_to_uint16 (image_utils.py:114-131) and save_depth
 * (image_utils.py:172-174):
 *   dst[i] = (uintN) clip(src[i] / scale * max, 0, max),   max = 255 (bits 8) | 65535 (bits 16).
 * The division and the product are each one IEEE float32 operation, the cast truncates toward
 * zero (0.999 * 255 -> 254).  Negatives and -inf give 0, values above 1 and +inf give max, and
 * NaN gives 0: numpy's clip passes NaN and the x86-64 float -> unsigned cast of it is 0.
 * scale = 1 is image_to_uintN; scale = 1000, bits = 16 is save_depth.  scale must be positive and
 * finite.  src (n) float32 and dst (n) uint8 / uint16 are device pointers of their natural
 * alignment; 16-byte aligned pointers take 16-byte loads and stores.  One pass, no workspace, no
 * handle, ordered on `stream`. */
int nfb_image_quantize(const float* src, long long n, int bits, float scale, void* dst, void* stream);

/* Colour maps: visualization.colorize (visualization.py:177-219) on the device, value for value
 * what numpy 2 computes, as float64 (height, width, 3) or, through image_utils.image_to_uint8
 * (image_utils.py:114-121), as uint8.  The value of pixel p comes from `source`:
 *   NFB_VIZ_VALUE       a[p]                                    (a: height * width float32)
 *   NFB_VIZ_RECIPROCAL  1 / a[p], IEEE                           (disparity, eval.py:94-95)
 *   NFB_VIZ_ABS_ERROR   (|a0 - b0| + |a1 - b1|) + |a2 - b2|      (a, b: (height, width, 3),
 *   NFB_VIZ_SQ_ERROR    the same with squares                     eval.py:129-132)
 *   NFB_VIZ_RGB         not a colour map: a is an (height, width, 3) image written as uint8 with a
 *                       float64 product, trunc(clip((double) a * 255, 0, 255)) (uint8 output only)
 * Scale: x = (v - cmin) / d in float32 with cmin rounded to float32.  Without the frame flags,
 * `d` is the divisor float32(max(cmax - cmin, eps)) computed by the caller (its subtraction is fp64
 * when the bounds are Python floats) and cmax is unused.  With NFB_VIZ_FRAME_MIN / _MAX the bound is
 * the frame's min / max of the source (NaN if the frame holds a NaN, as np.min), found by a first
 * launch into `workspace` (NFB_VIZ_WORKSPACE_BYTES, 4-byte aligned), and `d` must be float32(eps):
 * the divisor is then max(cmax - cmin, eps) in float32.  NFB_VIZ_INVERT maps 1 - x.  Then
 * t = 255 * y, a = floor(t), b = min(a + 1, 255), colour = table[a] + (table[b] - table[a]) * (t - a)
 * in float64; x > 1 gives 1.0 (0.0 inverted), x < 0 gives 0.0 (1.0 inverted), NaN a NaN colour
 * (0 as uint8).  `table`: device (256, 3) float64, row-major.
 * Output: out_f64 (height * width * 3, contiguous) or out_u8, exactly one of them.  Row r of out_u8
 * starts at out_u8 + r * pitch bytes (pitch >= 3 * width; pass the column offset in the pointer).
 * At most two launches, no allocation, no host synchronisation, ordered on `stream`. */
#define NFB_VIZ_VALUE      0
#define NFB_VIZ_RECIPROCAL 1
#define NFB_VIZ_ABS_ERROR  2
#define NFB_VIZ_SQ_ERROR   3
#define NFB_VIZ_RGB        4
#define NFB_VIZ_INVERT     1
#define NFB_VIZ_FRAME_MIN  2
#define NFB_VIZ_FRAME_MAX  4
#define NFB_VIZ_WORKSPACE_BYTES 2048
int nfb_colorize(const float* a, const float* b, int height, int width, int source, const double* table,
                 float cmin, float cmax, float d, int flags, void* workspace, double* out_f64,
                 unsigned char* out_u8, long long pitch, void* stream);

/* ---- capture processing (notebooks/Nerfies_Capture_Processing.ipynb) ----------------------
 * No handle, no allocation, ordered on `stream`.
 *
 * Image pyramid of one uint8 RGB frame (the notebook's "Resize images into different scales"):
 * src is (height, width, 3) with rows `src_pitch` bytes apart, already cropped to a multiple of the
 * largest scale (make_divisible: pass the crop's height and width with the full frame's pitch).
 * Level l is dst[l] (height / scales[l], width / scales[l], 3), contiguous: scale 1 copies the
 * frame; an even scale s gives each output pixel (a + b + c + d + 2) >> 2 over the 2x2 source block
 * at offsets s/2 - 1 and s/2, byte for byte what cv2.resize(image, (w, h)) with its default
 * INTER_LINEAR writes.  Every scale must divide the largest; at most 8 levels.  `scales` and `dst`
 * are host arrays (the pointers in dst are device pointers).  One launch; the frame is read once. */
int nfb_frame_pyramid(const unsigned char* src, int height, int width, long long src_pitch, int num_levels,
                      const int* scales, unsigned char* const* dst, void* stream);

/* Blur scores of num_frames (height, width, 3) uint8 RGB frames, contiguous: per frame,
 * cv2.Laplacian(cv2.cvtColor(rgb, COLOR_RGB2GRAY), CV_64F).var() into scores (num_frames) float64.
 * The Laplacian's integer sum and sum of squares are exact (int64), the variance one fp64 division
 * of an exact 128-bit numerator.  workspace: device, 8-byte aligned, at least
 * nfb_blur_scores_workspace_size bytes.  Two launches and one memset. */
long long nfb_blur_scores_workspace_size(int num_frames);
int nfb_blur_scores(const unsigned char* frames, int num_frames, int height, int width, void* workspace,
                    long long workspace_bytes, double* scores, void* stream);

/* Camera.project (camera.py:283-315) of float32 points (n, 3) -> pixels (n, 2), in float32
 * arithmetic operation for operation as numpy evaluates it.  `cam` is a host struct. */
int nfb_camera_project(const nfb_camera* cam, const float* points, long long n, float* pixels, void* stream);

/* Per-camera near/far planes of the notebook's estimate_near_far_for_image: for camera c, the
 * float64 points (num_points, 3) are projected in fp64 (the camera's float32 fields widened, as numpy
 * promotes them); those with 0 <= px <= width, 0 <= py <= height and depth > 0 are kept, and
 *   near[c] = np.quantile(depths, q_near), far[c] = np.quantile(depths, q_far)   ('linear' rule)
 * counts[c] = the number kept; near and far are NaN where it is 0.  `cameras` is a DEVICE array of
 * num_cameras structs.  The quantiles come from exact order statistics (radix select over the depths'
 * bit patterns), so no depth array is formed: the workspace (device, 256-byte aligned, at least
 * nfb_near_far_workspace_size bytes) grows with the cameras only.  17 launches and one memset; no
 * host synchronisation. */
long long nfb_near_far_workspace_size(int num_cameras);
int nfb_near_far(const nfb_camera* cameras, int num_cameras, const double* points, long long num_points,
                 double q_near, double q_far, void* workspace, long long workspace_bytes, double* near,
                 double* far, long long* counts, void* stream);

/* ---- surface extraction: marching cubes (no reference analogue) -----------------------------
 * grid: (nz, ny, nx) float32, C-contiguous, x fastest; value [k][j][i] lies at
 * origin + (i, j, k) * spacing.  Every side lies in [2, 1024].  No handle, ordered on `stream`.
 *   - a point is inside iff value > level, so NaN is outside (the mesh stays closed around
 *     non-finite cells) and value == level is outside;
 *   - one vertex per grid edge whose endpoints lie on different sides, shared by the cubes around the
 *     edge: the mesh is indexed and watertight.  Vertices are ordered by (edge axis, linear index of
 *     the edge's lower endpoint); faces by cube (linear index of its lowest corner), then table order;
 *   - vertex on the edge p0 -> p1 (values v0, v1; p1 one step along the edge's axis), in float32,
 *     each operation rounded once, no fused multiply-add:
 *       t = (level - v0) / (v1 - v0)                      (t = 0.5 when v0 or v1 is NaN)
 *       x0 = origin + float(index) * spacing, x1 = origin + float(index + 1) * spacing
 *       x  = x0 + t * (x1 - x0) along the edge's axis, x0 across it;
 *   - normal: the central-difference gradient of the grid over the spacing (one-sided on the border)
 *     at both endpoints, interpolated with the same t, normalised and negated (it points toward lower
 *     values, out of the surface).  A zero or non-finite gradient gives a zero normal;
 *   - triangles are counter-clockwise seen from outside (from lower values): the signed volume of a
 *     closed surface around a dense region is positive;
 *   - the mesh is open where the surface leaves the grid; it is not capped.
 * Two calls on the same grid write bitwise-equal meshes (no atomics).
 *
 * Bytes of device workspace for this grid (< 0: invalid size, or no device): 16 bytes per grid point
 * (a 32-bit vertex id per edge, a 32-bit face offset per cube) plus CUB's scan scratch. */
long long nfb_marching_cubes_workspace_size(int nx, int ny, int nz);
/* Classifies the grid into the workspace (device, 256-byte aligned, at least
 * nfb_marching_cubes_workspace_size bytes) and writes counts_out (device, 4 int64): the number of
 * vertices, the number of faces, and the ids of the first vertex on a y-edge and on a z-edge (vertices
 * before the first are on x-edges).  Asynchronous: two kernels and three CUB passes, no host
 * synchronisation. */
int nfb_marching_cubes_count(const float* grid, int nx, int ny, int nz, float level, void* workspace,
                             long long workspace_bytes, long long* counts_out, void* stream);
/* Writes the mesh the preceding nfb_marching_cubes_count call on the same grid, level and workspace
 * counted: vertices (V, 3) float32, normals (V, 3) float32 (nullable) and faces (F, 3) int32 vertex
 * indices.  origin and spacing are HOST arrays of 3 floats.  It first reads the two totals back (one
 * small copy and a stream synchronisation) and fails when either exceeds INT32_MAX. */
int nfb_marching_cubes(const float* grid, int nx, int ny, int nz, float level, const float* origin,
                       const float* spacing, void* workspace, long long workspace_bytes, float* vertices,
                       float* normals, int* faces, void* stream);
/* The case table, host only (needs no device).  Corner c of a cube sits at offset
 * (c & 1, c >> 1 & 1, c >> 2 & 1); edge e = 4 * axis + u + 2 v runs along `axis` from the corner whose
 * coordinates along the other two axes, the lower axis first, are (u, v).  Case bits: bit c set iff
 * corner c is inside.  Returns the largest triangle count of any case (M) and, when out is not NULL,
 * writes 256 rows of 1 + 3 M ints: the case's triangle count, then its triangles' edges (-1 padded). */
int nfb_marching_cubes_table(int* out);

/* Test hook for the abort path described in the conventions above: while enabled,
 * the weight producer of the tensor-core kernel first waits on an mbarrier that never
 * completes, so the launch must time out, drain and raise the abort flag
 * (tests/test_edge_cases_gpu.py).  The process cannot run further tensor-core
 * launches afterwards.  No reference analogue. */
int nfb_debug_provoke_timeout(nfb_handle* h, int enabled);

/* Test hook: while enabled, the tensor-core warp pass runs in 128-row tiles even where the warp
 * MLP (no layer wider than 128) fits the 256-row tiles it otherwise uses, so that tests can compare
 * the two bit for bit.  No reference analogue. */
int nfb_debug_one_row_block(nfb_handle* h, int enabled);

/* The asynchronous entry points (nfb_render_forward, nfb_render_samples, nfb_warp_forward, ...) return
 * before their kernels finish, so a tensor-core kernel's protocol time-out (see the conventions above)
 * is only seen by a LATER call.  nfb_check_abort reports it for the work already submitted: with
 * synchronize != 0 it first waits for `stream`; returns 0 or < 0 (nfb_last_error).  nfb_reset_abort
 * waits for the device and clears the process-wide flag, after which launches are accepted again.
 * No reference analogue. */
int nfb_check_abort(void* stream, int synchronize);
int nfb_reset_abort(void);

/* Hardware self-test of the wgmma building blocks (GMMA descriptors, 128-byte
 * swizzle, accumulator fragment layout): C[128,N] = bf16(A[128,K]) x bf16(W[K,N]),
 * fp32 accumulate.  K <= 320, N <= 256; device pointers. */
int nfb_selftest_gemm(int K, int N, const float* A, const float* W, float* C,
                      void* stream);

/* The fp16x3 form of the same: C (128 x N) = A (128 x K) W (K x N) as three fp16
 * chains (A_hi W_hi + A_lo W_hi + A_hi W_lo, fp32 accumulate), as the fp16x3 field
 * kernel evaluates a layer.  K <= 320, N <= 256; `reps` repeats the chains (the
 * result is divided by reps).  out (host, 2 x int64, nullable): cycles of the MMA
 * phase, number of MMAs per 64 x 16 output block and repetition.  Hardware
 * self-test; no reference analogue. */
int nfb_selftest_gemm3(int K, int N, const float* A, const float* W, float* C, int reps,
                       long long* out, void* stream);

/* Self-test of the training tier's GEMM: one Dense layer's GEMM through the same launch and
 * element functors nfb_train_value_and_grad uses.  The layer maps [X | IN] (rows x (k_x + k_in);
 * X: rows x k_x, ld ldx; IN: rows x k_in, ld ldin) to n outputs; W (k_x + k_in, ldw), bias (n),
 * Y and dY (rows, ldw), act an activation of nfb_config.  X may be NULL when k_x == 0, IN when k_in == 0.
 *   NFB_SGEMM_FORWARD: y = act([X | IN] W + bias), written to columns [0, n) of y.
 *   NFB_SGEMM_DX:      dZ = dY * act'(Y) (Y read from y);  dx += dZ W^T[:, :k_x] (rows, ldx),
 *                      din += dZ W^T[:, k_x:] (rows, ldin).
 *   NFB_SGEMM_DW:      dw (k_x + k_in, ldw) += [X | IN]^T dZ, the reduction over the rows split into slices
 *                      of k_split rows (0: the split the training step picks for this shape), partial sums
 *                      atomically added.
 * k_split must be 0 for the other modes.  k_split_used (host, nullable) receives the rows per slice.
 * Device pointers; allocates nothing; asynchronous on `stream`.  No reference analogue. */
enum { NFB_SGEMM_FORWARD = 0, NFB_SGEMM_DX = 1, NFB_SGEMM_DW = 2 };
int nfb_selftest_sgemm(int mode, long long rows, int n, int k_x, int k_in, int act,
                       const float* x, int ldx, const float* in, int ldin, const float* w, int ldw,
                       const float* bias, float* y, const float* dy, float* dx, float* din, float* dw,
                       long long k_split, long long* k_split_used, void* stream);

/* Training precision of a handle: the kernel of every GEMM of nfb_train_value_and_grad(_reg) and
 * nfb_warp_jacobian (Dense layer forward, dX and dW; the tangent rows of the warp Jacobian).
 *   NFB_TRAIN_FP32   (default): fp32 CUDA-core GEMMs.
 *   NFB_TRAIN_TF32X3: tensor-core GEMMs with every operand split into two tf32 parts, three wgmma
 *                     chains (A_small B_big, A_big B_small, A_big B_big) per k-block of 32 into an
 *                     fp32 partial, the partials summed in fp32: about 3 x 2^-22 relative per product
 *                     beside fp32's accumulation error.
 * Independent of nfb_config.precision (the render kernels).  Any other value fails (nfb_last_error)
 * and leaves the handle's precision as it was.  No reference analogue. */
enum { NFB_TRAIN_FP32 = 0, NFB_TRAIN_TF32X3 = 1 };
int nfb_set_train_precision(nfb_handle* h, int train_precision);

/* nfb_selftest_sgemm in a given training precision (NFB_TRAIN_*): the same arguments, launch and
 * functors; k_split = 0 picks the split that precision's training step uses. */
int nfb_selftest_train_gemm(int train_precision, int mode, long long rows, int n, int k_x, int k_in, int act,
                            const float* x, int ldx, const float* in, int ldin, const float* w, int ldw,
                            const float* bias, float* y, const float* dy, float* dx, float* din, float* dw,
                            long long k_split, long long* k_split_used, void* stream);

/* Number of CUDA kernels this handle has launched so far (bench accounting). */
long long nfb_kernel_launches(const nfb_handle* h);
/* Thread-local description of the last error returned on this thread. */
const char* nfb_last_error(void);
/* "nerfies_b200 <version> sm_90a" */
const char* nfb_version(void);

#ifdef __cplusplus
}
#endif
#endif  /* NERFIES_B200_H_ */
