/*
 * pmvs_b200.h -- C ABI of libpmvs_b200.so, the sm_90a implementation of the
 * PointMVSNet PointFlow hot path (reference: callmeray/PointMVSNet @ cacb2d7).
 *
 * Conventions (all entry points):
 *   - every pointer is a DEVICE pointer owned by the caller, contiguous in the layout
 *     stated, fp32 unless stated; nothing is allocated, freed or synchronised inside;
 *   - `stream` is the CUDA stream to enqueue on (cudaStream_t passed as void*);
 *     the reference launched on the legacy default stream
 *     (functions/csrc/gather_knn_kernel.cu:138) -- that latent bug is not reproduced;
 *   - return value 0 = success, non-zero = error (PMVS_ERR_*); the message is
 *     available from pmvs_last_error() (thread-local).  The Python shim raises
 *     RuntimeError, matching the reference's c10-error -> RuntimeError convention
 *     (gather_knn_kernel.cu:10-12,34-39);
 *   - re-entrant per device; no global mutable state except the launch counter.
 *
 * The reference's native boundary for this path is the pybind module `dgcnn_ext`
 * (functions/csrc/main.cpp:3-6, gather_knn.h:7-13).  Everything else on the hot path
 * is stock PyTorch in the reference (F.grid_sample, F.conv3d + topk, nn.Conv1d,
 * nn.BatchNorm), so each entry point below cites the Python call site it replaces.
 */
#ifndef PMVS_B200_H_
#define PMVS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PMVS_OK 0
#define PMVS_ERR_ARG 1      /* bad shape / unsupported size / NULL pointer */
#define PMVS_ERR_CUDA 2     /* a CUDA runtime call or launch failed */
#define PMVS_ERR_WORKSPACE 3 /* workspace too small */

#define PMVS_NUM_HYP 5      /* model.py:172 interval_list = [-2,-1,0,1,2] */
#define PMVS_FEAT_CH 136    /* 16 + 32 + 64 variance channels + 8 x xyz (model.py:193-197) */
#define PMVS_KNN 16         /* model.py:20,23 */
#define PMVS_MAX_VIEWS 12

typedef void* pmvs_stream_t; /* cudaStream_t */

/* ---- library info ---------------------------------------------------------------- */
int pmvs_version(void);
const char* pmvs_last_error(void);
/* number of kernels this library has launched since load (all threads, all devices) */
unsigned long long pmvs_launch_count(void);

/* Arithmetic of the per-point contractions (1x1 convolutions): 3 = wgmma tf32 with
 * error-compensated 3xTF32 (default, fp32-level accuracy), 1 = plain TF32 tensor cores,
 * 0 = fp32 SIMT FMA kernel.  Process-wide; not thread-safe against concurrent launches. */
int pmvs_set_gemm_mode(int mode);
int pmvs_get_gemm_mode(void);

/* Implementation switches of the fused path (process-wide, like the GEMM mode; for A/B measurements
 * and bisecting - every setting computes the same results; the first value listed is the default):
 *   PMVS_OPT_EDGE   EdgeConv statistics/apply: 1 = TMA halo tile (8x4 pixels x 5 layers) in shared memory,
 *                   0 = 16 L2 gathers per point (the kernels the stand-alone EdgeConv operator uses)
 *   PMVS_OPT_KNN    1 = batched sorting network + bitonic merge (kernel_size 5, knn 16),
 *                   0 = sorted insertion (the kernel every other (kernel_size, knn) uses)
 *   PMVS_OPT_FETCH  3 = option 1 fused with EdgeConvNoC(136, 32)'s contraction (one persistent launch, the
 *                   136-channel point features are not written); taken under PMVS_OPT_GEMM 3, gemm mode 3,
 *                   PMVS_OPT_EDGE != 0 and V <= 6, option 1 + the contraction otherwise (PMVS_OPT_GEMM_STRICT:
 *                   an error instead),
 *                   1 = consecutive hypotheses share the texel quad, fp32 pair math (3 CTAs / SM),
 *                   2 = the same with 2 CTAs / SM and a larger register budget, 0 = 4 taps per (hypothesis, view)
 *                   (the kernel used for V > 6)
 *   PMVS_OPT_GEMM   3 = weights stationary in shared memory, persistent, X through TMA rings (one per
 *                   consumer warpgroup, 4-16 stages of 8 KB), A fragments in registers, two ping-pong consumer
 *                   warpgroups (option 2 when the tensor map cannot be encoded), 2 = the same weights with a cp.async staging ring (2-3
 *                   chunks in flight), 1 = option 2 with register prefetch,
 *                   0 = points-as-M with shared-memory operands (the kernel plain-TF32 mode uses)
 *   PMVS_OPT_DEBUG_IDX  1 = also materialise int32 neighbour indices in the workspace
 *   PMVS_OPT_GEMM_STRICT  0 = off; 1 = under PMVS_OPT_GEMM 3, a contraction the TMA kernel does not take
 *                   returns PMVS_ERR_ARG instead of running on option 2, and so does a PMVS_OPT_FETCH 3 call
 *                   that the fused fetch kernel does not take (tests) */
#define PMVS_OPT_EDGE 1
#define PMVS_OPT_KNN 2
#define PMVS_OPT_FETCH 3
#define PMVS_OPT_GEMM 4
#define PMVS_OPT_DEBUG_IDX 5
#define PMVS_OPT_GEMM_STRICT 6
int pmvs_set_option(int key, int value);
int pmvs_get_option(int key);

/* Per-launch CUDA-event timing for bench.py's roofline: while enabled every kernel launch of
 * this library is bracketed by two events on its stream (do not enable during graph capture).
 * pmvs_profile_collect synchronises, writes '\n'-separated kernel names and durations (ms)
 * for up to max_records launches in launch order, clears the log, returns the count. */
int pmvs_profile_enable(int on);
int pmvs_profile_collect(char* names, size_t names_bytes, float* ms, int max_records);

/* ---- a13: gather_knn  (dgcnn_ext.gather_knn_forward/backward, main.cpp:4-5;
 *      GatherKNNForward gather_knn_kernel.cu:25-47, GatherKNNBackward :97-148) -------- */
/* out[b,c,n,k] = in[b,c,idx[b,n,k]];  in [B,C,N], idx [B,N,K] int64, out [B,C,N,K] */
int pmvs_gather_knn_forward(const float* input, const int64_t* index, float* output,
                            int B, int C, int N, int K, pmvs_stream_t stream);
/* grad_in[b,c,idx[b,n,k]] += grad_out[b,c,n,k]; grad_in [B,C,N] is zeroed inside. */
int pmvs_gather_knn_backward(const float* grad_output, const int64_t* index, float* grad_input,
                             int B, int C, int N, int K, pmvs_stream_t stream);
/* The same sums with a FIXED summation order (SURVEY.md 8 row f3): grad_in[b,c,j] adds its contributions
 * sequentially in ascending source position n*K + k, so the result is bit-reproducible (the reference's atomicAdd
 * scatter, gather_knn_kernel.cu:50-89, is not) and equals the CPU loop `for p: grad_in[idx[p]] += grad_out[p]`.
 * Any index tensor; out-of-range entries are skipped.  workspace: pmvs_gather_knn_backward_det_workspace_bytes(B, N, K)
 * bytes, 256-byte aligned, device memory. */
size_t pmvs_gather_knn_backward_det_workspace_bytes(int B, int N, int K);
int pmvs_gather_knn_backward_det(const float* grad_output, const int64_t* index, float* grad_input,
                                 int B, int C, int N, int K, void* workspace, size_t workspace_bytes,
                                 pmvs_stream_t stream);

/* ---- a10: get_knn_3d  (utils/torch_utils.py:16-61) ------------------------------- */
/* xyz [B,3,D,H,W] -> idx [B, D*H*W, knn]; exactly one of idx64 / idx32 may be NULL.
 * Window ksize^3 (ksize 3 or 5), zero padding, candidate order d*k*k+h*k+w, ties broken
 * by candidate id, linear index n + dd*H*W + dh*W + dw clamped to [0, D*H*W-1]
 * (torch_utils.py:44,49-59).  knn in {4,8,16,20,32}. */
int pmvs_knn3d(const float* xyz, int64_t* idx64, int32_t* idx32, int B, int D, int H, int W,
               int ksize, int knn, pmvs_stream_t stream);

/* ---- a6: FeatureFetcher.forward  (utils/feature_fetcher.py:13-60) ----------------- */
/* feature_maps [B,V,C,H,W], pts [B,3,N], K [B,V,3,3], E [B,V,3,4] (NULL = identity,
 * feature_fetcher.py:33-34) -> out [B,V,C,N]; bilinear, zeros padding,
 * align_corners=True semantics (PyTorch 1.0.1 grid_sample, README.md:33-37). */
int pmvs_feature_fetch(const float* feature_maps, const float* pts, const float* intrinsics,
                       const float* extrinsics, float* out, int B, int V, int C, int H, int W,
                       int N, pmvs_stream_t stream);
/* backward w.r.t. feature_maps (coordinates are under no_grad, feature_fetcher.py:29):
 * grad_maps [B,V,C,H,W] is zeroed inside, then scatter-added. */
int pmvs_feature_fetch_backward(const float* grad_out, const float* pts, const float* intrinsics,
                                const float* extrinsics, float* grad_maps, int B, int V, int C,
                                int H, int W, int N, pmvs_stream_t stream);
/* The same gradient with a FIXED summation order (FeatureFetcher's backward under
 * torch.use_deterministic_algorithms(True)).  Every unmasked tap of every point is a record (texel, weight w), zero
 * weights included; grad_maps[b,v,c,t] (every element written) is the fp32 sum, starting from 0, of the rounded products
 * fl(w * grad_out[b,v,c,n]) of the records that hit texel t, added one rounding at a time in ascending (n, tap) order,
 * taps in the order nw, ne, sw, se.  That is exactly what a sequential CPU loop over the records in that order computes,
 * and the same products the atomic entry adds in an arbitrary order.  The taps are the forward's, bit for bit.  The
 * result depends only on the (b, v)'s own inputs, not on B, V, the layouts of other views or the launch geometry.  No
 * allocation, no synchronisation.  Limits: those of pmvs_feature_fetch (H, W > 1, B*V <= 65535) and
 * 4*max(N, H*W) < 2^31.  workspace: pmvs_feature_fetch_backward_det_workspace_bytes(...) bytes, 256-byte aligned, device
 * memory. */
size_t pmvs_feature_fetch_backward_det_workspace_bytes(int B, int V, int C, int H, int W, int N); /* 0 + pmvs_last_error on a bad shape */
int pmvs_feature_fetch_backward_det(const float* grad_out, const float* pts, const float* intrinsics,
                                    const float* extrinsics, float* grad_maps, int B, int V, int C, int H, int W, int N,
                                    void* workspace, size_t workspace_bytes, pmvs_stream_t stream);
/* The forward's taps as records: texel [B,V,N,4] int64 (y*W + x of the nw, ne, sw, se tap, -1 where the tap is masked:
 * outside the map, or a non-finite projection) and weight [B,V,N,4] (the bilinear weights, also where masked).  The
 * records pmvs_feature_fetch_backward_det sums over. */
int pmvs_feature_fetch_taps(const float* pts, const float* intrinsics, const float* extrinsics, int64_t* texel,
                            float* weight, int B, int V, int H, int W, int N, pmvs_stream_t stream);

/* ---- (next row, SURVEY 8f-1) coarse-stage plane sweep: fetch + variance  (model.py:54-113) ------ */
/* features [B,V,C,h,w] (coarse_img_conv conv3 per view, view 0 = reference), cam_params
 * [B,V,2,4,4] at full image resolution (K rows 0,1 are divided by 2, and by 8 in total when
 * is_test, model.py:58-61; depth_start / interval / num_depth are read from cam_params[:,0,1,3,:])
 * -> cost [B,C,D,h,w]: variance over views of the features fetched at the D depth-hypothesis planes,
 * the reference view contributing its un-warped feature (model.py:103-113).  C % 16 == 0.
 * workspace: at least B*(28+24V)*4 bytes. */
int pmvs_cost_volume(const float* features, const float* cam_params, float* cost, void* workspace,
                     size_t workspace_bytes, int B, int V, int C, int h, int w, int D, int is_test,
                     pmvs_stream_t stream);

/* Backward of pmvs_cost_volume with respect to the features (the cameras get no gradient: the reference computes the
 * fetch coordinates under no_grad, feature_fetcher.py:29).  grad_cost [B,C,D,h,w] -> grad_features [B,V,C,h,w], every
 * element written.  View 0 gets sum_d g 2 (f_0 - mean) / V (its un-warped feature; its fetched samples are overwritten
 * in the forward and get nothing); view v >= 1 gets, per texel, the bilinear-weighted sum of g 2 (f_v - mean) / V over
 * the plane points whose unmasked taps hit it.  The taps are the forward's, bit for bit.  Deterministic: no
 * floating-point atomics, every sum in an order fixed by the shapes.  No allocation, no synchronisation.  Limits: those
 * of pmvs_cost_volume and (V-1)*4*D*h*w < 2^31.  workspace: pmvs_cost_volume_backward_workspace_bytes(...) bytes,
 * 256-byte aligned, device memory. */
size_t pmvs_cost_volume_backward_workspace_bytes(int B, int V, int C, int h, int w, int D); /* 0 + pmvs_last_error on a bad shape */
int pmvs_cost_volume_backward(const float* features, const float* cam_params, const float* grad_cost,
                              float* grad_features, void* workspace, size_t workspace_bytes, int B, int V, int C,
                              int h, int w, int D, int is_test, pmvs_stream_t stream);

/* ---- layout helpers used by the module-level API --------------------------------- */
/* batched 2-D transpose: in [batch, R, C] -> out [batch, C, R] */
int pmvs_transpose(const float* in, float* out, int batch, int R, int C, pmvs_stream_t stream);
int pmvs_idx64_to_idx32(const int64_t* in, int32_t* out, long long n, pmvs_stream_t stream);

/* ---- a11/a12: EdgeConvNoC / EdgeConv on points-major data  (networks.py:9-81) ----- */
/* One layer over `groups` BatchNorm groups of `rows_per_group` points each
 * (rows_per_group = clouds_per_group * N; neighbour indices are local to a cloud of N
 * points).  x [R, ldx] points-major (R = groups*rows_per_group), w12 [2*cout, cin]
 * (conv1.weight rows then conv2.weight rows), idx32 [R, K], gamma/beta BN affine
 * ([2*cout] if concat_central else [cout]).  BatchNorm uses batch statistics over
 * (clouds, N, K) per group (test.py:58 keeps train mode).  out [R, ldo] receives
 * (2*cout if concat_central else cout) channels starting at column 0 of `out`.
 * le_scratch [R, 2*cout] fp32 and stats_scratch [groups, 4*cout] fp64 are caller-provided
 * scratch.  bn_train != 0: stats_scratch is zeroed and filled with the batch sums per group
 * [sum_c, sumsq_c, sum_n, sumsq_n] x cout (sum_c over rows, sum_n over rows*K), which the
 * caller may use to update running statistics.  bn_train == 0 (module.eval()): the caller
 * pre-fills stats_scratch with sums that encode the statistics to normalise with
 * (mean*count, (var+mean^2)*count) and no batch statistics are computed. */
int pmvs_edgeconv_pm(const float* x, int ldx, const int32_t* idx32, const float* w12,
                     const float* gamma, const float* beta, float eps, int concat_central,
                     int bn_train, float* out, int ldo, float* le_scratch, double* stats_scratch,
                     int groups, int rows_per_group, int N, int K, int cin, int cout,
                     pmvs_stream_t stream);

/* Backward of pmvs_edgeconv_pm for ONE BatchNorm group of B*N rows (B clouds of N points; the
 * neighbour indices are local to a cloud).  Inputs are what the forward used or produced: x [B*N, ldx]
 * points-major, idx32 [B*N, K] and the same indices as int64 idx64 (for the inverse neighbour lists),
 * w12 [2*cout, cin], gamma/beta, le [B*N, 2*cout] (le_scratch after the forward) and stats [4*cout]
 * fp64 (stats_scratch after the forward: the batch sums when bn_train != 0, the caller's running-
 * statistic sums when bn_train == 0).  dy [B*N, lddy] is the points-major gradient of `out`.
 * Outputs: dx [B*N, lddx] points-major (NULL: not computed), dw12 [2*cout, cin], dgamma/dbeta (same
 * length as gamma).  The ReLU mask is recomputed from le and stats with the forward's arithmetic.
 * bn_train == 0 (frozen statistics): the batch-statistic terms of the BatchNorm backward are zero.
 * Deterministic: every sum has a fixed order (per-CTA partials over a fixed row partition combined
 * in order, inverse neighbour lists sorted by source position, weight gradients over fixed 1024-row
 * slabs), so the result is the same bits on every run and any H100.  Shape limits as the forward:
 * cout in {16, 32, 64, 128}, cin % 8 == 0, cin <= 224, B*N*K < 2^31; ldx, lddy, lddx multiples of 4.
 * workspace: pmvs_edgeconv_pm_backward_workspace_bytes(B, N, K, cin, cout) bytes (0 = unsupported
 * shape), 256-byte aligned, device memory. */
size_t pmvs_edgeconv_pm_backward_workspace_bytes(int B, int N, int K, int cin, int cout);
int pmvs_edgeconv_pm_backward(const float* x, int ldx, const int32_t* idx32, const int64_t* idx64,
                              const float* w12, const float* gamma, const float* beta, float eps,
                              int concat_central, int bn_train, const float* le, const double* stats,
                              const float* dy, int lddy, float* dx, int lddx, float* dw12,
                              float* dgamma, float* dbeta, void* workspace, size_t workspace_bytes,
                              int B, int N, int K, int cin, int cout, pmvs_stream_t stream);

/* ---- a14 building block: 1x1 convolution on points-major rows (nn/conv.py:21-30) ---------- */
/* y[r, 0:cout] = f(x[r, 0:cin]) * w[cout, cin]^T over groups * rows_per_group rows.
 * Optional fused input BatchNorm(batch statistics)+ReLU: in_stats [groups, 2*cin] fp64 sums and
 * sums of squares over in_count values, in_gamma/in_beta [cin].  Optional out_stats
 * [groups, 2*cout] fp64 (caller zeroes): per-column sum and sum of squares of y are ADDED.
 * cin % 8 == 0, cin <= 224, cout % 4 == 0, ldx/ldy % 4 == 0. */
int pmvs_linear_pm(const float* x, int ldx, const float* w, float* y, int ldy, int groups,
                   int rows_per_group, int cin, int cout, const double* in_stats,
                   const float* in_gamma, const float* in_beta, double in_count, float eps,
                   double* out_stats, pmvs_stream_t stream);

/* ---- a1..a15: one PointFlow iteration  (model.py:150-295, test branch :206-269,
 *      train branch :271-293 when is_test == 0) -------------------------------------- */
typedef struct pmvs_flow_weights {
  /* flow_edge_conv.{0,1,2}: w12 = [conv1.weight ; conv2.weight] stacked on dim 0 */
  const float* ec_w12[3];   /* [64,136], [64,32], [128,64] */
  const float* ec_gamma[3]; /* [32], [64], [128] */
  const float* ec_beta[3];
  /* flow_mlp.0.{0,1,2}.conv.weight + bn, flow_mlp.1.weight */
  const float* mlp_w[4];    /* [64,224], [64,64], [16,64], [1,16] */
  const float* mlp_gamma[3];
  const float* mlp_beta[3];
  /* optional BatchNorm running statistics (NULL = do not update); updated exactly as
   * nn.BatchNorm in train mode would after S = ratio^2 sequential calls */
  float* ec_run_mean[3];
  float* ec_run_var[3];
  float* mlp_run_mean[3];
  float* mlp_run_var[3];
  float momentum;           /* 0.1 (nn/conv.py:17, torch default) */
  float eps;                /* 1e-5 */
  /* optional BatchNorm num_batches_tracked counters (int64, NULL = skip): += S per call */
  long long* ec_nbt[3];
  long long* mlp_nbt[3];
} pmvs_flow_weights;

typedef struct pmvs_flow_shape {
  int B;          /* reference views (batch) processed together */
  int V;          /* views incl. the reference view (dataset.py:84) */
  int pyr_h[3], pyr_w[3]; /* pyramid level sizes: conv1 (H/2), conv2 (H/4), conv3 (H/8) */
  int prev_h, prev_w; /* size of the incoming depth map */
  int flow_h, flow_w; /* int(H*image_scale), int(W*image_scale) (model.py:154-155) */
  float image_scale;  /* 0.125 / 0.25 / 0.5 / 1.0 (config.py:70) */
  int ratio;          /* sub-grid stride: int(image_scale*8) in test mode for scales
                         0.25/0.5/1.0 (model.py:237), 1 otherwise; S = ratio^2 sub-clouds */
  int is_test;        /* 1: K *= image_scale (model.py:160-161); 0: K *= 4*image_scale
                         (model.py:162-163) */
  float interval_scale; /* the hypothesis spacing is interval[b] * interval_scale (fp32 product,
                           model.py:301 inter_scale * depth_interval); use 1 if pre-multiplied */
  /* Sub-cloud sharding over GPUs (SURVEY 8e): the ratio^2 strided sub-clouds of an iteration are independent
   * calls in the reference (model.py:236-267).  sub_count > 0 restricts this call to the sub-clouds
   * [sub_begin, sub_begin + sub_count) in the reference's (i, j) loop order s = i*ratio + j: only their
   * pixels of depth_out / prob_out are written, and the workspace is sized for sub_count sub-clouds.
   * sub_count == 0 (default): all of them. */
  int sub_begin, sub_count;
} pmvs_flow_shape;

/* bytes of device workspace pmvs_point_flow_iter needs for this shape */
size_t pmvs_point_flow_workspace_bytes(const pmvs_flow_shape* shape);

/* pyramids: three levels (conv1 16ch @H/2, conv2 32ch @H/4, conv3 64ch @H/8), each
 * CHANNELS-LAST [B,V,h_l,w_l,C_l] (use pmvs_pyramid_to_channels_last once per pass);
 * depth_prev [B,1,prev_h,prev_w]; cam_params [B,V,2,4,4] (io.py:31-45);
 * interval [B] (already multiplied by the iteration's inter_scale, model.py:301);
 * mean,std [B,3].  Outputs: depth_out [B,1,h,w] (h = int(H*image_scale)),
 * prob_out [B,5,h,w] (may be NULL). */
int pmvs_point_flow_iter(const pmvs_flow_shape* shape, const pmvs_flow_weights* weights,
                         const float* const pyramids_cl[3], const float* depth_prev,
                         const float* cam_params, const float* interval, const float* mean,
                         const float* std, float* depth_out, float* prob_out, void* workspace,
                         size_t workspace_bytes, pmvs_stream_t stream);

/* [B*V, C, h, w] -> [B*V, h, w, C] */
int pmvs_pyramid_to_channels_last(const float* nchw, float* nhwc, int BV, int C, int h, int w,
                                  pmvs_stream_t stream);

/* Debug/inspection view of the workspace after pmvs_point_flow_iter (used by the parity
 * tests to compare every stage with the oracle).  Returns byte offsets into workspace:
 * off[0]=feature [S,B,N,136], off[1]=xyz [S,B,3,N], off[2]=idx32 [S,B,N,16] (valid if off[9]),
 * off[3]=edge cat [S,B,N,224], off[4]=mlp h2 [S,B,N,16], off[5]=LE scratch, off[6]=BN sums,
 * off[7]=total bytes, off[8]=kNN neighbour codes [S,B,N,16] uint16 (inside the grid: (dd+2)*96 +
 * (dh+2)*12 + (dw+2), the row offset in the EdgeConv halo tile; outside: bit 15 + candidate id
 * d*25+h*5+w of the 5x5x5 window), off[9]=1 if idx32 was materialised;
 * S = ratio^2, N = 5*h'*w'. */
int pmvs_point_flow_debug_offsets(const pmvs_flow_shape* shape, size_t off[10]);

/* Rewrites the feature region (off[0]) of a workspace after pmvs_point_flow_iter with the unfused fetch kernel:
 * under PMVS_OPT_FETCH 3 the iteration does not write it.  Needs the camera blocks and the resized pyramid map the
 * iteration left in the workspace and the same depth_prev [B,1,prev_h,prev_w]; the values are bit-identical to
 * the rows the iteration contracted.  Also rewrites xyz with the same values. */
int pmvs_point_flow_debug_feature(const pmvs_flow_shape* shape, const float* depth_prev, void* workspace,
                                  pmvs_stream_t stream);

/* ---- backward of one PointFlow iteration (train branch, model.py:150-204, 271-293) ------------ */
/* Output pointers of pmvs_point_flow_backward.  Every output is overwritten, not accumulated.  The parameter
 * gradients are required; the input gradients may be NULL ("not needed").  ec_dw12[l] is [conv1.weight ; conv2.weight]
 * stacked as in pmvs_flow_weights.  dpyramids_cl[l] is [B,V,h_l,w_l,C_l] (the forward's channels-last layout),
 * ddepth_prev [B,1,prev_h,prev_w]. */
typedef struct pmvs_flow_grads {
  float* ec_dw12[3];
  float* ec_dgamma[3];
  float* ec_dbeta[3];
  float* mlp_dw[4];
  float* mlp_dgamma[3];
  float* mlp_dbeta[3];
  float* dpyramids_cl[3];
  float* ddepth_prev;
} pmvs_flow_grads;

/* bytes of device workspace pmvs_point_flow_backward needs; 0 (with pmvs_last_error) for a shape it does not take.
 * The backward takes one cloud per call: ratio 1 (every train-branch call and the test branch at scale 0.125) and
 * sub_count 0. */
size_t pmvs_point_flow_backward_workspace_bytes(const pmvs_flow_shape* shape);

/* Gradients of one pmvs_point_flow_iter call with respect to the flow parameters, the pyramids and depth_prev, given
 * grad_depth_out [B,1,h,w] and grad_prob_out [B,5,h,w] (NULL = zero).  The inputs are those of the forward call and
 * fwd_workspace is its workspace, unchanged since, with the implementation options (pmvs_set_option,
 * pmvs_set_gemm_mode) as they were for it; it is only read, so the call can be repeated.  BatchNorm uses the batch
 * statistics the forward computed.  When neither a pyramid nor depth_prev gradient is requested the fetch backward is
 * skipped.  Deterministic: no floating-point atomics, every sum in an order fixed by the shapes.  The weight gradients
 * follow pmvs_set_gemm_mode like the stand-alone EdgeConv backward.  workspace:
 * pmvs_point_flow_backward_workspace_bytes(shape) bytes, 256-byte aligned, device memory. */
int pmvs_point_flow_backward(const pmvs_flow_shape* shape, const pmvs_flow_weights* weights,
                             const float* const pyramids_cl[3], const float* depth_prev,
                             const float* cam_params, const float* interval, const float* mean,
                             const float* std, const void* fwd_workspace, const float* grad_depth_out,
                             const float* grad_prob_out, const pmvs_flow_grads* grads, void* workspace,
                             size_t workspace_bytes, pmvs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PMVS_B200_H_ */
