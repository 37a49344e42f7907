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

/* ---- depth-map fusion (the step the reference hands to the external fusibile binary, tools/depthfusion.py:173-192) */
/* A fusibile-style fusion with this library's own rule (DESIGN 3.10); not bit-compatible with fusibile, and no normal
 * test.  depth [V,H,W]: a pixel is valid iff 0 < d <= FLT_MAX.  cam_block [V,40] (host-built by
 * utils/depthfusion.py:fusion_camera_block): Kinv[9], Rinv[9], t[3], R[9], K[9], pad, fp32, K at the depth maps'
 * resolution.  Reference views r are taken in ascending order; a valid pixel of r that no accepted point has claimed
 * (used[r,y,x] == 0 at r's turn) is checked against every other view j in ascending order: back-project at the pixel
 * centre, project into j, read depth[j] at the floored position, back-project that pixel centre, project into r; j is
 * consistent when both projections are in front of their camera, the round trip lands within reproj_thresh pixels and
 * the depths agree within depth_thresh * depth[j].  count_out[r,y,x] = the number of consistent views (-1 where the
 * pixel is not processed); xyz_out[r,y,x] = (X + sum_j Y_j) / (count + 1), summed in ascending j (0 where count = -1).
 * A pixel with count >= num_consistent is accepted and sets used = 1 at the pixel of every consistent j.  Every
 * operation is one fp32 rounding (no FMA contraction), so the result is a function of the inputs alone.  used_out
 * [V,H,W] (may be NULL) receives the final used map.  Limits: V, H, W >= 1, V*H*W < 2^31, num_consistent >= 1,
 * thresholds finite and >= 0.  One launch per view, no allocation, no synchronisation; the used map lives in the
 * workspace (pmvs_fuse_depth_maps_workspace_bytes(V, H, W) bytes, 256-byte aligned, device memory) and is zeroed
 * inside with an async memset. */
size_t pmvs_fuse_depth_maps_workspace_bytes(int V, int H, int W); /* 0 + pmvs_last_error on a bad shape */
int pmvs_fuse_depth_maps(const float* depth, const float* cam_block, int V, int H, int W, int num_consistent,
                         float depth_thresh, float reproj_thresh, int* count_out, float* xyz_out,
                         unsigned char* used_out, void* workspace, size_t workspace_bytes, pmvs_stream_t stream);

/* ---- point-cloud evaluation (DESIGN 3.11): accuracy / completeness of a fused cloud against a reference scan ---- */
/* The library's own DTU-style rule, not claimed to reproduce the DTU MATLAB evaluation's numbers.  xyz arrays are
 * [n,3] fp32 device memory; a point with a non-finite coordinate is never kept by thinning and is nobody's neighbour.
 * d2(p, q) = (dx*dx + dy*dy) + dz*dz with dx = q.x - p.x, every operation one fp32 rounding (no FMA contraction).
 * Both searches run over a hashed grid of side `cell`, a power of two in [2^-60, 2^60]; the results do not depend on
 * it (it only sets the speed: about dst for thinning, max_dist / 16 for distances).  Counts n, nq, nt are in
 * [0, 2^31 - 1).  No floating-point atomics, no allocation, no synchronisation; results do not depend on thread order.
 *
 * Greedy radius thinning: visit the points in the order `order` (int64 [n], a permutation of 0..n-1); a visited point
 * that has not been removed is kept and removes every q with d2 <= fl(dst*dst).  Computed as rounds of the parallel
 * greedy maximal independent set, whose outcome equals the sequential one: in round r an undecided point with a
 * neighbour kept before r is removed, and one with no such neighbour and no neighbour still undecided at the start of
 * r earlier in the order is kept.  One call runs rounds [first_round, first_round + rounds); call it with first_round =
 * 0, then again with first_round advanced by `rounds` while undecided[rounds - 1] > 0 (a round after the last useful
 * one returns at once).  state [n] int32 (device) carries the rounds between calls: 0 undecided, 2r+2 kept in round
 * r, 2r+3 removed in round r, 1 removed (non-finite); kept = state > 0 && even.  undecided [rounds] int32 (device):
 * points still undecided after each round of the call.  dst finite > 0; first_round + rounds <= 2^29.  workspace:
 * pmvs_thin_cloud_workspace_bytes(n) bytes, 256-byte aligned, device memory (the grid is rebuilt by every call). */
size_t pmvs_thin_cloud_workspace_bytes(int n); /* 0 + pmvs_last_error on a bad shape */
int pmvs_thin_cloud(const float* xyz, const int64_t* order, int n, float dst, float cell, int first_round, int rounds,
                    int* state, int* undecided, void* workspace, size_t workspace_bytes, pmvs_stream_t stream);
/* Exact nearest-neighbour distances: dist[i] = sqrt(min over the target of d2(query_i, t)) (correctly rounded) when
 * that is <= max_dist, +inf otherwise (also for an empty target), NaN for a query with a non-finite coordinate.
 * max_dist finite >= 0.  workspace: pmvs_nearest_distances_workspace_bytes(nt) bytes, 256-byte aligned, device
 * memory. */
size_t pmvs_nearest_distances_workspace_bytes(int nt); /* 0 + pmvs_last_error on a bad shape */
int pmvs_nearest_distances(const float* query, int nq, const float* target, int nt, float max_dist, float cell,
                           float* dist, void* workspace, size_t workspace_bytes, pmvs_stream_t stream);
/* Filters of the evaluation, flags [n] uint8 (device): bit 0 "in the box" fl(bb[c] - margin) <= p_c <
 * fl(bb[3+c] + margin) on every axis; bit 1 "observed": in the box and, with a mask, g_c = rintf((p_c - bb[c]) / res)
 * inside mask_dims with obs_mask[(g0*dims1 + g1)*dims2 + g2] != 0; bit 2 "above the plane" ((P0 x + P1 y) + P2 z) + P3
 * > 0.  Each operation is one fp32 rounding.  A filter not given (bb / plane NULL) passes every finite point; a point
 * with a non-finite coordinate gets 0.  bb [6] (BB[0] xyz then BB[1] xyz), mask_dims [3] and plane [4] are HOST
 * arrays read during the call; obs_mask is device memory, C order, and needs bb, mask_dims and res finite > 0. */
int pmvs_cloud_filter(const float* xyz, int n, const float* bb, float margin, const unsigned char* obs_mask,
                      const int* mask_dims, float res, const float* plane, unsigned char* flags,
                      pmvs_stream_t stream);

/* ---- coarse stage: VolumeConv and the depth regression (DESIGN 3.12; networks.py:127-167, model.py:115-130) ---- */
/* The parameters of a conv-BatchNorm tower of 11 convolutions, the first ten followed by BatchNorm (VolumeConv,
 * ImageConv).  weight[l] is the PyTorch tensor as stored; running_mean / running_var are read in eval mode only and
 * never written. */
typedef struct pmvs_conv_bn_weights {
  const float* weight[11];
  const float* gamma[10];
  const float* beta[10];
  const float* running_mean[10];
  const float* running_var[10];
  float eps[10];
} pmvs_conv_bn_weights;

/* Gradients of a conv-BatchNorm tower in the PyTorch layouts, overwritten (not accumulated), like pmvs_flow_grads. */
typedef struct pmvs_conv_bn_grads {
  float* weight[11];
  float* gamma[10];
  float* beta[10];
} pmvs_conv_bn_grads;

/* The 11 layers in the reference's attribute order: conv0_1, conv1_0, conv2_0, conv3_0, conv1_1, conv2_1, conv3_1,
 * conv4_0, conv5_0, conv6_0, conv6_2.  weight[l] is Conv3d [Cout, Cin, 3, 3, 3] (l != 7, 8, 9), ConvTranspose3d [Cin,
 * Cout, 3, 3, 3] (l = 7, 8, 9).  The BatchNorm arrays cover the first ten layers (conv6_2 has none). */
typedef pmvs_conv_bn_weights pmvs_volume_weights;

/* x [B, Cin, D, H, W] fp32 (the layout of the cost volume) -> out [B, 1, D, H, W]: the forward of VolumeConv with
 * BatchNorm on batch statistics (train != 0; biased variance for normalising) or on the running statistics (train ==
 * 0).  In train mode batch_sums (fp64 device memory, may be NULL) receives, per BatchNorm layer in the order above,
 * the sums and then the sums of squares of that layer's convolution output over B * D' * H' * W' (D' = D >> level):
 * [sum[Cout_l], sumsq[Cout_l]] for l = 0..9, 576 doubles for (64, 8); the caller updates its running statistics from
 * them.  Supported: (in_channels, base_channels) = (64, 8), D, H, W positive multiples of 8, D*H*W <= 2^30, B <= 8192.
 * fp32 FMA arithmetic; reductions in a fixed order (no floating-point atomics), so two calls give the same bits.  22
 * launches, no allocation, no synchronisation; workspace: pmvs_volume_conv_workspace_bytes(...) bytes, 256-byte
 * aligned, device memory. */
size_t pmvs_volume_conv_workspace_bytes(int B, int in_channels, int base_channels, int D, int H, int W); /* 0 + error */
int pmvs_volume_conv(const float* x, const pmvs_volume_weights* weights, int train, float* out, double* batch_sums,
                     void* workspace, size_t workspace_bytes, int B, int in_channels, int base_channels, int D, int H,
                     int W, pmvs_stream_t stream);
/* filtered [B, D, H, W] fp32 (VolumeConv's output), cams [B, V, 2, 4, 4] fp32, both device memory -> depth_out and
 * prob_out [B, H, W]: p = softmax(-filtered) over D, depth = sum_d depth_d p_d with depth_d = torch.linspace(start,
 * end, D) as computed on a CUDA device, end = start + (D - 1) * interval in fp32, start / interval =
 * cams[b, 0, 1, 3, 0:2] read on the device; prob = p[clamp(floor(t))] + p[clamp(ceil(t))], t = (depth - start) /
 * interval.  The [B, D, H, W] probability volume is never written.  One launch. */
int pmvs_coarse_depth(const float* filtered, const float* cams, int B, int V, int D, int H, int W, float* depth_out,
                      float* prob_out, pmvs_stream_t stream);

/* ---- image towers: ImageConv for every view in one call (DESIGN 3.14; networks.py:84-124, model.py:71-77,133-148) */
/* The 11 layers in module order: conv0.0, conv0.1, conv1.0, conv1.1, conv1.2, conv2.0, conv2.1, conv2.2, conv3.0,
 * conv3.1, conv3.2.  weight[l] is the PyTorch Conv2d tensor, [Cout, Cin, K, K] (K = 5 for the stride-2 layers conv1.0,
 * conv2.0, conv3.0, else 3).  The BatchNorm arrays cover the first ten layers (conv3.2 is a plain convolution). */
typedef pmvs_conv_bn_weights pmvs_image_weights;

/* Bytes of device workspace pmvs_image_conv needs; 0 (with pmvs_last_error) for a shape it does not serve.  With
 * N = B*V images, level sizes h_0 = H, h_k = ceil(h_(k-1) / 2) (w alike), layer l writing C_l channels at level k_l,
 * nb_l = ceil(h_(k_l) * ceil(w_(k_l) / px_l) / 128) CTAs per image (px_l = 8 for conv0.1, else 4) and up(n) = n
 * rounded up to a multiple of 256:
 *   sum_l up(4 K_l^2 Cin_l C_l)                         packed weights
 * + 2 up(max_{l < 10} 4 N h_(k_l) w_(k_l) C_l)          two ping-pong pre-BatchNorm activations (NHWC)
 * + up(max_{l < 10} 16 V C_l B nb_l)                    per-CTA BatchNorm partials of one layer
 * + 2 up(512 V)                                         two ping-pong per-view scale / shift sets.
 * The activation term is conv0's, 32 N H W bytes, so the total is about 64 B V H W bytes.  Supported:
 * base_channels = 8, B, V >= 1, B*V <= 65535, 1 <= H, W <= 32768, H*W <= 2^28. */
size_t pmvs_image_conv_workspace_bytes(int B, int V, int H, int W, int base_channels);
/* img [B, V, 3, H, W] fp32 -> the feature pyramid of every view, as ImageConv run on each view img[:, v]: level_out[k]
 * (k = 0..3 for conv0 .. conv3; NULL = not written) receives [B, V, h_k, w_k, C_k] (channels_last != 0) or
 * [B, V, C_k, h_k, w_k] (channels_last == 0), C = 8, 16, 32, 64.  conv0 .. conv2 are ReLU(BN(.)) of their stage's last
 * layer, conv3 the plain conv3.2.  BatchNorm uses each view's own batch statistics over (B, h, w) (train != 0; biased
 * variance for normalising) or the running statistics (train == 0); train mode needs B*h_3*w_3 >= 2.  In train mode
 * batch_sums (fp64 device memory, may be NULL) receives, per view v and per BatchNorm layer in the order above, the
 * sums and then the sums of squares of that layer's convolution output over (B, h, w): row v is [sum[C_l],
 * sumsq[C_l]] for l = 0..9, 576 doubles per view; the caller updates its running statistics from them, view by view.
 * Zero padding applies to the activated tensor.  fp32 FMA arithmetic; reductions in a fixed order (no floating-point
 * atomics), so two calls give the same bits.  Every argument is checked before any launch.  No allocation, no
 * synchronisation.  workspace: pmvs_image_conv_workspace_bytes(...) bytes, 256-byte aligned, device memory; level
 * outputs 16-byte aligned. */
int pmvs_image_conv(const float* img, const pmvs_image_weights* weights, int train, float* const* level_out,
                    int channels_last, double* batch_sums, void* workspace, size_t workspace_bytes, int B, int V,
                    int H, int W, int base_channels, pmvs_stream_t stream);

/* The forward of a training step (DESIGN 3.15): pmvs_image_conv with the same arguments, the same launches on the same
 * plan and bit-identical level outputs and batch sums, but a workspace that keeps what pmvs_image_conv_backward reads:
 * every BatchNorm layer's pre-BatchNorm output (NHWC) and per-view scale / shift at its own offset and, in eval mode,
 * a copy of the running statistics it normalised with (one more launch).  Bytes, with the notation above and
 * P_l = h_(k_l) w_(k_l):
 *   sum_l up(4 K_l^2 Cin_l C_l)                          packed weights (as pmvs_image_conv)
 * + sum_{l < 10} [up(4 N P_l C_l) + up(8 V C_l)]          each layer's pre-BatchNorm output and scale / shift
 * + up(max_{l < 10} 16 V C_l B nb_l)                     per-CTA BatchNorm partials of one layer
 * + up(2304)                                             the running statistics of eval mode (576 floats).
 * The activation term is (64 + 48 + 24 + 8) N H W, about 144 B V H W bytes: 566 MB at B = 4, V = 3, 512 x 640. */
size_t pmvs_image_conv_keep_workspace_bytes(int B, int V, int H, int W, int base_channels);
int pmvs_image_conv_keep(const float* img, const pmvs_image_weights* weights, int train, float* const* level_out,
                         int channels_last, double* batch_sums, void* workspace, size_t workspace_bytes, int B, int V,
                         int H, int W, int base_channels, pmvs_stream_t stream);

/* Outputs of pmvs_image_conv_backward: weight[l] Conv2d [Cout, Cin, K, K]. */
typedef pmvs_conv_bn_grads pmvs_image_grads;

/* Bytes of device workspace pmvs_image_conv_backward needs; 0 (with pmvs_last_error) for a shape the forward does not
 * take.  With the notation above, E_l = K_l^2 Cin_l C_l the weights of layer l, and
 * n_l = max(1, min(ceil(4224 / (K_l q_l (C_l / 8) N)), ceil(P_l / 1024))) the weight-gradient chunks per image, where
 * q_l = 1 for conv0.0 and Cin_l / 4 otherwise (chunks of c_l = ceil(P_l / n_l) output pixels, ceil(P_l / c_l) of them):
 *   sum_{l >= 1} up(4 E_l)                               packed data-gradient weights
 * + 2 up(max_l 4 N P_l C_l)                              two gradient buffers, conv0's 32 N H W bytes each
 * + up(max_{l < 10} 16 V C_l B ceil(P_l / max(1, 16384 / C_l)))   BatchNorm-backward partials
 * + up(1024 V)                                           per-view constants of G
 * + up(max_l 8 E_l N ceil(P_l / c_l))                    weight-gradient partials.
 * About 64 B V H W bytes plus the partials: 262 MB at B = 4, V = 3, 512 x 640. */
size_t pmvs_image_conv_backward_workspace_bytes(int B, int V, int H, int W, int base_channels);
/* Gradients of one pmvs_image_conv_keep call.  grad_level[k] (k = 0..3) is the gradient of level k in the layout the
 * forward wrote it ([B, V, h_k, w_k, C_k] with channels_last != 0, else [B, V, C_k, h_k, w_k]), 16-byte aligned; NULL
 * means zero.  Every gradient in grads is written: a layer that no given level depends on (above the coarsest level
 * with a gradient) gets zeros, and its kernels are not launched.  The images get no gradient.  fwd_workspace is that
 * call's workspace, with the same shapes, weights and train flag, not modified since; it is only read, so the call can
 * be repeated.  The ReLU masks and the scale of eval mode are the forward's own kept scale / shift; batch_sums (that
 * call's output, required in train mode) gives each view's batch statistics, and eval mode uses the forward's kept
 * copy of the running statistics: weights->running_mean / running_var are not read, so an update of the module's
 * buffers between forward and backward changes nothing.  Padding gets no gradient.  Per view v, train mode:
 * G = gamma invstd_v (dz - sum dz / n - xhat sum dz xhat / n), eval: G = scale dz; dgamma = sum_v sum dz xhat and
 * dbeta = sum_v sum dz, added in view order.  Every argument is checked before any launch.  fp32 FMA products; per-CTA
 * and final sums in a fixed order (fp64 across threads and CTAs), no floating-point atomics, so two calls give the same
 * bits.  No allocation, no synchronisation.  workspace: pmvs_image_conv_backward_workspace_bytes(...) bytes, 256-byte
 * aligned, device memory (as is fwd_workspace). */
int pmvs_image_conv_backward(const float* img, const pmvs_image_weights* weights, int train, const void* fwd_workspace,
                             const double* batch_sums, const float* const* grad_level, int channels_last,
                             const pmvs_image_grads* grads, void* workspace, size_t workspace_bytes, int B, int V,
                             int H, int W, int base_channels, pmvs_stream_t stream);

/* Outputs of pmvs_volume_conv_backward: weight[l] Conv3d [Cout, Cin, 3, 3, 3]; ConvTranspose3d (l = 7, 8, 9)
 * [Cin, Cout, 3, 3, 3]. */
typedef pmvs_conv_bn_grads pmvs_volume_grads;

/* Bytes of device workspace pmvs_volume_conv_backward needs; 0 (with pmvs_last_error) for a shape the forward does not
 * take.  With V_k = D*H*W / 8^k the voxels of level k, layer l reading Cin_l channels at V_in,l voxels and writing
 * Cout_l at V_out,l, w_l = 27 Cin_l Cout_l and up(n) = n rounded up to a multiple of 256:
 *   sum_l up(4 w_l)                                             packed data-gradient weights
 * + sum_{l < 10} up(4 B Cout_l V_out,l) + up(16 Cout_l)          G_l (the pre-BatchNorm gradient) and its constants
 * + sum_{l != conv1_0} up(4 B Cin_l V_in,l)                      data gradients (conv0_1's: its share of grad_x)
 * + up(max_{l < 10} 16 Cout_l B ceil(V_out,l / 4096))            BatchNorm-backward partials
 * + up(max_l 8 w_l B n_l)                                        weight-gradient partials,
 * n_l = max(1, min(ceil(4224 / (3 Cin_l (Cout_l / c_l) B)), ceil(P_l / 1024))), c_l = 8 (1 for conv6_2), P_l = V_in,l
 * for the transposed layers and V_out,l otherwise.  For (64, 8) that is about 4 B D H W (64 + 3 * 8 + 12) bytes. */
size_t pmvs_volume_conv_backward_workspace_bytes(int B, int in_channels, int base_channels, int D, int H, int W);
/* Gradients of one pmvs_volume_conv call given grad_out [B, 1, D, H, W]: grad_x [B, Cin, D, H, W] (NULL: skipped, with
 * the two largest launches) and, in grads, every weight, gamma and beta.  fwd_workspace is the workspace of a
 * pmvs_volume_conv call with the same shapes, weights and train flag, not modified since; it is only read, so the call
 * can be repeated.  batch_sums is that call's output and is required in train mode (the batch statistics are
 * recomputed from it); eval mode reads the running statistics in weights.  The ReLU masks are the forward's own
 * activations (no gradient at exactly 0, as PyTorch); padding gets no gradient.  Train mode: dgamma = sum dz xhat,
 * dbeta = sum dz, G = gamma invstd (dz - dbeta / n - xhat dgamma / n); eval: G = gamma invstd dz.  Every argument is
 * checked before any launch.  fp32 products; per-CTA and final sums in a fixed order (fp64 across threads and CTAs), no
 * floating-point atomics, so two calls give the same bits.  No allocation, no synchronisation.  workspace:
 * pmvs_volume_conv_backward_workspace_bytes(...) bytes, 256-byte aligned, device memory (as is fwd_workspace). */
int pmvs_volume_conv_backward(const float* x, const pmvs_volume_weights* weights, int train,
                              const void* fwd_workspace, const double* batch_sums, const float* grad_out,
                              float* grad_x /* NULL: skip */, const pmvs_volume_grads* grads, void* workspace,
                              size_t workspace_bytes, int B, int in_channels, int base_channels, int D, int H, int W,
                              pmvs_stream_t stream);
/* Backward of pmvs_coarse_depth with respect to filtered: grad_filtered[b, d] = g p_d (depth - z_d), with g =
 * grad_depth [B, H, W], p = softmax(-filtered) and the planes z_d as the forward computes them, and depth the forward's
 * fp64 expectation before rounding (exactly 0 for D = 1).  The cameras and the probability map get no gradient.  One
 * launch, every element of grad_filtered [B, D, H, W] written. */
int pmvs_coarse_depth_backward(const float* filtered, const float* cams, const float* grad_depth,
                               float* grad_filtered, int B, int V, int D, int H, int W, pmvs_stream_t stream);

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
  /* BatchNorm mode of the six flow layers.  0 (default): batch statistics per sub-cloud, as under model.train(); the
   * running statistics are updated when given.  1: the running statistics, as under model.eval(): ec_run_mean/var and
   * mlp_run_mean/var are required inputs and nothing is written to them, *_nbt and momentum are ignored.  Served by
   * the default kernel families only (PMVS_ERR_ARG otherwise, e.g. under edge=0); pmvs_point_flow_backward rejects it
   * (its backward is pmvs_point_flow_eval_backward, after pmvs_point_flow_eval_keep).
   * An eval call needs a smaller workspace: no BatchNorm sums and no flow_mlp activations. */
  int bn_eval;
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

/* ---- backward with running-statistics BatchNorm (bn_eval = 1: fine-tuning with frozen BatchNorm) ------------- */
/* bytes of device workspace pmvs_point_flow_eval_keep needs: pmvs_point_flow_workspace_bytes plus h0, h1, h2
 * (R x 144 floats), the raw flow_mlp outputs (R floats) and a copy of the running statistics, R = 5 B flow_h flow_w.
 * 0 (with pmvs_last_error) unless bn_eval = 1, ratio 1 and sub_count 0. */
size_t pmvs_point_flow_eval_keep_workspace_bytes(const pmvs_flow_shape* shape);

/* pmvs_point_flow_iter with bn_eval = 1 (required; anything else is PMVS_ERR_ARG), one cloud per call, that also keeps
 * in its workspace what pmvs_point_flow_eval_backward reads: flow_mlp's pre-BatchNorm outputs, the flow head's
 * inputs and the running mean and variance of the six layers as this call read them.  Same launches as the eval
 * iteration; depth_out and prob_out are bit-identical to pmvs_point_flow_iter's. */
int pmvs_point_flow_eval_keep(const pmvs_flow_shape* shape, const pmvs_flow_weights* weights,
                              const float* const pyramids_cl[3], const float* depth_prev,
                              const float* cam_params, const float* interval, const float* mean,
                              const float* std, float* depth_out, float* prob_out, void* workspace,
                              size_t workspace_bytes, pmvs_stream_t stream);

/* bytes of device workspace pmvs_point_flow_eval_backward needs; 0 (with pmvs_last_error) for a shape it does not
 * take (bn_eval != 1, ratio != 1, sub_count != 0). */
size_t pmvs_point_flow_eval_backward_workspace_bytes(const pmvs_flow_shape* shape);

/* pmvs_point_flow_backward for a pmvs_point_flow_eval_keep forward: fwd_workspace is that call's workspace, unchanged
 * since.  Each BatchNorm is the affine map of the running statistics the forward read (its kept copy; the live
 * buffers are not read): dx = g gamma / sqrt(running_var + eps), dgamma = sum g xhat, dbeta = sum g, g the upstream
 * gradient after the forward's ReLU mask, recomputed from the forward's own coefficients.  The running statistics
 * are not written.  Same outputs, options and determinism as pmvs_point_flow_backward. */
int pmvs_point_flow_eval_backward(const pmvs_flow_shape* shape, const pmvs_flow_weights* weights,
                                  const float* const pyramids_cl[3], const float* depth_prev,
                                  const float* cam_params, const float* interval, const float* mean,
                                  const float* std, const void* fwd_workspace, const float* grad_depth_out,
                                  const float* grad_prob_out, const pmvs_flow_grads* grads, void* workspace,
                                  size_t workspace_bytes, pmvs_stream_t stream);

/* Debug/inspection view of the workspace after pmvs_point_flow_backward (eval = 0) or pmvs_point_flow_eval_backward
 * (eval = 1), for a call that requested every input gradient (the fetch regions are only written when an input
 * gradient is requested, dfv and the records only when a pyramid gradient is).  Byte offsets into that workspace, with
 * R = 5 B flow_h flow_w points and P = B flow_h flow_w pixels:
 * off[0]=df0 [R,136] (the gradient of the point features, rows in pmvs_point_flow_debug_offsets' feature order),
 * off[1]=d depth_up [P] (the upsampled previous depth), off[2]=d f_v [P,5,V,112] (the fetched features, per pixel,
 * hypothesis and view), off[3]=tap records [P,5,V,4] int64 (NW, NE, SW, SE texel of the view's [V*h*w] block of
 * the batch element's warp source, -1 for a masked tap), off[4]=tap weights [P,5,V,4], off[5]=d warp source
 * [B][V*h*w + 1][112] (the trailing texel of each batch element is not written), off[6]=total bytes.
 * Refuses exactly the shapes the matching *_workspace_bytes function refuses. */
int pmvs_point_flow_backward_debug_offsets(const pmvs_flow_shape* shape, int eval, size_t off[7]);

/* ---- training loss and metrics (DESIGN 3.16; model.py:308-420, networks.py:170-181 MAELoss) ------------------- */
/* The T predicted depth maps a step is scored on: T = 1 (coarse_depth_map, isFlow false) or T = 3 (coarse_depth_map,
 * flow1, flow2).  pred[t] is [B, 1, h[t], w[t]] fp32 device memory.  Where h[t - 1] == h[t], w[t - 1] must equal w[t]
 * (model.py:362 resizes the previous map only when its height differs). */
typedef struct pmvs_depth_terms {
  const float* pred[3];
  int h[3], w[3];
  int T;
} pmvs_depth_terms;

/* Replaces PointMVSNetLoss.forward and PointMVSNetMetric.forward (model.py:314-339, 382-420).  gt [B, 1, Hg, Wg] and
 * cams [B, V, 2, 4, 4] fp32 device memory.  Term t reads the ground truth at F.interpolate(gt, (h[t], w[t])) (mode
 * nearest, source index min(floor(dst * (float)in / out), in - 1) in fp32), gathered on the fly, and the interval
 * iv_t[b] = s_t * cams[b, 0, 1, 3, 1] in fp32 with s = (1, 0.75, 0.375).  m = (g != 0).
 *   loss_out[t]         = (1 / T) sum_b (sum_p m |p - g| / iv_t[b]) / (sum_p m + 1e-7)          (MAELoss / T)
 *   metric_out[2t + k]  = sum_{b,p} mv [|p - g| / iv_t <= thr_k] / (sum_{b,p} mv + 1e-7), thr = (1, 3) (batch-wide)
 * with mv = m for the coarse term and mv = m [|q - g| / iv_t < valid_threshold] for a flow term, q the previous term
 * (nearest-resized to the term's grid when its height differs).  Divisions are IEEE fp32, so the counts equal an fp32
 * restatement's; sums are fp64 in a fixed order.  stats [T, B, 5] fp64 (written): per (t, b) sum m |p - g|, sum m,
 * sum mv and the two threshold counts, read by the backward.  Two launches, no allocation, no synchronisation, no
 * floating-point atomics. */
int pmvs_depth_loss(const pmvs_depth_terms* terms, const float* gt, int Hg, int Wg, const float* cams, int B, int V,
                    float valid_threshold, float* loss_out, float* metric_out, double* stats, pmvs_stream_t stream);
/* Gradient of the T losses of pmvs_depth_loss with respect to the predictions (the backward of model.py:320-334):
 * grad_pred[t] [B, 1, h[t], w[t]] = grad_loss[t] m sign(p - g) / (T iv_t[b] (sum m + 1e-7)), sign(0) = 0.  grad_loss
 * [T] fp32 and stats (the forward's) are read on the device; every grad_pred[t] is overwritten.  One launch. */
int pmvs_depth_loss_backward(const pmvs_depth_terms* terms, const float* gt, int Hg, int Wg, const float* cams, int B,
                             int V, const double* stats, const float* grad_loss, float* const grad_pred[3],
                             pmvs_stream_t stream);

/* ---- input side: resize, crop and normalise every view of a batch (DESIGN 3.19) ---------------------------------- */
/* bytes of device workspace pmvs_prepare_views needs (the exact per-view sums, 48 N bytes rounded up to 256); 0 (with
 * pmvs_last_error) for arguments pmvs_prepare_views rejects. */
size_t pmvs_prepare_views_workspace_bytes(int N, int V, int H0, int W0, double scale, int crop_y, int crop_x, int H,
                                          int W);
/* src [N, H0, W0, 3] uint8 (N = B V views, as cv2.imread returns them, BGR kept) -> img_out [N, 3, H, W] float32.
 * Each view is resized by `scale` (0 < scale <= 1) to round(H0 scale) x round(W0 scale) (half to even) with OpenCV's
 * 8-bit bilinear rule, bit for bit with cv2.resize(view, None, fx=scale, fy=scale, interpolation=INTER_LINEAR)
 * (which copies the view when that size is H0 x W0),
 * cropped to H x W at (crop_y, crop_x) of the resized frame (the uncropped image is never written), and normalised
 * per (view, channel): (x - mean) / (sqrt(var) + 1e-7) in IEEE float32, where mean and the population variance are
 * the exact statistics of the cropped uint8 values, each correctly rounded to float32.  ref_out (NULL: not written)
 * [N / V, H, W, 3] uint8 receives the crop of view 0 of each group of V views.  Rejected (PMVS_ERR_ARG): N < 1 or
 * > 65535, N not a multiple of V, scale outside (0, 1], a crop outside the resized view, H0 W0 or H W >= 2^31.  Two
 * launches and one memset on `stream`; no floating-point atomics, so two calls give the same bits. */
int pmvs_prepare_views(const unsigned char* src, int N, int V, int H0, int W0, double scale, int crop_y, int crop_x,
                       int H, int W, float* img_out, unsigned char* ref_out, void* workspace, size_t workspace_bytes,
                       pmvs_stream_t stream);

/* ---- probability filter: zero the depths of low flow / coarse confidence (DESIGN 3.20) ---------------------------- */
/* Interpolation modes, with OpenCV's values: 0 NEAREST, 1 LINEAR, 2 CUBIC, 4 LANCZOS4 (K = 1, 2, 4, 8 taps). */
#define PMVS_INTER_NEAREST 0
#define PMVS_INTER_LINEAR 1
#define PMVS_INTER_CUBIC 2
#define PMVS_INTER_LANCZOS4 4
/* bytes of device workspace pmvs_probability_filter needs (the tables plus one [V, Hs, Wd] horizontal-pass buffer per
 * map that is resized); 0 (with pmvs_last_error) for arguments it rejects. */
size_t pmvs_probability_filter_workspace_bytes(int V, int Hd, int Wd, int Hf, int Wf, int Hc, int Wc, int mode);
/* depth [V,Hd,Wd], flow_conf [V,Hf,Wf], init_conf [V,Hc,Wc] fp32 device memory -> out [V,Hd,Wd]: out = depth, or 0
 * where the flow confidence resized to Hd x Wd is < flow_thr or the coarse one is < init_thr (a NaN confidence keeps
 * the depth).  A map already at Hd x Wd is read as is.  The resize is cv2.resize's float32 rule for `mode`, computed
 * from host tables (`tables`, int32 words, copied to the workspace inside): for each resized map in the order flow,
 * coarse, [Wd*K] source columns, [Wd*K] float column coefficients, [Hd*K] source rows, [Hd*K] float row coefficients
 * (utils/depthfusion.py:resize_tables builds them); table_words must be 2 K (Wd + Hd) per resized map.  Horizontal
 * taps are summed first to last; vertical taps last to first where x < (Wd & ~3) and first to last elsewhere, as
 * cv2's 4-lane SIMD loop and its scalar tail do; every product and sum is one fp32 rounding.  Rejected
 * (PMVS_ERR_ARG, before any launch): an unknown mode, a NaN or negative threshold, V or a size < 1, V*H*W >= 2^31 for
 * any map or horizontal-pass buffer, a NULL pointer, a table of the wrong length or with an index outside its map,
 * and LINEAR at an exact 2x downsample in both axes (cv2's area path).  Two launches on `stream`, no atomics. */
int pmvs_probability_filter(const float* depth, const float* flow_conf, const float* init_conf, int V, int Hd, int Wd,
                            int Hf, int Wf, int Hc, int Wc, float flow_thr, float init_thr, int mode,
                            const int* tables, size_t table_words, float* out, void* workspace,
                            size_t workspace_bytes, pmvs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PMVS_B200_H_ */
