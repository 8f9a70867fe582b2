/* libdss_b200 -- C ABI of the H100-native deep-spectral hot path.
 *
 * The reference (lukemelas/deep-spectral-segmentation) has no FFI/plugin interface: the hot path is two Python
 * callables, extract_features (extract/extract.py:21-116) and _extract_eig (extract/extract.py:119-244), that call
 * torch / scipy / pymatting directly. This header declares the entry points a ctypes binding in those two
 * functions uses instead of the library calls, and those of the stages after them (segmentations, semantic
 * segmentation, the dense-CRF refinement); each one cites the reference lines it replaces.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes. Every data pointer is a DEVICE pointer owned by the caller unless
 *     the name ends in _host. The library never synchronises the device and never frees caller memory; all work
 *     is enqueued on the caller's stream (a cudaStream_t passed as void*).
 *   - Scratch memory comes from the caller: query dss_*_workspace_bytes, pass (ws, ws_bytes). Workspaces must be
 *     256-byte aligned. A dss_vit_t handle owns only its packed weights.
 *   - Return value: DSS_OK (0) or a negative dss_status; dss_last_error() gives a thread-local message.
 *     Asynchronous numerical outcomes (eigensolver convergence) are reported through device-side info arrays.
 *   - Row-major, C-contiguous tensors; shapes are written [outer, ..., inner].
 */
#ifndef DSS_B200_H
#define DSS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* dss_stream_t; /* cudaStream_t */

typedef enum {
  DSS_OK = 0,
  DSS_ERR_BAD_ARG = -1,
  DSS_ERR_CUDA = -2,
  DSS_ERR_WORKSPACE = -3,
  DSS_ERR_UNSUPPORTED = -4
} dss_status;

const char* dss_last_error(void);
int dss_version(void);            /* 100 * major + minor */
int dss_device_sm_count(void);    /* SM count of the current device (132 on H100 SXM), <0 on error */

/* Launch accounting: number of kernels this library has launched in this process. */
long long dss_kernel_launch_count(void);
/* Per-kernel-class device timing for roofline reports: while enabled, every kernel launch is bracketed by CUDA
 * events on its stream. dss_profile_enable(1) starts a fresh recording, dss_profile_read synchronises the recorded
 * events and returns the number of classes written to `out` (<0 on error). Not for use inside timed regions. */
typedef struct { const char* name; long long launches; double total_ms; } dss_profile_entry;
void dss_profile_enable(int on);
int dss_profile_read(dss_profile_entry* out, int max_entries);

/* ------------------------------------------------------------------------------------------------------------
 * DINO ViT feature extractor  (replaces utils.get_model + model.get_intermediate_layers + the qkv hook,
 * extract/extract_utils.py:40-50, extract/extract.py:49-53,82-98)
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct dss_vit dss_vit_t;

typedef struct {
  int patch;     /* 16 or 8 */
  int dim;       /* 384 (ViT-S) or 768 (ViT-B); head dim must be 64 */
  int depth;     /* 12 */
  int heads;     /* 6 / 12 */
  int mlp_ratio; /* 4 */
  int grid0;     /* side of the training positional grid: 224 / patch */
  float ln_eps;  /* 1e-6 */
} dss_vit_config;

/* fp32 device pointers in the upstream state_dict layout (torch Linear weight = [out, in]) */
typedef struct {
  const float *ln1_w, *ln1_b;   /* [d] */
  const float *qkv_w, *qkv_b;   /* [3d, d], [3d] */
  const float *proj_w, *proj_b; /* [d, d], [d] */
  const float *ln2_w, *ln2_b;   /* [d] */
  const float *fc1_w, *fc1_b;   /* [4d, d], [4d] */
  const float *fc2_w, *fc2_b;   /* [d, 4d], [d] */
} dss_vit_block_weights;

typedef struct {
  const float* patch_w;   /* [d, 3, P, P] conv weight */
  const float* patch_b;   /* [d] */
  const float* cls_token; /* [d] */
  const float* pos_embed; /* [1 + grid0*grid0, d] */
  const dss_vit_block_weights* blocks; /* host array of `depth` entries */
  const float *norm_w, *norm_b; /* [d] final LayerNorm; may be NULL (only dss_vit_forward_cls needs them) */
} dss_vit_weights;

int dss_vit_create(const dss_vit_config* cfg, dss_vit_t** out);
void dss_vit_destroy(dss_vit_t* h);
/* Arithmetic of a handle's ViT forward. The two modes compute different results:
 *   DSS_VIT_PRECISION_FP16 (the default): fp16 operands in every GEMM and in attention, fp32 accumulation; K features
 *     within about 3e-3 relative L2 of the fp32 model. The throughput path.
 *   DSS_VIT_PRECISION_FP32: every operand of the GEMMs and of attention's two products split as x = hi + lo into three
 *     fp16 values (hi, hi/64, 64 lo), so that each fp16 tensor-core product is hi hi' + hi lo' + lo hi'
 *     (fp32-equivalent; error bound in DESIGN.md section 3); softmax, LayerNorm and exact-erf GELU in fp32. Reproduces
 *     the fp32 reference; three times the tensor-core work, three times the weight memory and a larger workspace.
 * Call before dss_vit_load_weights (the weights are packed for the mode); afterwards, or with another value,
 * DSS_ERR_BAD_ARG. The workspace queries report the size for the handle's mode. */
enum { DSS_VIT_PRECISION_FP16 = 0, DSS_VIT_PRECISION_FP32 = 1 };
int dss_vit_set_precision(dss_vit_t* h, int precision);
/* Packs the weights into the library's fp16 operand layout. The copies run on `stream`: the source buffers must stay
 * valid until it has run them. */
int dss_vit_load_weights(dss_vit_t* h, const dss_vit_weights* w, dss_stream_t stream);

size_t dss_vit_workspace_bytes(const dss_vit_t* h, int B, int H, int W);

/* images_u8 [B, H, W, 3] RGB bytes (what cv2.imread+BGR2RGB yields, extract_utils.py:30-31). The library applies
 * ToTensor + Normalize(ImageNet) (extract_utils.py:53-59) and the top-left crop to patch multiples
 * (extract.py:82-88) on the fly, runs blocks [0, which_block) fully and block `which_block` up to its K projection
 * and writes k_out [B, N, d] fp32 == output_dict['k'] (extract.py:98), N = (H/P)*(W/P).
 * which_block may be negative (python indexing, default -1). */
int dss_vit_forward_k(dss_vit_t* h, const uint8_t* images_u8, int B, int H, int W, int which_block, float* k_out,
                      void* ws, size_t ws_bytes, dss_stream_t stream);

/* Debug/parity hook: residual stream x [B, T, d] fp32 after `n_blocks` full blocks (T = N + 1, CLS first). Like
 * dss_vit_forward_cls it takes the image uncropped: a grid0 x grid0 patch grid from an H != W image gets the
 * resampled positional embedding, as upstream interpolate_pos_encoding decides from the pixel sizes. */
int dss_vit_forward_tokens(dss_vit_t* h, const uint8_t* images_u8, int B, int H, int W, int n_blocks, float* x_out,
                           void* ws, size_t ws_bytes, dss_stream_t stream);

/* The model's own forward (upstream VisionTransformer.forward: all blocks, final LayerNorm, CLS token), which the
 * reference calls on bounding-box crops (extract/extract.py:537-541, extract_bbox_features): cls_out [B, d] fp32.
 * The crop is not cut to patch multiples first, so the stored positional grid is used only when H == W (pixels) and
 * the patch grid is grid0 x grid0, as upstream decides; otherwise it is interpolated. */
int dss_vit_forward_cls(dss_vit_t* h, const uint8_t* images_u8, int B, int H, int W, float* cls_out, void* ws,
                        size_t ws_bytes, dss_stream_t stream);

/* Ragged batches: B images of any sizes in one forward, each treated exactly as the uniform call treats it alone
 * (the crop to patch multiples, its positional grid and the identity rule of interpolate_pos_encoding: pixel H == W for
 * _cls, Hp == Wp for _k), so every image's outputs are the bits of that image run alone.
 * images_u8 packs the images one after another: [sum H_b W_b, 3] uint8 RGB, image b at byte offset
 * 3 * sum_{i<b} H_i W_i; dims_host [B, 2] = {H_b, W_b} (host memory). Outputs are packed the same way:
 * k_out [sum N_b, d] fp32 (image b's N_b = (H_b/P)(W_b/P) rows follow image b-1's), cls_out [B, d] fp32.
 * Workspace: dss_vit_ragged_workspace_bytes(h, dims_host, B, mode) with mode DSS_VIT_RAGGED_K or DSS_VIT_RAGGED_CLS
 * (0 for a bad batch), 256-byte aligned. Checked on the host before any device work: null pointers, B <= 0, negative
 * sizes, an image smaller than one patch (the message names the image) and a small or misaligned workspace are
 * DSS_ERR_BAD_ARG; a batch whose token rows exceed the tensor-map extents (2^31) is DSS_ERR_UNSUPPORTED. Both precision
 * modes. */
enum { DSS_VIT_RAGGED_K = 0, DSS_VIT_RAGGED_CLS = 1, DSS_VIT_RAGGED_PAD = 3 };
size_t dss_vit_ragged_workspace_bytes(const dss_vit_t* h, const int* dims_host, int B, int mode);
int dss_vit_forward_k_ragged(dss_vit_t* h, const uint8_t* images_u8, const int* dims_host, int B, int which_block,
                             float* k_out, void* ws, size_t ws_bytes, dss_stream_t stream);
int dss_vit_forward_cls_ragged(dss_vit_t* h, const uint8_t* images_u8, const int* dims_host, int B, float* cls_out,
                               void* ws, size_t ws_bytes, dss_stream_t stream);

/* The positional tables a ragged forward adds (mode DSS_VIT_RAGGED_*): pos_out [sum T_b, d] fp32 (device), image b's
 * [T_b, d] table at its token rows, as upstream VisionTransformer.interpolate_pos_encoding computes it (bicubic, scale
 * (Hp+0.1)/grid0, the identity rule above). Same arguments and workspace as the forwards. Every forward, uniform or
 * ragged, computes its tables on the device this way, per call: the handle keeps no per-shape state. */
/* dss_vit_forward_last over a ragged batch (images_u8 and dims_host as above). pad = 1: every image on its zero-padded
 * ceil(H_b/P) x ceil(W_b/P) grid, so an image may be smaller than one patch (workspace mode DSS_VIT_RAGGED_PAD);
 * pad = 0: the crop (mode DSS_VIT_RAGGED_K). The identity rule goes by the patch grid, as dss_vit_forward_last's.
 * Outputs are PADDED, not packed: feats_out [B, n_max, d] fp32 (image b's N_b rows at b * n_max) and cls_attn_out
 * [B, heads, n_max] fp32, either may be NULL; n_max >= every N_b. Every row is written: an image's N_b rows are the bits
 * dss_vit_forward_last gives for that image alone, the rows past N_b are +0.0. All checks run on the host before any
 * device work: those of the ragged forwards, pad and which, n_max below an image's N_b (the message names the image),
 * B > 65535 with cls_attn_out (DSS_ERR_BAD_ARG), and B * n_max past 2^31 (DSS_ERR_UNSUPPORTED). Both precision
 * modes. */
int dss_vit_forward_last_ragged(dss_vit_t* h, const uint8_t* images_u8, const int* dims_host, int B, int pad, int which,
                                float* feats_out, int n_max, float* cls_attn_out, void* ws, size_t ws_bytes,
                                dss_stream_t stream);

int dss_vit_pos_embed_ragged(dss_vit_t* h, const int* dims_host, int B, int mode, float* pos_out, void* ws,
                             size_t ws_bytes, dss_stream_t stream);
/* The same interpolation on HOST buffers (pure CPU, no CUDA call): pos_embed_host [1+grid0^2, d] -> out_host
 * [1+Hp*Wp, d], with the stored grid for Hp == Wp == grid0. The device tables are this routine's bits. */
int dss_pos_embed_interp_host(const float* pos_embed_host, int grid0, int d, int Hp, int Wp, float* out_host);

/* ------------------------------------------------------------------------------------------------------------
 * Low-level operators (unit-test surface of the ViT kernels). fp16 operands are IEEE binary16.
 * ------------------------------------------------------------------------------------------------------------ */
typedef enum {
  DSS_EPI_BIAS_F16 = 0,      /* out f16 [M, N] = acc + bias                                   */
  DSS_EPI_BIAS_GELU_F16 = 1, /* out f16 [M, N] = gelu_erf(acc + bias)                         */
  DSS_EPI_BIAS_RESID_F32 = 2,/* out f32 [M, N] += acc + bias   (in-place residual)            */
  DSS_EPI_BIAS_F32 = 3,      /* out f32 [M, N] = acc + bias                                   */
  DSS_EPI_PATCH_F32 = 4,     /* out f32 row (m/rin)*rout + m%rin + 1 = acc + bias + aux[m%rin + 1, :]  (patch embed) */
  DSS_EPI_DROPCLS_F32 = 5    /* out f32 row (m/rin)*rout + m%rin - 1 = acc + bias, rows with m%rin == 0 skipped */
} dss_epilogue;

/* out = epilogue(A[M,K] (f16) * Wt[N,K]^T (f16) + bias[N]) on Hopper tensor cores (TMA-fed wgmma, register accumulator).
 * K % 8 == 0, N % 32 == 0, lda == K, ldw == K. aux/rin/rout only for the row-remapping epilogues. */
int dss_op_gemm_f16(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K, int epilogue,
                    const float* aux, int rin, int rout, dss_stream_t stream);
/* Same contract on CUDA cores (slow, fp32 FMA): in-GPU checker for the tensor-core kernel, used by tests only. */
int dss_op_gemm_f16_simt(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K,
                         int epilogue, const float* aux, int rin, int rout, dss_stream_t stream);
/* Tuning probe: dss_op_gemm_f16 with the plain bias->f16 epilogue and an explicit tile width bn in {128,192,256}
 * (stages is ignored: the ring depth follows from the shared-memory budget of bn). Not used by the product path. */
int dss_debug_gemm_cfg(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K, int bn,
                       int stages, dss_stream_t stream);
/* Debug: dss_op_gemm_f16 with one of the four TMA-store epilogues (BIAS_F16, BIAS_GELU_F16, BIAS_RESID_F32, BIAS_F32)
 * under either GEMM schedule, on the same inputs. schedule 0 = cooperative (both MMA warp groups on one 128 x BN tile,
 * BN the widest of 256 / 192 / 128 dividing N); 1 = ping-pong (each MMA warp group owns 128 x 128 tiles, the groups
 * alternate on the tensor cores; what dss_op_gemm_f16 runs for these epilogues). Not used by the product path. */
int dss_debug_gemm_schedule(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K,
                            int epilogue, int schedule, dss_stream_t stream);
/* Same, with a phase trace (a separately compiled kernel variant): trace (device) receives, per CTA c of the
 * persistent launch (2 * clusters CTAs, clusters = min(items, SMs / 2), items = ceil(ceil(M / 128) / 2) * ceil(N / BN)),
 * S = 4 + 8 * ceil(items / clusters) words at c * S: [0] = ns the TMA producer waited on empty ring slots, then for
 * consumer warp group w and its j-th tile, at 4 + 4 * (w * ceil(items / clusters) + j), the %globaltimer stamps
 * {tile start, first operand slab arrived, last wgmma retired, epilogue issued}; records of tiles not run stay 0.
 * trace_bytes smaller than needed is rejected (DSS_ERR_BAD_ARG, the message names the size). */
int dss_debug_gemm_trace(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K, int epilogue,
                         int schedule, unsigned long long* trace, size_t trace_bytes, dss_stream_t stream);
/* y f16 [M, d] = LayerNorm(x f32 [M, d]) * gamma + beta, d in {384, 768} */
int dss_op_layernorm_f16(const float* x, const float* gamma, const float* beta, void* y, int M, int d, float eps,
                         dss_stream_t stream);
/* qkv f16 [B, T, 3*d] (q | k | v, heads of 64 inside each) -> out f16 [B, T, d] = softmax(q k^T / 8) v, d = 64 * heads,
 * on wgmma (TMA-fed QK^T and PV, S, P and O in registers); the attention of the ViT forward */
int dss_op_attention_tc_f16(const void* qkv, void* out, int B, int T, int heads, dss_stream_t stream);
/* images_u8 [B,H,W,3] -> patches f16 [B*N, 3*P*P], column order (c, py, px), normalised */
int dss_op_im2col_f16(const uint8_t* images_u8, void* patches, int B, int H, int W, int P, dss_stream_t stream);
/* Split-fp16 operators of DSS_VIT_PRECISION_FP32. Each fp32 value v becomes hi = fp16(v), hi/64 and 64 (v - hi), stored
 * as three groups of a row: A order [hi | hi/64 | 64 lo] for activations, B order [hi | 64 lo | hi/64] for weights, so
 * that dss_op_gemm_f16 over K' = 3 K of an A-order [M, 3K] and a B-order [N, 3K] operand is the fp32-equivalent product.
 * x [rows, cols] fp32 -> out f16 [rows, 3 cols]; order 0 = A, 1 = B. */
int dss_op_split_f16(const float* x, void* out, int rows, int cols, int order, dss_stream_t stream);
/* dss_op_layernorm_f16's fp32 value, split: y f16 [M, 3d] in A order */
int dss_op_layernorm_split_f16(const float* x, const float* gamma, const float* beta, void* y, int M, int d, float eps,
                               dss_stream_t stream);
/* h f32 [M, n] -> out f16 [M, 3n] = split(gelu(h)) in A order, exact-erf GELU in fp32 (0.5 x (1 + erf(x / sqrt 2))) */
int dss_op_gelu_split_f16(const float* h, void* out, int M, int n, dss_stream_t stream);
/* dss_op_im2col_f16's fp32 value (pad != 0: dss_op_im2col_pad_f16's grid), split: patches f16 [B*N, 3 * 3P^2] in A order */
int dss_op_im2col_split_f16(const uint8_t* images_u8, void* patches, int B, int H, int W, int P, int pad,
                            dss_stream_t stream);
/* Attention of DSS_VIT_PRECISION_FP32: qkv f32 [B, T, 3d] (q | k | v, heads of 64) -> out f16 [B, T, 3d] = split(softmax(
 * q k^T / 8) v) in A order (each group d wide, head h at columns 64 h), the proj GEMM's operand. qkv_split f16
 * [B, T, 9d] is scratch: per head h, Q' = split(q) in A order at columns 192 h, K' and V' = split(k), split(v) in B order
 * at 3d + 192 h and 6d + 192 h. S = Q' K'^T and P V on the fp16 tensor cores with P split in registers; softmax fp32. */
int dss_op_attention_split_f16(const float* qkv, void* qkv_split, void* out, int B, int T, int heads, dss_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * Affinity + graph Laplacian eigensolver (replaces extract/extract.py:148,191-195,207-235,237-240)
 * ------------------------------------------------------------------------------------------------------------ */
enum { DSS_AFF_NORMALIZE = 1, DSS_AFF_THRESHOLD_AT_ZERO = 2, DSS_AFF_NO_MAX_SCALE = 4 };

size_t dss_affinity_workspace_bytes(int B, int N, int d);
/* feats [B, N, d] fp32 -> Wmat [B, N, ldw] fp32 (row pitch ldw >= N, ldw % 4 == 0, pad columns written as 0):
 *   F^ = F / max(||F||, 1e-12) rowwise (if NORMALIZE)                      extract.py:148
 *   W  = F^ F^T ; W *= (W > 0) (if THRESHOLD) ; W /= max(W)                extract.py:191-194
 *        (NO_MAX_SCALE skips the division: the 'affinity' / 'affinity_svd' branches, extract.py:160-172)
 *   W += color_counts * color_lambda  (if color_counts != NULL)            extract.py:213,221
 *   degree[b, i] = sum_j W[b, i, j]   (if degree != NULL)                  extract_utils.py:217 (row_sum)
 * color_counts [B, N, N] uint8 is the dense KNN colour affinity of dss_knn_color_counts.
 * W is symmetric: only the tiles on or above the diagonal are computed on the tensor cores and each is stored twice
 * (W[i,j] and W[j,i] are the same bits). The row sums are accumulated in the same epilogue (fixed summation order,
 * bit-reproducible) so that the eigensolver does not need another pass over W; pass the result to
 * dss_eigsh_laplacian. A colour term added AFTER this call (dss_rw_affinity_add) updates `degree` itself. */
int dss_affinity(const float* feats, int B, int N, int d, int flags, const uint8_t* color_counts, float color_lambda,
                 float* Wmat, int ldw, float* degree, void* ws, size_t ws_bytes, dss_stream_t stream);
/* Tuning probe (not used by the product path): dss_affinity with the affinity GEMM's phase trace, in the layout of
 * dss_debug_gemm_trace, items = B * (sum over row-tile pairs p of max(ceil(N / 128) - 2 p, 0)). Tiles the pair discards record an epilogue of zero length. */
int dss_debug_affinity_trace(const float* feats, int B, int N, int d, int flags, const uint8_t* color_counts,
                             float color_lambda, float* Wmat, int ldw, float* degree, void* ws, size_t ws_bytes,
                             unsigned long long* trace, size_t trace_bytes, dss_stream_t stream);

/* Colour KNN affinity (extract_utils.py:151-188): rgb [B, Hl*Wl, 3] fp32 in [0,1] (the /255 low-res image of
 * extract.py:199-204). Two exact-KNN passes (k=20, w=2.0) and (k=10, w=0.1) over points (r,g,b,w*x,w*y),
 * x,y = linspace(0,1); counts[i,j] += 1 and counts[j,i] += 1 per directed neighbour pair (self included), i.e.
 * the dense form of the reference's duplicate-summing csr_matrix. counts [B, N, N] uint8 is overwritten; the buffer
 * must be 4-byte aligned and its capacity rounded up to a multiple of 4 bytes (bytes are updated with 32-bit atomics;
 * any N, odd included). */
size_t dss_knn_workspace_bytes(int B, int N);
int dss_knn_color_counts(const float* rgb, int B, int Hl, int Wl, uint8_t* counts, void* ws, size_t ws_bytes,
                         dss_stream_t stream);

/* Eigensolver. Wmat [B, N, ldw] symmetric, non-negative (row pitch ldw as written by dss_affinity). Only the upper
 * triangle (j >= i) of every matrix is read. degree [B, N] = row sums of W as written by dss_affinity, or NULL (the
 * solver then computes them with one more pass over W).
 *   lapnorm != 0: K smallest pairs of (D - W) v = lambda D v, D = diag(rowsum W) (entries < 1e-12 -> 1,
 *                 extract_utils.py:217-218); eigenvectors D-orthonormal            extract.py:225-229
 *   lapnorm == 0: K smallest pairs of (D - W) v = lambda v, unit 2-norm vectors    extract.py:230-234
 * Outputs: evals [B, K] ascending, evecs [B, K, N] with the reference's sign rule applied (extract.py:237-240),
 * info [B, 4] int32, resid [B, K] fp32 residual estimates (may be NULL):
 *   info[b,0] Lanczos steps taken, restarts included
 *   info[b,1] 1 when the K pairs returned are eigenpairs to tol * max(1, ||A||) (vectors orthonormal), else 0: the
 *             step budget ran out first; pairs that do not exist yet are NaN. An exactly repeated eigenvalue breaks
 *             the recurrence down and is returned with all its copies (restarts, info[b,3]); a cluster of distinct
 *             but nearly equal eigenvalues (relative spread ~1e-6) straddling the K-th does not break it down, and
 *             copies from it can be missed while info[b,1] is 1. The tolerance has an absolute floor: scale A so
 *             that ||A|| >= 1 for a relative one (cluster.pca_components does).
 *   info[b,2] dss_eigsh_topk only: a negative eigenvalue is larger in magnitude than the K-th (see below); else 0
 *   info[b,3] restarts: Lanczos breakdowns (an invariant Krylov subspace, e.g. at an eigenvalue of multiplicity > 1)
 *             continued from a fresh start vector orthogonal to the basis; 0 on ordinary spectra
 * Method: Lanczos with full re-orthogonalisation on D^-1/2 W D^-1/2 (null vector deflated analytically), Ritz
 * values by Sturm bisection in fp64. tol <= 0 selects 1e-6; max_steps <= 0 selects min(N-1, 320) (min(N, 320) for
 * dss_eigsh_topk). Restarts draw on the same budget. The Lanczos tridiagonal lives in shared memory, so a budget
 * that does not fit (e.g. N - 1 above N = 3816) is DSS_ERR_UNSUPPORTED. */
size_t dss_eigsh_workspace_bytes(int B, int N, int K, int max_steps);
/* Largest max_steps whose shared memory fits the solver at N, capped at N - 1 (mode 0 / 1: dss_eigsh_laplacian) or N
 * (mode 2: dss_eigsh_topk); 0 when no budget fits or the arguments are invalid. No device work. */
int dss_eigsh_max_steps(int N, int mode);
int dss_eigsh_laplacian(const float* Wmat, const float* degree, int ldw, int B, int N, int K, int lapnorm, float tol,
                        int max_steps, float* evals, float* evecs, int* info, float* resid, void* ws, size_t ws_bytes,
                        dss_stream_t stream);

/* K algebraically largest eigenpairs of the symmetric matrices Amat [B, N, lda], descending, unit 2-norm vectors,
 * reference sign rule applied. Serves which_matrix='affinity' (eigsh(W, which='LM', k=K), extract.py:166-172; for a
 * non-negative affinity the largest-magnitude eigenvalues are the largest positive ones -- info[b,2] is set to 1 if a
 * negative eigenvalue of larger magnitude exists) and 'affinity_svd' (left singular vectors of F^ = eigenvectors of
 * F^ F^T, extract.py:160-163). Same workspace / info / resid conventions as dss_eigsh_laplacian. */
int dss_eigsh_topk(const float* Amat, int lda, int B, int N, int K, float tol, int max_steps, float* evals,
                   float* evecs, int* info, float* resid, void* ws, size_t ws_bytes, dss_stream_t stream);
/* Debug: dss_eigsh_laplacian (mode 0 = lapnorm, 1 = unnormalised) or dss_eigsh_topk (mode 2, degree ignored) with the
 * instantiation forced: variant 1 = <2, 2, 512>, 2 = <4, 1, 512> (the default), 3 = <4, 2, 256>. The paired variants 1
 * and 3 run two CTAs per SM, each with its own scratch slice, so they need up to twice the workspace of
 * dss_eigsh_workspace_bytes; a paired variant whose two CTAs do not fit in shared memory is DSS_ERR_UNSUPPORTED (no
 * fall-back). A bad variant or mode is DSS_ERR_BAD_ARG (the workspace query returns 0). Not used by the product path. */
size_t dss_debug_eigsh_workspace_bytes(int B, int N, int K, int max_steps, int variant);
int dss_debug_eigsh(const float* Wmat, const float* degree, int ldw, int B, int N, int K, int mode, float tol,
                    int max_steps, int variant, float* evals, float* evecs, int* info, float* resid, void* ws,
                    size_t ws_bytes, dss_stream_t stream);

/* Random-walk colour affinity (which_color_matrix='rw', extract_utils.py:191-204 -> pymatting _rw_laplacian with
 * radius 1): Wmat[b, i, j] += float32(sum over the 3x3 clamped neighbourhood offsets that land on j of
 * exp(-coef * ||z_i - z_j||^2)) * color_lambda, z = rgb_u8 / 255 in float64; the same amount is added to degree[b, i]
 * (may be NULL). rgb_u8 [B, Hl*Wl, 3] is the low-resolution image of extract.py:199-204 BEFORE the /255.
 * pymatting hard-codes coef = 900 (its sigma argument is unused); pass 1/sigma^2 for the textbook kernel. */
int dss_rw_affinity_add(const uint8_t* rgb_u8, int B, int Hl, int Wl, float color_lambda, double coef, float* Wmat,
                        int ldw, float* degree, dss_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * Segmentations from the eigenvectors (replace extract/extract.py:283-349 and :364-390), fused after the eigensolve
 * ------------------------------------------------------------------------------------------------------------ */
/* mask[b, n] = 255 if evecs[b, which, n] > threshold else 0   (the 'L' image the reference saves; which = 1) */
int dss_segment_threshold(const float* evecs, int B, int K, int N, int which, float threshold, uint8_t* mask,
                          dss_stream_t stream);
/* Batched K-means (k-means++ seeding, Lloyd, scikit-learn's stopping rules: tol * mean feature variance on the centre
 * shift, strict label convergence, max_iter; empty clusters are re-seeded with the farthest point). One CTA per image.
 * Point n of image b has coordinates points[b * image_stride + n * point_stride + j * dim_stride], j < dims -- the
 * eigenvector embedding evecs[b, 1 + j, n] is (K*N, 1, N) from &evecs[b=0, 1, 0]; raw features [B, N, d] are (N*d, d, 1).
 * n_clusters [B] int32 (device) gives k per image (the reference's adaptive mode), capped by max_clusters <= 64.
 * If infer_bg_index, labels are taken on a grid_h x grid_w grid (grid_h * grid_w == N) and the label with the largest
 * border share is swapped with 0 (extract_utils.py:124-135). labels [B, N] uint8; info [B, 2] = {iterations,
 * converged}; inertia [B] (may be NULL). As in scikit-learn's _kmeans_single_lloyd: a run that stops on tol or at
 * max_iter re-runs the E step, so the labels and the inertia (sum of squared distances) belong to the final centres; an
 * empty cluster takes the point farthest from its centre while the point keeps its E-step label, so the next iteration
 * counts label changes against the E step. seed: counter-based generator keyed by (seed, image_keys[b]) -- image_keys [B]
 * int32 (device; e.g. the `indices` field of the feature files) makes an image's clustering independent of the batch it
 * is processed in; NULL uses the position in the batch. (The reference's clustering is unseeded.) */
int dss_segment_kmeans(const float* points, long long image_stride, long long point_stride, long long dim_stride, int B,
                       int N, int dims, const int* n_clusters, const int* image_keys, int max_clusters, int grid_h,
                       int grid_w, int infer_bg_index, unsigned int seed, int max_iter, float tol, uint8_t* labels,
                       int* info, float* inertia, dss_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * Semantic segmentation: boxes, PCA and data-set k-means (replace extract/extract.py:429-599)
 * ------------------------------------------------------------------------------------------------------------ */
/* Bounding boxes of every segment of a batch of label maps (_extract_bbox, extract.py:429-470): for every label value v
 * of segmaps [B, H, W] uint8, mask = (segmap == v) is eroded num_erode times and then dilated num_dilate times with the
 * 3x3 cross footprint (skimage binary_erosion / binary_dilation: pixels outside the image count as set for erosion and
 * unset for dilation); a step whose result is empty is discarded (extract_utils.py:115-121). boxes [B, 256, 4] int32 =
 * {xmin, ymin, xmax + 1, ymax + 1} on the grid, present [B, 256] uint8 = 1 where v occurs (boxes of absent values are
 * 0). H * W <= 16384 (DSS_ERR_UNSUPPORTED otherwise). One CTA per (image, value). */
int dss_segment_bboxes(const uint8_t* segmaps, int B, int H, int W, int num_erode, int num_dilate, int* boxes,
                       uint8_t* present, dss_stream_t stream);

/* Column mean [d] fp32 and covariance cov [d, ldc] fp32 = (X - mean)^T (X - mean) / (M - 1) of X [M, d] fp32, both
 * accumulated in fp64 through fixed per-CTA partials (bit-reproducible). M >= 2, d <= 1024. cov can be handed to
 * dss_eigsh_topk (ldc % 4 == 0 there) for the covariance-eigh route of scikit-learn's PCA (extract.py:574-577). */
size_t dss_covariance_workspace_bytes(int M, int d);
int dss_covariance(const float* X, int M, int d, float* mean, float* cov, int ldc, void* ws, size_t ws_bytes,
                   dss_stream_t stream);
/* Y [M, p] = (X [M, d] - mean [d]) V^T, V [p, d] the principal axes (PCA.transform without whitening); p <= 64. */
int dss_pca_project(const float* X, int M, int d, const float* mean, const float* V, int p, float* Y,
                    dss_stream_t stream);

/* K-means of all M points of X [M, dims] fp32 (extract_bbox_clusters, extract.py:579-582). Same algorithm and rules as
 * dss_segment_kmeans -- greedy k-means++ seeding with 2 + ln k local trials drawn from the D^2 distribution
 * (deterministic prefix sums), full-batch Lloyd iterations, scikit-learn's stopping rules (centre shift <= tol * mean
 * column variance, strict label convergence, max_iter), empty clusters re-seeded with the farthest points -- with the
 * counter-based generator keyed by `seed`. The reference runs MiniBatchKMeans, a stochastic approximation of the same
 * objective; its label numbers are not reproducible, so results compare up to relabelling. Bit-reproducible: centre sums
 * are 64-bit fixed point, every floating-point reduction has a fixed order. Nothing synchronises: max_iter iterations
 * are enqueued and become no-ops once a device-side flag says the run stopped.
 * centers [k, dims] fp32, labels [M] int32, info [2] int32 = {iterations, converged}, inertia [1] fp32 (may be NULL);
 * labels and inertia belong to the final centres and relocated points keep their E-step labels, as in dss_segment_kmeans.
 * Supported: k <= 64 at dims <= 768, k <= 256 at dims <= 64 (DSS_ERR_UNSUPPORTED otherwise); k <= M.
 * max_iter <= 0 selects 300, tol < 0 selects 1e-4. The workspace query returns 0 for an unsupported shape. */
size_t dss_kmeans_workspace_bytes(int M, int dims, int k);
int dss_kmeans(const float* X, int M, int dims, int k, unsigned int seed, int max_iter, float tol, float* centers,
               int* labels, int* info, float* inertia, void* ws, size_t ws_bytes, dss_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * Dense-CRF refinement to pixel resolution (replaces SimpleCRF's denseCRF.densecrf in _extract_crf_segmentations,
 * extract/extract.py:650-693)
 * ------------------------------------------------------------------------------------------------------------ */
/* Ragged batch of B images: images [sum H*W, 3] uint8 RGB and segmaps [sum seg_h*seg_w] uint8 patch label maps, packed
 * image after image; dims_host [B, 4] = {H, W, seg_h, seg_w} (host), P the downsample factor (H, W >= P).
 * The label of pixel (y, x) is the map's cell under cv2.resize(INTER_NEAREST) to (H_pad, W_pad) = (H, W) rounded down
 * to multiples of P inside that block and to (H, W) in the remaining rows and columns (extract.py:679-681); a caller
 * maps a {0, 255} map to {0, 1} first. Labels must be < num_classes (a larger one gets log eps on every class).
 * Model (Kraehenbuehl & Koltun, Potts, symmetric normalisation; filters on the permutohedral lattice):
 *   -U(l) = 0 at the pixel's label, log(unary_eps) elsewhere; Q0 = softmax(-U);
 *   `iterations` times Q = softmax(-U + w1 n_b L_b(n_b Q) + w2 n_s L_s(n_s Q)), n = 1/sqrt(L(1) + 1e-20);
 *   L_b on features (x/alpha, y/alpha, r/beta, g/beta, b/beta), L_s on (x/gamma, y/gamma), see dss_op_lattice_filter.
 * labels_out [sum H*W] uint8 = argmax Q (first class on ties); prob_out [sum H*W, num_classes] fp32 = Q (may be NULL);
 * info [B, 2] int32 (device) = lattice points {bilateral, spatial} of every image. Deterministic: no floating-point
 * atomics, an image gets the same bits alone or in any batch. 2 <= num_classes <= 64 and lattice keys (image index +
 * coordinates, sized from the largest image and alpha / beta / gamma) within 64 bits, else DSS_ERR_UNSUPPORTED.
 * The workspace covers the worst case of every vertex its own lattice point (about 2.5 KB per pixel at 21 classes);
 * the query returns 0 for an unsupported or malformed shape list. */
size_t dss_crf_workspace_bytes(const int* dims_host, int B, int num_classes);
int dss_crf_segment(const uint8_t* images, const uint8_t* segmaps, const int* dims_host, int B, int P, int num_classes,
                    double w1, double alpha, double beta, double w2, double gamma, int iterations, double unary_eps,
                    uint8_t* labels_out, float* prob_out, int* info, void* ws, size_t ws_bytes, dss_stream_t stream);

/* Permutohedral-lattice Gaussian filter (unit-test surface of dss_crf_segment's filters): features [N, d] fp32,
 * d in {2, 5}, values [N, C] fp32, 1 <= C <= 64. out [N, C] = L(values): elevation with scale
 * sqrt(2/3) (d+1) / sqrt((i+1)(i+2)) on feature i (fp64, no FMA contraction), splat with barycentric weights, blur
 * [1/2, 1, 1/2] along the d+1 lattice directions in order (a missing neighbour counts as 0), slice, times 1/(1 + 2^-d).
 * normalize != 0: out = n L(n values), n = 1/sqrt(L(1) + 1e-20). lattice_points [1] int32 (device, may be NULL).
 * Synchronises `stream`: the feature range is read back to size the 64-bit lattice keys. */
size_t dss_lattice_filter_workspace_bytes(int N, int d, int C);
int dss_op_lattice_filter(const float* features, int N, int d, const float* values, int C, int normalize, float* out,
                          int* lattice_points, void* ws, size_t ws_bytes, dss_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * Object localization (replaces object-localization/object_discovery.py of the reference: get_bbox_from_patch_mask,
 * lost / patch_scoring / detect_box, dino_seg, and the ViT hooks of object-localization/main.py:219-322)
 * ------------------------------------------------------------------------------------------------------------ */
/* Per-image outcomes written to status [B] int32 (device) by the box kernels; the box of a failed image is 0. */
enum { DSS_LOC_OK = 0, DSS_LOC_NO_GRID = 1, DSS_LOC_SEED_IN_BACKGROUND = 2, DSS_LOC_EMPTY_COMPONENT = 3 };

/* The box kernels hold one patch grid of at most 16384 cells (128 x 128) per CTA in shared memory and label it with
 * one union-find whose component roots are their smallest raster index -- the numbering of scipy.ndimage.label and
 * skimage.measure.label. Larger grids are rejected with DSS_ERR_UNSUPPORTED. Boxes [B, 4] int32 = {xmin, ymin, xmax,
 * ymax} in pixels, the max exclusive.
 *
 * Eigen-segmentation (get_bbox_from_patch_mask + get_largest_cc_box): row `which` of evecs [B, K, N] fp32; dims_host
 * [B, 2] = the un-cropped image size {H, W} (host). The grid is the first of (H/8, W/8) P 8, (H/16, W/16) P 16,
 * (2 (H/16), 2 (W/16)) P 8, (4 (H/32), 4 (W/32)) P 8 with N cells (integer division), else status DSS_LOC_NO_GRID.
 * mask = v > 0, complemented if 0.5 < mean < 1 or empty; the largest 8-connected component (ties: the first in
 * label order); box {x0 P, y0 P, min((x1 + 1) P, W), min((y1 + 1) P, H)}. */
size_t dss_eigseg_boxes_workspace_bytes(int B);
int dss_eigseg_boxes(const float* evecs, int B, int K, int N, int which, const int* dims_host, int* boxes, int* status,
                     void* ws, size_t ws_bytes, dss_stream_t stream);
/* LOST on A [B, N, ldw] fp32 = F F^T (dss_affinity with DSS_AFF_NO_MAX_SCALE and no other flag), grid_h x grid_w == N
 * cells of P pixels, un-padded image H x W (all images of the batch). degree_i = #{j != i : A_ij > 0}; patches in
 * ascending degree, ties by index (the reference's unstable argsort leaves ties unspecified); seed = the first;
 * similars = the first min(k_patches, N) with A[seed, p] > 0; M = sum of their rows in that order (fp32); the
 * 4-connected component of M > 0 holding the seed gives {x0 P, y0 P, min((x1 + 1) P, W), min((y1 + 1) P, H)}.
 * M[seed] <= 0: status DSS_LOC_SEED_IN_BACKGROUND. seeds [B] int32 (may be NULL) receives the seed patch. */
size_t dss_lost_workspace_bytes(int B, int N);
int dss_lost_boxes(const float* A, int B, int N, int ldw, int grid_h, int grid_w, int H, int W, int P, int k_patches,
                   int* boxes, int* seeds, int* status, void* ws, size_t ws_bytes, dss_stream_t stream);
/* DINO-seg on the CLS attention cls_attn [B, heads, N] fp32 (dss_vit_forward_last), head < heads: a patch is kept iff
 * the running sum (fp64 accumulator, each prefix rounded to fp32, as torch's CPU cumsum) of the ascending-sorted
 * values (ties by index), each divided by their fp32 total, exceeds float(1 - 0.6). 4-connected labels 1 .. n; as in
 * the reference (which sizes labels 0 .. n-1 only), n >= 2 selects the largest of labels 1 .. n-1 and n <= 1 selects
 * label 0, the cells not kept (status DSS_LOC_EMPTY_COMPONENT if there are none). Box {x0 P, y0 P, (x1+1) P, (y1+1) P},
 * not clipped. */
int dss_dinoseg_boxes(const float* cls_attn, int B, int heads, int N, int head, int grid_h, int grid_w, int P,
                      int* boxes, int* status, dss_stream_t stream);
/* The same two methods on a ragged batch in the padded layout of dss_vit_forward_last_ragged: image b has its own
 * grid and N_b = gh_b gw_b <= n_max cells, and its rows start at b * n_max. Each image's boxes, seeds and status are
 * those of the uniform call on that image alone.
 * LOST: A [B, n_max, ldw] = dss_affinity of the padded features [B, n_max, d] at N = n_max with DSS_AFF_NO_MAX_SCALE
 * (the pad rows are zero, so image b's N_b x N_b block is the affinity of the image alone); dims_host [B, 4] = {gh, gw,
 * H, W} per image (host). DINO-seg: cls_attn [B, heads, n_max]; dims_host [B, 2] = {gh, gw}. Checked on the host
 * before any device work: null pointers, shapes, a grid larger than n_max or with no cells, a small workspace
 * (DSS_ERR_BAD_ARG / DSS_ERR_WORKSPACE) and a grid past 16384 cells (DSS_ERR_UNSUPPORTED); the message names the
 * image. */
size_t dss_lost_ragged_workspace_bytes(int B, int n_max);
int dss_lost_boxes_ragged(const float* A, int B, int n_max, int ldw, const int* dims_host, int P, int k_patches,
                          int* boxes, int* seeds, int* status, void* ws, size_t ws_bytes, dss_stream_t stream);
size_t dss_dinoseg_ragged_workspace_bytes(int B);
int dss_dinoseg_boxes_ragged(const float* cls_attn, int B, int heads, int n_max, int head, const int* dims_host, int P,
                             int* boxes, int* status, void* ws, size_t ws_bytes, dss_stream_t stream);

/* Last-block ViT outputs for localization. pad != 0 zero-pads the NORMALISED image up to multiples of P
 * (object-localization/main.py:227-235) and runs on the ceil(H/P) x ceil(W/P) grid; pad == 0 crops like
 * dss_vit_forward_k. Blocks [0, depth-1) run fully, then the last block's LN1 and:
 *   feats_out [B, N, d] fp32 (may be NULL): the `which` third of its qkv projection (0 = q, 1 = k, 2 = v), CLS row
 *     dropped (the qkv hook of main.py:283-322);
 *   cls_attn_out [B, heads, N] fp32 (may be NULL): softmax(q_0 k_j / 8) over all T = N + 1 tokens, patch entries
 *     (get_last_selfattention(...)[:, :, 0, 1:]), from the fp16 qkv the attention kernels read (the fp32 qkv under
 *     DSS_VIT_PRECISION_FP32).
 * At least one output is required. Workspace: dss_vit_forward_last_workspace_bytes (0 if the image is smaller than a
 * patch in crop mode). */
size_t dss_vit_forward_last_workspace_bytes(const dss_vit_t* h, int B, int H, int W, int pad);
int dss_vit_forward_last(dss_vit_t* h, const uint8_t* images_u8, int B, int H, int W, int pad, int which,
                         float* feats_out, float* cls_attn_out, void* ws, size_t ws_bytes, dss_stream_t stream);
/* qkv f16 [B, T, 3*d] (heads of 64) -> cls_attn [B, heads, T - 1] fp32 = softmax_j(q_0 . k_j / 8)[1:], fp32
 * arithmetic, one CTA per (image, head). T >= 2. */
int dss_op_cls_attention(const void* qkv, int B, int T, int heads, float* cls_attn, dss_stream_t stream);
/* images_u8 [B,H,W,3] -> patches f16 [B*N, 3*P*P] on the ceil(H/P) x ceil(W/P) grid, pixels outside the image 0
 * (after normalisation) */
int dss_op_im2col_pad_f16(const uint8_t* images_u8, void* patches, int B, int H, int W, int P, dss_stream_t stream);

/* Bilinear up-sampling of patch features (align_corners=False, as F.interpolate at extract.py:185-188):
 * feats [B, Hp*Wp, d] fp32 -> out [B, Hl*Wl, d] fp32. Used when image_downsample_factor != patch size. */
int dss_upsample_bilinear(const float* feats, int B, int Hp, int Wp, int d, int Hl, int Wl, float* out,
                          dss_stream_t stream);
/* Row-wise L2 normalisation x / max(||x||, 1e-12) (F.normalize, extract.py:148): feats [rows, d] -> out [rows, d]. */
int dss_normalize_rows(const float* feats, int rows, int d, float* out, dss_stream_t stream);

/* Pillow's Image.resize((W_out, H_out), Image.BILINEAR) of whole images, bit for bit (the low-resolution colour image
 * of extract.py:199-204): images [B, H, W, 3] uint8 RGB, all of one size -> out [B, H_out * W_out, 3],
 *   DSS_RESIZE_U8:       uint8 pixels (which_color_matrix='rw');
 *   DSS_RESIZE_UNIT_F32: fp32 float(pixel / 255.0), the double division rounded once ('knn').
 * Per axis the caller builds (host, int32) bounds [out, 2] = {first input index, count} and weights [out, taps] in
 * fixed point with 22 fractional bits, zero past count (resize.py restates Pillow's arithmetic). Downscaling only:
 * H_out <= H and W_out <= W. Null pointers, empty sizes, a larger output, an unknown kind and windows or weights
 * outside their ranges are DSS_ERR_BAD_ARG; B or H_out above 65535 is DSS_ERR_UNSUPPORTED. All checks run before any
 * device work. Workspace: dss_resize_workspace_bytes(H_out, W_out, taps_y, taps_x). */
enum { DSS_RESIZE_U8 = 0, DSS_RESIZE_UNIT_F32 = 1 };
size_t dss_resize_workspace_bytes(int H_out, int W_out, int taps_y, int taps_x);
int dss_resize_bilinear(const uint8_t* images, int B, int H, int W, int H_out, int W_out, const int* bounds_y_host,
                        const int* weights_y_host, int taps_y, const int* bounds_x_host, const int* weights_x_host,
                        int taps_x, int kind, void* out, void* ws, size_t ws_bytes, dss_stream_t stream);

/* Segmentation evaluation counts of a ragged batch of (prediction, target) uint8 label maps (the pixel loops of the
 * reference's semantic-segmentation/eval.py and object-segmentation/main.py). images_host [B, DSS_SEGEVAL_FIELDS] int64
 * per image: {pred_offset, pred_h, pred_w, target_offset, target_h, target_w, top, left, h, w, block_h, block_w,
 * table_offset}: maps are row-major at byte offsets of preds / targets (device); output pixel (y, x), 0 <= y < h,
 * 0 <= x < w, reads target (top + y, left + x) and prediction (rows[y], cols[x]), where tables_host (int32, host) holds
 * at table_offset rows_in[h], rows_out[h], cols_in[w], cols_out[w]: pixels with y < block_h and x < block_w use the
 * _in halves, all others the _out halves.
 *   DSS_SEGEVAL_SEMANTIC: target 255 is ignored; counts [256, num_classes + 1] int64 (device) += pixels per
 *     (prediction value, target bin), bin = target if target < num_classes else num_classes. 2 <= num_classes + 1
 *     <= 64, else DSS_ERR_UNSUPPORTED.
 *   DSS_SEGEVAL_BINARY: prediction != 0 against target >= 128; counts [B, 4] int64 (device) = {TP, FP, FN, TN}.
 * Integer arithmetic only: an image gets the same counts alone or in any batch. Table entries outside the prediction,
 * crops outside the target, offsets outside the buffers, maps of 2^31 cells or rows wider than 2^24 pixels:
 * DSS_ERR_UNSUPPORTED. Workspace: dss_segeval_workspace_bytes(B, table entries). */
#define DSS_SEGEVAL_FIELDS 13
enum { DSS_SEGEVAL_SEMANTIC = 0, DSS_SEGEVAL_BINARY = 1 };
size_t dss_segeval_workspace_bytes(int B, long long table_entries);
int dss_segeval_counts(const uint8_t* preds, long long preds_bytes, const uint8_t* targets, long long targets_bytes,
                       const long long* images_host, int B, const int* tables_host, long long table_entries, int mode,
                       int num_classes, long long* counts, void* ws, size_t ws_bytes, dss_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DSS_B200_H */
