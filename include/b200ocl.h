/*
 * b200ocl.h -- C ABI of libb200ocl.so: the replay-step hot path of
 * RaptorMai/online-continual-learning as hand-written sm_90a CUDA.
 *
 * The reference is pure Python/PyTorch and has no FFI of its own (SURVEY.md
 * section 8b); each entry point below therefore names the reference *Python*
 * interface whose arithmetic it replaces (file:line under /root/reference).
 * INTEGRATION.md shows the ctypes stub a reference maintainer would add.
 *
 * Conventions
 *   - plain C: pointers, sizes, a cudaStream_t passed as void*; no torch types;
 *   - every pointer is a BORROWED DEVICE pointer, contiguous row-major, owned by
 *     the caller and kept alive until the stream work completes;
 *   - fp32 data, int64 labels/indices (the reference's dtypes, data_utils.py:41,
 *     buffer.py:23);
 *   - no hidden allocation: scratch is caller-provided, sized by the matching
 *     *_workspace_bytes() query (must be 256-byte aligned); kernel attributes are cached per device;
 *   - every function returns 0 on success or a B200OCL_E* code; the message is
 *     available from b200ocl_last_error() (thread-local); nothing throws;
 *   - launches are asynchronous on `stream`; no function synchronises.
 */
#ifndef B200OCL_H_
#define B200OCL_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200OCL_OK 0
#define B200OCL_EINVAL 1      /* bad argument (null pointer, negative size, ...)   */
#define B200OCL_EUNSUPPORTED 2 /* shape outside what the kernels cover            */
#define B200OCL_EWORKSPACE 3  /* workspace too small or misaligned               */
#define B200OCL_ECUDA 4       /* a CUDA runtime call failed                      */

#define B200OCL_KNN_MAX_CAND 1024 /* candidates the fused (register-sorted) kNN-SV kernel takes */
#define B200OCL_KNN_MAX_CAND_LARGE 262144 /* beyond that: the scratch-line kernel (knn_sv_large.cu), same results */

const char* b200ocl_last_error(void);
int b200ocl_version(void);
/* Number of kernel launches issued through this library since load (bench.py reports it). */
uint64_t b200ocl_launch_count(void);
/* The SM count the current device's launches are planned for: its multiprocessor count, or B200OCL_SM_COUNT when
 * that is set to a smaller positive value (read once per device per process). */
int b200ocl_sm_count(void);
/* Optional per-launch device timing for bench.py's roofline: between begin and end every launch of
 * this library is bracketed by CUDA events on its launch stream and accumulated per kernel class
 * together with its algorithmic work (FLOPs for conv/wgrad classes, bytes otherwise).
 * profile_end synchronises the device and returns the number of classes. */
void b200ocl_profile_begin(void);
int b200ocl_profile_end(void);
int b200ocl_profile_get(int k, char* name, int name_len, double* ms, int* launches, double* work);

/* ---------------------------------------------------------------- kNN Shapley values
 * Replaces compute_knn_sv minus its network forward: sorted_cand_ind +
 * euclidean_distance + the Shapley recurrence + scatter (utils/buffer/aser_utils.py:29-59,
 * 94-116; utils/utils.py:93-95) and the row reductions its callers take
 * (aser_retrieve.py:79,82,86; aser_update.py:80), in ONE kernel.
 *   eval_f [E,d] f32, eval_y [E] i64, cand_f [C,d] f32, cand_y [C] i64, k neighbours.
 * Outputs (each nullable): sv [E,C] Shapley matrix in candidate order; col_sum /
 * col_max / col_min [C] reductions over eval rows.  Distance is the squared L2 in
 * direct-difference form; equal distances rank lowest candidate index first.
 * Reductions are deterministic (fixed-order, no float atomics).  C <= 262144 (one fused launch up to 1024
 * candidates, the scratch-line kernel beyond; the workspace query covers both). */
size_t b200ocl_knn_sv_workspace_bytes(int E, int C, int d);
int b200ocl_knn_sv(const float* eval_f, const int64_t* eval_y, const float* cand_f, const int64_t* cand_y,
                   int E, int C, int d, int k,
                   float* sv, float* col_sum, float* col_max, float* col_min,
                   void* workspace, size_t workspace_bytes, void* stream);

/* The launch b200ocl_knn_sv makes for E eval rows, C candidates and width d on a GPU with sms SMs (0: the current
 * device), with aligned != 0 when eval_f and cand_f are 16-byte aligned and want_red != 0 when any column reduction is
 * asked for.  family: the fused kernel (C <= 1024) with kpl keys per lane, te eval rows per tile and, for kpl = 32 /
 * te = 16, the wide phase 1 (wide = 1) or the row-tiled one; or the scratch-line kernel (C > 1024) over cpad keys per
 * row, sorted in shared-memory blocks of block_keys keys with far_stages compare stages through global memory.
 * grid: CTAs; tiles_per_cta: the most eval tiles (fused) or rows (large) one CTA takes; smem_bytes: dynamic shared
 * memory, smem_limit: the limit the launcher raises the kernel to; part_bytes: the column partials the launch writes
 * (at workspace offset 256); key_offset / key_bytes: the large kernel's key lines; workspace_bytes: what
 * b200ocl_knn_sv_workspace_bytes returns on a GPU with sms SMs.  Host only, launches nothing; exists so that tests can
 * check which kernels a shape reaches and that every plan fits on any SM count. */
#define B200OCL_KNN_FUSED 0
#define B200OCL_KNN_LARGE 1
typedef struct {
  int family;
  int kpl, te, wide;
  int cpad, block_keys, far_stages;
  int grid, n_tiles, tiles_per_cta;
  size_t smem_bytes, smem_limit, part_bytes, key_offset, key_bytes, workspace_bytes;
  int sms;
} b200ocl_knn_launch;
int b200ocl_knn_sv_plan(int E, int C, int d, int aligned, int want_red, int sms, b200ocl_knn_launch* out);

/* ---------------------------------------------------------------- ranking
 * score[i] = a[i]*sa + (b ? b[i]*sb : 0); idx_out[0..n_out) = positions of the n_out
 * largest scores in descending order, ties lowest index first (the reference's
 * sv.argsort(descending=True)[:n], aser_retrieve.py:82-91, aser_update.py:80-93;
 * MIR's scores.sort(descending=True)[1][:n], mir_retrieve.py:28-29).  n <= 4096.
 * score_out [n] nullable. */
int b200ocl_rank_desc(const float* a, float sa, const float* b, float sb, int n,
                      int64_t* idx_out, int n_out, float* score_out, void* stream);

/* ---------------------------------------------------------------- SupCon loss
 * Replaces SupConLoss.forward (+ its autograd backward), all-views-anchor mode
 * (utils/loss.py:19-96): features [B,V,d] f32, labels [B] i64 -> loss[1] and, when
 * dfeats != NULL, dL/dfeatures [B,V,d].  d <= 1024.
 * An anchor without positives (V = 1, a class with one sample) makes the loss NaN, as in the reference (loss.py:90);
 * the gradient stays finite: that anchor's positive term is taken as 0, so it contributes the gradient of lse_i / A
 * (its log-sum-exp over the other anchors) and nothing else.  Autograd on the reference gives NaN everywhere. */
size_t b200ocl_supcon_workspace_bytes(int B, int V, int d);
int b200ocl_supcon(const float* feats, const int64_t* labels, int B, int V, int d, float temperature,
                   float* loss, float* dfeats, void* workspace, size_t workspace_bytes, void* stream);

/* The launch b200ocl_supcon makes for B x V anchors of width d on a GPU with sms SMs (0: the current device), with
 * aligned != 0 when feats (and dfeats, if given) are 16-byte aligned.  family: the fused kernel with the whole
 * contrast set resident in shared memory (rm x rn = 1 x 4), with a two-slot ring of 16-anchor units (1 x 2) or of
 * 64-anchor units (4 x 4), all with nc = ceil(d / 64) float4 columns per thread; or the stats kernel + grad kernel
 * with dch = 4/8/16/32 columns per lane.  grid: CTAs of the launch (each of the fallback's two); n_units: anchor blocks
 * (the entries of the workspace's loss partials it writes); units_per_cta: the most units one CTA takes; smem_bytes:
 * dynamic shared memory of the largest launch, smem_limit: the limit the launcher raises the kernel to; tx_bytes: the
 * largest single mbarrier transaction a fused launch expects (0 for the fallback).  Host only, launches nothing; exists
 * so that tests can check which kernels a shape reaches and that every plan fits on any SM count. */
#define B200OCL_SUPCON_RESIDENT 0
#define B200OCL_SUPCON_RING16 1
#define B200OCL_SUPCON_RING64 2
#define B200OCL_SUPCON_FALLBACK 3
typedef struct {
  int family;
  int rm, rn, nc, dch;
  int grid, n_units, units_per_cta;
  size_t smem_bytes, smem_limit, tx_bytes;
  int sms;
} b200ocl_supcon_launch;
int b200ocl_supcon_plan(int B, int V, int d, int aligned, int sms, b200ocl_supcon_launch* out);

/* ---------------------------------------------------------------- buffer rows
 * dst[i,:] = src[idx[i],:]  /  dst[idx[i],:] = src[i,:]   rows of row_bytes bytes
 * (buffer_img[indices], buffer_img[idx] = x: buffer_utils.py:19-21,115-116;
 * reservoir_update.py:59-60; aser_update.py:111-112).  row_bytes % 4 == 0.
 * Scatter with duplicate idx is undefined, as in the reference's index_put. */
int b200ocl_gather_rows(const void* src, const int64_t* idx, int n_rows, size_t row_bytes, void* dst, void* stream);
int b200ocl_scatter_rows(const void* src, const int64_t* idx, int n_rows, size_t row_bytes, void* dst, void* stream);

/* ---------------------------------------------------------------- evaluate() (agents/base.py:118-175)
 * Nearest-class-mean classification on encoder features.  class_means: for each class_ids[k] the normalised mean
 * of the normalised features of the samples with that label (base.py:121-141); counts[k] == 0 leaves means[k]
 * untouched (the reference draws a random vector there).  classify: pred[b] = class_ids[arg-min_k ||f_b/||f_b|| -
 * means[k]||^2] (first minimum), *n_correct += #(pred == truth) (truth / pred / n_correct nullable).
 * linear_argmax: pred[b] = arg-max_c (feats[b] . weight[c] + bias[c]) -- the classifier branch (base.py:172-175).
 * class_means takes d <= B200OCL_NET_MAX_DIM; classify and linear_argmax take any d. */
int b200ocl_ncm_class_means(const float* feats, const int64_t* labels, int n, int d, const int64_t* class_ids, int K,
                            float* means, int* counts, void* stream);
int b200ocl_ncm_classify(const float* feats, int B, int d, const float* means, int K, const int64_t* class_ids,
                         const int64_t* truth, int64_t* pred, uint64_t* n_correct, void* stream);
int b200ocl_linear_argmax(const float* feats, int B, int d, const float* weight, const float* bias, int C,
                          const int64_t* truth, int64_t* pred, uint64_t* n_correct, void* stream);
/* linear_argmax with the error analysis of base.py:144-226 (--error_analysis): the same pred and *n_correct, bit for
 * bit, and per row b, with p the predicted class: pred_task[b] = class_task[p] (-1: unmapped); set_sums[2b+j] = the
 * row's logits f.w_c + b_c summed in fp64, in class order, over the classes c with bit j of class_sets[c] (bit 0: the
 * last task's labels, bit 1: the older labels without them); counts[0..2] += 1 when truth[b] != p and p has bit 0 /
 * bit 1 / neither; counts[3] += 1 when class_task[p] == -1.  class_sets [C] uint8, class_task [C]; truth, class_sets,
 * class_task, pred_task, set_sums and counts are required, pred and n_correct nullable.
 * rows_mean: out[0] = mean of weight[rows] ([n, d] elements), out[1] = mean of bias[rows], each summed in fp64 and
 * rounded to fp32 once; n == 0 gives NaN.  rows must lie in [0, C). */
int b200ocl_linear_argmax_ea(const float* feats, int B, int d, const float* weight, const float* bias, int C,
                             const int64_t* truth, const uint8_t* class_sets, const int64_t* class_task, int64_t* pred,
                             uint64_t* n_correct, int64_t* pred_task, double* set_sums, uint64_t* counts, void* stream);
int b200ocl_rows_mean(const float* weight, const float* bias, int C, int d, const int64_t* rows, int n, float* out,
                      void* stream);
/* PCR's evaluation (Lin et al., CVPR 2023): pred[b] = arg-max_c <f_b / (||f_b|| + eps), w_c / (||w_c|| + eps)>, eps =
 * 1e-6, over the C rows of weight (the classifier's; no bias); the first maximum wins.  *n_correct += #(pred == truth).
 * The classify body of b200ocl_linear_argmax, one warp per row; truth, pred and n_correct nullable. */
int b200ocl_cosine_argmax(const float* feats, int B, int d, const float* weight, int C, const int64_t* truth,
                          int64_t* pred, uint64_t* n_correct, void* stream);

/* The network's linear layer on its own: y [N,out] = x [N,in] . W[out,in]^T + b (relu != 0: then ReLU), the kernel the
 * classifier and projection heads run.  Each output sums its lane-strided products in a fixed order (no atomics).
 * 1 <= in <= B200OCL_NET_MAX_DIM. */
int b200ocl_linear_fwd(const float* x, const float* W, const float* b, float* y, int N, int in, int out, int relu,
                       void* stream);

/* A-GEM gradient projection (agents/agem.py:60-80) on flat gradient arenas: out = g - (g.g_ref / g_ref.g_ref) g_ref if
 * g.g_ref < 0, else out = g (out may alias g_ref or g).  dots_out (nullable, [2] f32) receives g.g_ref and g_ref.g_ref.
 * Deterministic: fp64 partials reduced in CTA order. */
size_t b200ocl_agem_project_workspace_bytes(void);
int b200ocl_agem_project(const float* g, const float* g_ref, float* out, size_t n, float* dots_out, void* workspace,
                         size_t workspace_bytes, void* stream);

/* GSS-greedy scores (utils/buffer/gss_greedy_update.py:84,120 with cosine_similarity of buffer_utils.py:50-55): cosine
 * similarity of the flat gradient g [n] with each of the K <= 64 stored gradients mem_grads [K,n] (cos_out [K], nullable)
 * and their maximum (max_out [1], nullable).  Deterministic fp64 partials. */
size_t b200ocl_grad_cosine_workspace_bytes(int K);
int b200ocl_grad_cosine(const float* mem_grads, const float* g, int K, size_t n, float* cos_out, float* max_out, void* workspace,
                        size_t workspace_bytes, void* stream);

/* GEM's projection (Lopez-Paz & Ranzato, NeurIPS 2017; the authors' project2cone2 with margin = memory_strength) on
 * flat gradient arenas: the t task gradients G [t,n] (row k at G + k * pitch, pitch >= n elements) and the stream
 * gradient g [n].  P = G G^T and q = G g in fp64 (every product of two floats exact, fp64 sums in a fixed order);
 * *flag_out = (min_k q_k < 0).  When the flag is set, v [t] (fp64, v_out) minimises 1/2 v^T (P + eps I) v + q^T v subject
 * to v_k >= margin, solved exactly by an active-set method with a Cholesky solve of the free block per iteration, and
 * out[i] = fl32((double)g[i] + sum_k v_k (double)G[k,i]) summed in k order (out may alias g).  When it is clear, v_out
 * is 0 and out is neither read nor written.  A QP that exhausts the kernel's iteration bound sets *err_flag = 1
 * (nullable, never cleared) and leaves its last feasible iterate in v_out.  kkt_out (nullable, [4] fp64): the primal,
 * dual and complementarity residuals of w = v - margin and the number of Cholesky solves.  Three launches (Gram, QP,
 * projection), no host synchronisation, no floating-point atomics: bit-identical on repeat at a given SM count.
 * B200OCL_EINVAL for a null pointer, t or n < 1, pitch < n, a margin that is negative or not finite or an eps that is
 * not finite and positive; B200OCL_EUNSUPPORTED for t > 64. */
size_t b200ocl_gem_project_workspace_bytes(int t, size_t n);
int b200ocl_gem_project(const float* G, size_t pitch, int t, const float* g, float* out, size_t n, double margin,
                        double eps, double* v_out, int* flag_out, int* err_flag, double* kkt_out, void* workspace,
                        size_t workspace_bytes, void* stream);

/* The launches b200ocl_gem_project makes for t task gradients of length n on a GPU with sms SMs (0: the current
 * device).  rows = t + 1 (the Gram is taken of [G; g]), padded to rows_padded = 4 * row_blocks; each of the
 * block_pairs = row_blocks (row_blocks + 1) / 2 upper-triangle 4 x 4 blocks of pairs is formed by `lanes` threads over
 * interleaved columns of each staged tile of tile_cols columns (row stride tile_stride floats, two stages; smem_bytes of
 * dynamic shared memory).  grid CTAs, each owning chunk consecutive columns (tiles_per_cta tiles; the last CTA fewer,
 * none without columns), write pairs = rows (rows + 1) / 2 fp64 partials each: part_bytes, inside workspace_bytes.  The
 * projection runs proj_grid CTAs of 256 threads.  Host only, launches nothing; exists so that tests can check every
 * plan on any SM count.  B200OCL_EINVAL unless 1 <= t <= 64 and n >= 1. */
typedef struct {
  int rows, rows_padded, row_blocks, block_pairs, lanes, tile_cols, tile_stride, pairs;
  int grid, tiles_per_cta, proj_grid, sms;
  size_t chunk, smem_bytes, part_bytes, workspace_bytes;
} b200ocl_gem_launch;
int b200ocl_gem_plan(int t, size_t n, int sms, b200ocl_gem_launch* out);

/* Stream feeder (continuum/data_utils.py:38-54: ToTensor on every sample + DataLoader shuffle): dst[i] = image
 * src[perm[i]] converted uint8 HWC -> fp32 CHW in [0,1] with an IEEE division by 255 (bit-identical to the
 * reference's CPU ToTensor).  perm may be NULL (identity).  h*w*3 % 4 == 0. */
int b200ocl_stream_prepare(const uint8_t* src_hwc, const int64_t* perm, int n, int h, int w, float* dst_chw, void* stream);

/* Stream feeder for the non-stationary tasks (continuum/non_stationary.py:9-124 hand the agents float64 HWC images in
 * [0,1]; continuum/data_utils.py:38-54 applies ToTensor, a transpose only for float input, then .float()): dst[i] =
 * image src[perm[i]] converted float64 HWC -> fp32 CHW, rounded to nearest even as the CPU's conversion does
 * (subnormals kept, overflow to inf, NaN kept with its sign and payload).  perm may be NULL (identity).  src 8-byte
 * aligned; offsets are 64-bit. */
int b200ocl_stream_prepare_f64(const double* src_hwc, const int64_t* perm, int n, int h, int w, float* dst_chw,
                               void* stream);

/* ASER memory replacement on the device (reference utils/buffer/aser_update.py:88-112: current samples ranked
 * inside the first n_cand_buf places of the descending SV ranking replace, pairwise in rank order, the buffered
 * candidates ranked below).  order[n_total] ranks positions of [buffered candidates | current batch];
 * cand_slot[n_cand_buf] are the candidates' buffer slots.  Moves image rows and labels; pairs_out (nullable,
 * [1 + 2*n_cur] int64 = count, src positions, dst slots, -1 padded) lets the host mirror follow asynchronously. */
int b200ocl_aser_replace(const int64_t* order, int n_total, int n_cand_buf, const int64_t* cand_slot, const void* cur_x,
                         const int64_t* cur_y, int n_cur, size_t row_bytes, void* buffer_img, int64_t* buffer_label,
                         int64_t* pairs_out, void* stream);

/* ---------------------------------------------------------------- SGD
 * p -= lr * (g + wd * p) over a flat arena of n floats: torch.optim.SGD without
 * momentum (utils/setup_elements.py:73-75) and MIR's virtual step
 * theta' = theta - lr*g when out != p (mir_retrieve.py:43-46).  out may alias p. */
int b200ocl_sgd_step(const float* p, const float* g, float* out, size_t n, float lr, float wd, void* stream);


/* ---------------------------------------------------------------- Reduced-ResNet18 engine
 * The only network on the replay-step path (models/resnet.py:14-37,69-116 BasicBlock ResNet
 * with nf=20; :140-168 SupConResNet; per-dataset classifier, utils/setup_elements.py:46-68).
 *   head: 0 classifier (logits [N,num_classes]); 1/2/3 SupConResNet with 'linear'/'mlp'/'None'
 *   head (L2-normalised projection [N,feat_dim]).
 * State = flat arenas owned by the caller:
 *   params / grads  every learnable tensor in torch parameters() order and torch layout
 *                   (a reference nn.Module can alias its Parameters onto it);
 *   packed          kernel-layout copies of the conv weights, refreshed by b200ocl_net_pack /
 *                   b200ocl_net_sgd_step;
 *   bn_stats        per BatchNorm2d running_mean[c], running_var[c] in module order;
 *   bn_tracked      num_batches_tracked per BatchNorm2d.
 * Images are fp32 NCHW [N,3,H,W] exactly as the reference feeds them (no normalisation,
 * setup_elements.py:29-43); activations are NHWC inside the engine. */
#define B200OCL_NET_MAX_DIM 4096 /* largest flattened feature size (dim_in) and output size (out_dim) of a network */

typedef struct {
  int in_h, in_w;      /* 32x32 CIFAR, 84x84 Mini-ImageNet, 128x128 CORe50 (setup_elements.py:11-17) */
  int nf;              /* 20 (Reduced_ResNet18, resnet.py:112-116) */
  int num_classes;     /* classifier width when head == 0 */
  int head;            /* 0 classifier | 1 linear | 2 mlp | 3 none */
  int feat_dim;        /* SupCon projection size (128) */
} b200ocl_net_desc;

typedef struct {
  float* params;
  float* grads;
  float* packed;
  float* bn_stats;
  int64_t* bn_tracked;
} b200ocl_net_state;

/* Sizes (in elements) of the arenas and basic shape facts.  A description whose dim_in or out_dim exceeds
 * B200OCL_NET_MAX_DIM (160 dim_in at 32x32, 640 at 84x84, 2560 at 128x128) is refused with B200OCL_EUNSUPPORTED. */
typedef struct {
  size_t n_params, n_packed, n_bn_stats;
  int n_bn, n_tensors, dim_in, out_dim;
} b200ocl_net_info;
int b200ocl_net_query(const b200ocl_net_desc* desc, b200ocl_net_info* info);
/* i-th parameter tensor in parameters() order: offset/numel in the arena, has_grad = 0 for the
 * SupConResNet encoder classifier that never receives a gradient. */
int b200ocl_net_tensor(const b200ocl_net_desc* desc, int i, size_t* offset, size_t* numel, int* has_grad);

/* packed <- params (call after loading weights). */
int b200ocl_net_pack(const b200ocl_net_desc* desc, const b200ocl_net_state* st, void* stream);

/* Batch limit of every pass below (features_eval, the forwards, backward): N times the largest activation of one image
 * must stay within INT_MAX elements, the range the kernels' 32-bit pixel and element indices cover (N <= 104857 at
 * 32x32, 15217 at 84x84, 6553 at 128x128).  A larger N is refused with B200OCL_EUNSUPPORTED before anything launches. */

/* model.eval(); model.features(x) under no_grad (utils/utils.py:45-90): feat [N,dim_in]. */
size_t b200ocl_net_eval_workspace_bytes(const b200ocl_net_desc* desc, int N);
int b200ocl_net_features_eval(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, int N,
                              float* feat, void* workspace, size_t workspace_bytes, void* stream);

/* model.train(); out = model.forward(x): batch-statistics BN, running stats and
 * num_batches_tracked updated (momentum 0.1, unbiased variance); activations are kept in
 * `workspace` for b200ocl_net_backward.  out [N,out_dim]. */
size_t b200ocl_net_train_workspace_bytes(const b200ocl_net_desc* desc, int N);

/* Where a train workspace of N images keeps conv layer `layer`'s tensors (layers in BatchNorm2d module order) and the
 * launches b200ocl_net_backward makes for it on the current device.  Byte offsets are from the workspace start:
 * z / a the raw / activated output [N,hout,wout,cout] (a block's conv2 slot holds the block output), mean / invstd the
 * saved BN statistics [cout], feat / hid / proj the head tensors [N,dim_in] / [N,dim_in] / [N,out_dim] (the same for every
 * layer), wg_part the start of the weight-gradient partials and wg_layer this layer's wgrad_splits partials of
 * [ks*ks*cin][cout] floats.  bn_fused: 1 fused BN backward, 0 reduce + apply, over bn_grid CTAs.  wgrad_kernel: 0 stem,
 * 1 wgmma (wgrad_tc.cu), 2 fp32.  Host only, launches nothing; exists so that tests can read what the engine's forward
 * left behind and check which launch geometries a batch size reaches.  B200OCL_EINVAL for N < 1 or a layer out of range. */
typedef struct {
  size_t bytes;
  size_t z, a, mean, invstd;
  size_t feat, hid, proj;
  size_t wg_part, wg_layer;
  int cin, cout, ks, stride, hout, wout;
  int bn_fused, bn_grid;
  int wgrad_kernel, wgrad_splits;
  int sms;
} b200ocl_net_ws_layout;
int b200ocl_net_train_ws_layout(const b200ocl_net_desc* desc, int N, int layer, b200ocl_net_ws_layout* out);

/* The convolution kernel one launch runs, with its template parameters and grid.  kernel: 0 stem, 1 wgmma fed from a
 * halo strip (conv_tcp.cu, template nt), 2 wgmma with im2col tiles (conv_tc.cu, nt), 3 patch (bn, pt), 4 tiled (bn, pt),
 * 5 k-split (pt, kwarps), -1 none covers it.  th / tw / ti: the patch kernel's spatial tile.  stat_bytes: the batch-statistics
 * partials a train-mode launch writes (grid_x * channels * 2 doubles; 0 for the other passes); stat_region: the bytes
 * the workspace keeps for them.  sms: the SM count the plan is for.  tp_ps / tp_bs: the halo-strip kernel's patch
 * stages and weight ring depth (0 for the other kernels). */
typedef struct {
  int kernel;
  int nt, bn, pt, kwarps;
  int grid_x, grid_y;
  int th, tw, ti;
  size_t stat_bytes, stat_region;
  int sms;
  int tp_ps, tp_bs;
} b200ocl_conv_geom;
/* The launch of conv layer `layer` (BatchNorm2d module order) over N images in pass 0 train-mode forward, 1 eval-mode
 * forward or 2 data gradient (layers >= 1), on a GPU with sms SMs (0: the current device), and the statistics region of
 * the train workspace of N images planned for that SM count.  Host only, launches nothing; exists so that tests can
 * check which kernels a batch size reaches and that the workspace holds what they write on any SM count. */
int b200ocl_net_conv_geom(const b200ocl_net_desc* desc, int N, int layer, int pass, int sms, b200ocl_conv_geom* out);

int b200ocl_net_forward_train(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, int N,
                              float* out, void* workspace, size_t workspace_bytes, void* stream);

/* model.eval(); out = model.forward(x) WITH activations kept for a backward pass (utils/buffer/gss_greedy_update.py:16,
 * 80-83, 118-120: GSS-greedy differentiates the network in eval mode): BatchNorm uses the running statistics, nothing is
 * updated.  Its backward is b200ocl_net_backward with bit 1 of `accumulate` set. */
int b200ocl_net_forward_evalgrad(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, int N,
                                 float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Train-mode forward with DEFERRED running statistics: identical outputs and saved activations, but the BatchNorm running
 * statistics (and num_batches_tracked) are not touched; the batch statistics of every BN stay in `workspace` until
 * b200ocl_net_apply_running_stats applies them (running = 0.9 running + 0.1 batch, tracked += 1).  The train-mode passes of
 * one replay step (exp_replay.py:40,62,84; scr.py:55) only interact through those statistics, so a caller may run them
 * concurrently on different streams and then apply their statistics in the reference's order. */
int b200ocl_net_forward_train_deferred(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, int N,
                                       float* out, void* workspace, size_t workspace_bytes, void* stream);
int b200ocl_net_apply_running_stats(const b200ocl_net_desc* desc, const b200ocl_net_state* st, int N, void* workspace,
                                    size_t workspace_bytes, void* stream);

/* loss.backward() for the forward kept in `workspace` (same x): dout [N,out_dim] -> st->grads
 * (overwritten, or added to when accumulate != 0 -- exp_replay.py:55,77 accumulate two
 * backward passes before one opt.step()).  accumulate bit 1 (value 2): the forward was b200ocl_net_forward_evalgrad.
 * accumulate bit 2 (value 4): the pass starts from the encoder features: dout is dL/dfeatures [N,dim_in] (the `feat` the
 * forward kept, b200ocl_net_train_ws_layout), the head's backward is skipped and the head's gradient entries are left as
 * they are; bit 0 still selects overwriting or adding for every other entry (PCR's loss writes the classifier's own).
 * The weight-gradient launches run on a helper stream that is forked from / joined into `stream` with events (captured
 * as parallel branches when `stream` is being captured into a CUDA graph); the helper stream and its four events (one set per
 * caller stream, at most four caller streams per device) are the one piece of state the library creates itself, on the first call (B200OCL_WG_ASYNC=0: everything on `stream`). */
int b200ocl_net_backward(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, const float* dout,
                         int N, void* workspace, size_t workspace_bytes, int accumulate, void* stream);

/* opt.step() of torch.optim.SGD without momentum over every tensor that has a gradient
 * (setup_elements.py:73-75), then refresh `packed`.  With dst != NULL the updated weights go
 * to dst->params / dst->packed instead (MIR's virtual step theta - lr*grad on a copy,
 * mir_retrieve.py:34-47); tensors without gradient are copied. */
int b200ocl_net_sgd_step(const b200ocl_net_desc* desc, const b200ocl_net_state* st, float lr, float weight_decay,
                         const b200ocl_net_state* dst, void* stream);

/* GDumb's step (agents/gdumb.py:82-83): torch.nn.utils.clip_grad_norm_(parameters, max_norm) then opt.step().
 * Launch 1 takes the L2 norm of every tensor that has a gradient (the tensors b200ocl_net_sgd_step skips are left out)
 * and the coefficient coef = min(max_norm / (norm + 1e-6), 1) in fp32, rounded as torch/nn/utils/clip_grad.py
 * (_clip_grads_with_norm_) rounds it: the division is Tensor.__rdiv__, (norm + 1e-6).reciprocal() * max_norm.  The
 * norm comes from per-CTA fp64 partials reduced in CTA order by the last CTA, no floating-point atomics, so repeated
 * launches are bit-identical.  Launch 2 writes g * coef back to the gradient arena (torch scales
 * .grad in place, and by coef = 1 too) and applies the SGD update of b200ocl_net_sgd_step with it; then `packed` is
 * refreshed.  The coefficient stays on the device.  norm_out (nullable, device): the norm before clipping.  workspace:
 * b200ocl_net_sgd_step_clipped_workspace_bytes(desc) bytes of device memory, no initial contents needed. */
size_t b200ocl_net_sgd_step_clipped_workspace_bytes(const b200ocl_net_desc* desc);
int b200ocl_net_sgd_step_clipped(const b200ocl_net_desc* desc, const b200ocl_net_state* st, float lr,
                                 float weight_decay, float max_norm, float* norm_out, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* EWC++ state (agents/ewc_pp.py): four fp32 device arenas in the parameter arena's layout (n_params floats each):
 * running_fisher, tmp_fisher, normalized_fisher and prev_params. */
typedef struct {
  float* running;
  float* tmp;
  float* normalized;
  float* prev;
} b200ocl_ewc_state;

#define B200OCL_EWC_PENALTY 1 /* the penalty lambda * sum F * (p - prev)^2 is in the loss (from the second call on) */
#define B200OCL_EWC_EMA 2     /* update_running_fisher fires before this step */

/* One EWC++ step after the backward pass (ewc_pp.py:40-62), one launch and one pass per element, then `packed` is
 * refreshed as by b200ocl_net_sgd_step.  In order, each with torch's separate fp32 roundings (no fma):
 *   EMA:      running = ema_keep * running + ema_add * tmp, then tmp = 0, with ema_keep = fp32(1 - alpha) and
 *             ema_add = fp32(1/fua * alpha) formed in double by the caller;
 *   PENALTY:  g += (up * normalized) * (2 * (p - prev)), written back to the gradient arena; `up` is the gradient
 *             autograd delivers to the regulariser: fp32(lambda), times the kd_trick / kd_trick_star mixing weights
 *             in fp32 from the outermost inward;
 *   always:   tmp += g * g, then the SGD update of b200ocl_net_sgd_step with g.
 * The tensors b200ocl_net_sgd_step skips are left untouched in every arena.  penalty_out (nullable, device): with
 * PENALTY sum normalized * (p - prev)^2 over the pre-step weights, from per-CTA fp64 partials added in CTA order by
 * the last CTA (no floating-point atomics: repeated launches are bit-identical); 0 without.  workspace:
 * b200ocl_net_sgd_step_ewc_workspace_bytes(desc) bytes of device memory, no initial contents needed. */
size_t b200ocl_net_sgd_step_ewc_workspace_bytes(const b200ocl_net_desc* desc);
int b200ocl_net_sgd_step_ewc(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const b200ocl_ewc_state* ewc,
                             float lr, float weight_decay, float up, int flags, float ema_keep, float ema_add,
                             float* penalty_out, void* workspace, size_t workspace_bytes, void* stream);

/* The end of an EWC++ train_learner call (ewc_pp.py:71-78), two launches, nothing read back: prev = params, then
 * normalized = (running - mn) / ((mx - mn) + 1e-32) with mn / mx the min / max of running over every tensor, in fp32
 * with an IEEE division.  The tensors b200ocl_net_sgd_step skips are left out and untouched.  workspace:
 * b200ocl_ewc_consolidate_workspace_bytes(desc) bytes, no initial contents needed. */
/* ---------------------------------------------------------------- Adam
 * torch.optim.Adam (utils/setup_elements.py:76-78, --optimizer Adam) with amsgrad, maximize and decoupled weight
 * decay off.  The scalars are what torch/optim/adam.py forms in double on the host for one step, each rounded to fp32
 * as torch converts it to the kernels' op-math type:
 *   step_size = -(lr / (1 - beta1**step)), bc2_sqrt = (1 - beta2**step)**0.5, bc2_sqrt_inv = 1 / bc2_sqrt (the
 *   reciprocal formed in double), eps, beta1_c = 1 - beta1, beta2, beta2_c = 1 - beta2, weight_decay;
 *   grad_scale: with B200OCL_ADAM_GRAD_SCALE the gradient is first replaced by g * grad_scale and written back: the
 *   review trick's p.grad.clone() / 10. (agents/base.py:84-88), which torch computes as g * fp32(1 / 10.).
 * Per element, each torch op with its own rounding (fma where torch's kernels contract):
 *   g' = g + wd * p (when wd != 0; g is not written), exp_avg.lerp_(g', beta1_c),
 *   exp_avg_sq = exp_avg_sq * beta2 + beta2_c * g' * g', denom = sqrt(exp_avg_sq) / bc2_sqrt + eps,
 *   p += step_size * exp_avg / denom.
 * B200OCL_ADAM_FOREACH: the division by bc2_sqrt is an IEEE division, as torch's default multi-tensor path
 * (_foreach_div_ by a scalar list) rounds it; without, it is a multiplication by bc2_sqrt_inv, as foreach=False
 * (CUDA Tensor / Python float) rounds it.  Either way the result is bit-identical to that path on the device. */
typedef struct {
  float step_size, bc2_sqrt, bc2_sqrt_inv, eps, beta1_c, beta2, beta2_c, weight_decay, grad_scale;
} b200ocl_adam_scalars;

#define B200OCL_ADAM_FOREACH 1
#define B200OCL_ADAM_GRAD_SCALE 2

/* One Adam step over flat fp32 buffers of n floats: p, exp_avg m and exp_avg_sq v updated in place, g read (written
 * only with B200OCL_ADAM_GRAD_SCALE).  One launch. */
int b200ocl_adam_step(float* p, float* g, float* m, float* v, size_t n, const b200ocl_adam_scalars* s, int flags,
                      void* stream);

/* Adam state of the network: exp_avg and exp_avg_sq in the parameter arena's layout (n_params floats each). */
typedef struct {
  float* exp_avg;
  float* exp_avg_sq;
} b200ocl_adam_state;

/* opt.step() of torch.optim.Adam over every tensor that has a gradient, one launch, then `packed` is refreshed as by
 * b200ocl_net_sgd_step.  The tensors b200ocl_net_sgd_step skips are left untouched in all four arenas (torch creates no
 * state for a parameter whose .grad is None). */
int b200ocl_net_adam_step(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const b200ocl_adam_state* adam,
                          const b200ocl_adam_scalars* s, int flags, void* stream);

/* The EWC++ step of b200ocl_net_sgd_step_ewc with the Adam update of b200ocl_net_adam_step in place of the SGD one, in
 * the same single launch: EMA, penalty gradient (written back), tmp += g * g, then Adam with that g.  adam_flags:
 * B200OCL_ADAM_FOREACH only.  workspace: b200ocl_net_sgd_step_ewc_workspace_bytes(desc) bytes. */
int b200ocl_net_adam_step_ewc(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const b200ocl_ewc_state* ewc,
                              const b200ocl_adam_state* adam, const b200ocl_adam_scalars* s, int adam_flags, float up,
                              int flags, float ema_keep, float ema_add, float* penalty_out, void* workspace,
                              size_t workspace_bytes, void* stream);

size_t b200ocl_ewc_consolidate_workspace_bytes(const b200ocl_net_desc* desc);
int b200ocl_ewc_consolidate(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const b200ocl_ewc_state* ewc,
                            void* workspace, size_t workspace_bytes, void* stream);

/* Mean cross-entropy (agents/base.py:95,113) over logits [N,C], labels [N]:
 * loss[1]; per_sample [N] (F.cross_entropy(reduction='none'), mir_retrieve.py:26-27), formed as
 * (max - logit[label]) + log sum exp(logits - max) so that a small loss at large logits keeps its relative precision;
 * dlogits [N,C] = d(mean CE)/dlogits; n_correct[1] = #(argmax == label) (ties lowest index).  Each output nullable.
 * A label outside [0,C) sets *err_flag = 1 (nullable, never cleared): its row's dlogits are 0, its per_sample is NaN,
 * and it adds nothing to loss (which still divides by N) or n_correct.  One CTA, fixed-order sums, no atomics:
 * repeated launches are bit-identical. */
int b200ocl_ce_loss(const float* logits, const int64_t* labels, int N, int C, float* loss, float* per_sample,
                    float* dlogits, int64_t* n_correct, int* err_flag, void* stream);

/* The training-trick criteria of agents/base.py:93-107 with the distillation term of utils/kd_manager.py:6-28 mixed in
 * (exp_replay.py:41-47, agem.py:40-46, lwf.py:38-40), over logits [N,C], labels [N], in one launch:
 *   loss[1] = w_ce * criterion + w_kd * kd, dlogits [N,C] = its gradient, n_correct[1] = #(argmax over all C == label)
 *   (ties lowest index).  Outputs nullable.
 * criterion by mode:
 *   B200OCL_CLS_CE         mean CE over all C columns;
 *   B200OCL_CLS_LABELS     labels trick: CE over the columns of the classes present in this batch (found on the device),
 *                          C <= B200OCL_CLS_MAX_C;
 *   B200OCL_CLS_SEPARATED  separated softmax: cols[n_cols] = old_labels ++ new_labels (duplicates allowed), log-softmax
 *                          over cols[0,n_old) and over cols[n_old,n_cols) separately, NLL at position pos_table[label]
 *                          (table_len entries, -1 = unmapped); only the target's segment gets a gradient, and a column
 *                          held at several positions sums their terms in position order.
 * kd = 4 * mean_i sum_c -softmax(teacher_ic/2) * log_softmax(logits_ic/2) (temperature 2) when teacher != NULL,
 * else kd = 0.  A label outside [0,C), or unmapped in the table, sets *err_flag = 1 (nullable, never cleared) and adds
 * nothing to the loss or gradient.  One CTA, fixed-order sums, no atomics: repeated launches are bit-identical. */
#define B200OCL_CLS_CE 0
#define B200OCL_CLS_LABELS 1
#define B200OCL_CLS_SEPARATED 2
#define B200OCL_CLS_MAX_C 12288
int b200ocl_cls_loss(const float* logits, const int64_t* labels, int N, int C, int mode, const int64_t* cols,
                     int n_cols, int n_old, const int64_t* pos_table, int table_len, const float* teacher, float w_ce,
                     float w_kd, float* loss, float* dlogits, int64_t* n_correct, int* err_flag, void* stream);

/* iCaRL's criterion (agents/icarl.py:42-62) over logits [N,C] in one launch:
 *   loss[1] = (1/N) sum_i sum_{j<K} [max(z,0) - z*t + log1p(exp(-|z|))]   (BCE with logits, summed over the K columns,
 *   averaged over the rows), dlogits [N,C] = (sigmoid(z) - t)/N for j < K and 0 for j >= K (nullable).
 * Targets t: rows i < n_stream are the stream batch, one-hot at pos_table[labels[i]] (pos_len entries, the
 * lbl_inv_map of this task); rows i >= n_stream are the memory rows, target 0; in the columns j < n_old the target is
 * sigmoid(teacher[i,j]) for every row (teacher [N,C], the previous model's logits; NULL only when n_old == 0).
 * Needs 0 <= n_old <= K <= C, K >= 1 and 0 <= n_stream <= N.  A stream label outside the table, or whose position lies
 * outside [n_old, K), sets *err_flag = 1 (nullable, never cleared) and its row adds nothing to the loss or gradient.
 * One CTA, fixed-order sums, no atomics: repeated launches are bit-identical. */
int b200ocl_icarl_loss(const float* logits, const float* teacher, const int64_t* labels, const int64_t* pos_table,
                       int pos_len, int N, int n_stream, int C, int K, int n_old, float* loss, float* dlogits,
                       int* err_flag, void* stream);

/* DER++'s logit-matching term (Buzzega et al., NeurIPS 2020) over the logits z [n,C] of a memory batch and the logit
 * memory mem [mem_rows,C], read in place through the int64 slot indices idx [n] (repeats allowed):
 *   loss[1] = alpha * sum (z - mem[idx])^2 / (n*C)      (alpha * F.mse_loss(z, mem[idx]), reduction 'mean'),
 *   dz [n,C] = alpha * 2 (z - mem[idx]) / (n*C).
 * Each difference and gradient element is formed in double and rounded once; the squares are summed in double in a
 * fixed order, with no atomics, so repeated launches are bit-identical.  One launch (one CTA) for every n >= 1, C >= 1.
 * A slot outside [0, mem_rows) sets *err_flag = 1 (nullable, never cleared): its row gets a zero gradient and adds
 * nothing to the loss (which still divides by n*C).  B200OCL_EINVAL for a null z, mem, idx, loss or dz, or a size < 1. */
int b200ocl_logit_mse(const float* z, const float* mem, int mem_rows, const int64_t* idx, int n, int C, double alpha,
                      float* loss, float* dz, int* err_flag, void* stream);

/* PCR's proxy-contrastive loss (Lin et al., CVPR 2023) over features F [R,d] with labels [R] (int64) and the proxies, the
 * classifier weight W [C,d]; eps = 1e-6, tau = temperature:
 *   u_i = F_i / (||F_i|| + eps),  v_c = W_c / (||W_c|| + eps),  g_ic = <u_i, v_c> / tau,
 *   n_c = #rows labelled c,  m_ic = n_c - [c = y_i],  Z_i = sum_c m_ic exp(g_ic),  l_i = log Z_i - g_{i,y_i},
 *   loss[1] = (1/R) sum_i l_i.
 * With p_ic = m_ic exp(g_ic) / Z_i: dL/du_i = (sum_c p_ic v_c - v_{y_i}) / (tau R) and dL/dv_c = sum_i (p_ic - [y_i = c])
 * u_i / (tau R), each taken through its normalisation (dx = g / (n + eps) - x <x, g> / (n (n + eps)^2), the second term
 * 0 at n = 0) into dfeats [R,d] and dproxies [C,d]; dbias [C] is zeroed (the bias never enters the loss).  dproxies and
 * dbias are meant to be the classifier's slices of the gradient arena.  A row of dproxies whose class no row carries is
 * exactly 0.  An anchor whose class occurs once has no positive pair: the loss is NaN (SupConLoss's 0/0, as in
 * b200ocl_supcon) and its gradients keep only the log Z_i part.  A label outside [0, C) sets *err_flag = 1 (nullable,
 * never cleared): its row adds nothing to the loss (which still divides by R), is not counted in n_c and gets a zero
 * dfeats row.  Two launches, every reduction in a fixed order with no floating-point atomics: repeated calls are
 * bit-identical on any GPU; no host synchronisation.  B200OCL_EINVAL for a null pointer, R < 2, d or C < 1, or a
 * temperature that is not finite and positive; B200OCL_EUNSUPPORTED for R > 4096, d > 2560 or C > 1024. */
size_t b200ocl_pcr_loss_workspace_bytes(int R, int C);
int b200ocl_pcr_loss(const float* feats, const int64_t* labels, int R, int d, const float* proxies, int C,
                     float temperature, float* loss, float* dfeats, float* dproxies, float* dbias, int* err_flag,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------- SCR augmentation
 * The second view of agents/scr.py:18-24,54 (kornia RandomResizedCrop -> RandomHorizontalFlip ->
 * ColorJitter -> RandomGrayscale) in one kernel over NCHW fp32 images in [0,1].
 * params [N,12] f32 (device), per sample: x0, y0, crop_w, crop_h, flip, jitter_on,
 * brightness delta, contrast factor, saturation factor, hue shift in turns, order code
 * (four 2-bit ids, 0 brightness 1 contrast 2 saturation 3 hue, first op in the low bits), gray.
 * The random draws are the caller's; kornia's exact arithmetic is parity-unpinned (absent). */
int b200ocl_scr_augment(const float* x, float* out, const float* params, int N, int H, int W, void* stream);

/* ---------------------------------------------------------------- tensor-core self test
 * D[128,N] = A[128,K] * B[N,K]^T on wgmma (tf32, fp32 register accumulator) with the descriptor
 * encodings the tensor-core convolution uses; mode 0 single TF32 pass, mode 1 the 3xTF32 split.
 * status[0] = 0 on completion. */
int b200ocl_selftest_umma_tf32(const float* A, const float* B, float* D, int N, int K, int mode, int* status,
                               void* stream);

/* One convolution (ks = 3 pad 1, or ks = 1 pad 0; stride 1 or 2; dgrad = 0: out[N,Hout,Wout,cout] = x[N,H,W,cin] * w;
 * dgrad = 1, 3x3 stride 1 only: its data gradient, x = dz[N,H,W,cout] -> out[N,H,W,cin]) through a chosen kernel
 * family, NHWC fp32, weights OIHW: path 0 automatic, 1 CUDA-core kernels, 2 wgmma with im2col tiles
 * (conv_tc.cu), 3 wgmma fed from a halo strip (conv_tcp.cu).  mode 0 raw store, 1 accumulate into out, 2 train
 * (forward only): raw store plus stats_out[4*cout] = batch mean, 1/sqrt(var+eps), running mean, running var
 * updated from zero with momentum 0.1; 3 eval (forward only): out = (conv - mean) * gamma / sqrt(var + eps) + beta
 * with stats_out[4*cout] = mean, var, gamma, beta as input; 4 the same plus x as the residual, then ReLU (cin == cout).
 * Exists so that tests can pin every convolution kernel against a reference convolution; fails with
 * B200OCL_EUNSUPPORTED when the path does not cover the shape.  Path 3 covers 3x3 stride-1 convolutions in every mode
 * but 2: train mode, stride 2 and 1x1 return B200OCL_EUNSUPPORTED. */
size_t b200ocl_conv_selftest_workspace_bytes(int N, int cin, int cout, int H, int W, int ks, int stride);
/* Host only: the launch b200ocl_conv_selftest makes for these arguments on a GPU with sms SMs (0: the current device),
 * and in stat_region the statistics region its workspace keeps for that SM count. */
int b200ocl_conv_selftest_geom(int N, int H, int W, int cin, int cout, int ks, int stride, int dgrad, int path, int mode,
                               int sms, b200ocl_conv_geom* out);
int b200ocl_conv_selftest(const float* x, const float* w_oihw, float* out, int N, int H, int W, int cin, int cout,
                          int ks, int stride, int dgrad, int path, int mode, float* stats_out, void* workspace,
                          size_t workspace_bytes, void* stream);
/* The eval forward of one 3x3 stride-1 C -> C convolution through a chosen path (as b200ocl_conv_selftest: 0 automatic,
 * 1 CUDA-core kernels, 2 conv_tc.cu, 3 conv_tcp.cu) with the epilogue's inputs given separately, as the network's
 * eval pass gives them: out = (conv - mean) * gamma / sqrt(var + eps) + beta with bn[4*C] = mean, var, gamma, beta;
 * plus residual[N,H,W,C] when residual is not null (a buffer other than x, like a block's input); then ReLU when
 * relu != 0.  The workspace is b200ocl_conv_selftest_workspace_bytes(N, C, C, H, W, 3, 1). */
int b200ocl_conv_selftest_eval(const float* x, const float* w_oihw, const float* bn, const float* residual, int relu,
                               float* out, int N, int H, int W, int C, int path, void* workspace, size_t workspace_bytes,
                               void* stream);

/* Window variant: A is read in place from a larger swizzled buffer P[rows][32] of 128-byte rows (tile row
 * 8g + r = P row start_row + g * sbo_rows + r), start address unaligned to the swizzle repeat when
 * start_row % 8 != 0; base_off_mode 1 sets the descriptor's base-offset field to (start row of each 64-row half) & 7.  Validates the
 * addressing the halo-patch tensor-core convolution relies on.  D[128,N] = A_window * B[N,32]^T, single TF32 pass. */
int b200ocl_selftest_umma_window(const float* P, const float* B, float* D, int rows, int start_row, int sbo_rows,
                                 int base_off_mode, int N, int* status, void* stream);

/* Weight gradient of one 3x3 stride-1 pad-1 convolution through the wgmma kernel (wgrad_tc.cu), NHWC fp32 inputs,
 * dw in OIHW: the cuDNN weight-gradient call behind loss.backward() for nn.Conv2d (models/resnet.py:11-12).  Exists so
 * that tests can pin the kernel against a reference; B200OCL_EUNSUPPORTED when the geometry is not covered. */
size_t b200ocl_wgrad_tc_selftest_workspace_bytes(int N, int H, int W, int cin, int cout);
typedef struct {
  int eligible;         /* the kernel covers the geometry; the fields below are 0 otherwise */
  int slices;           /* CTA columns: 20-channel slices of the activation */
  int cout_blocks;      /* CTA layers: blocks of at most 40 output channels */
  int bn;               /* MMA N of a block */
  int tiles;            /* 128-position tiles of the zero-padded strip */
  int tpc;              /* tiles per tensor-core accumulation chain */
  int chains;           /* partials per (slice, block) */
  int chains_per_cta;   /* chains one CTA walks: ceil(chains / CTAs), made even when above 1 */
  int ctas_x;           /* CTAs per (slice, block) */
  int sm_share;         /* sms / (slices * cout_blocks): the CTAs per (slice, block) the SM count allows */
  int sms;
} b200ocl_wgrad_tc_geom;
/* Host only: the launch b200ocl_wgrad_tc_selftest makes for these arguments on a GPU with sms SMs (0: the current
 * device). */
int b200ocl_wgrad_tc_selftest_geom(int N, int H, int W, int cin, int cout, int sms, b200ocl_wgrad_tc_geom* out);
int b200ocl_wgrad_tc_selftest(const float* x, const float* dz, float* dw_oihw, int N, int H, int W, int cin, int cout,
                              void* workspace, size_t workspace_bytes, void* stream);

/* ---- task snapshots (checkpoint.py, B200OCL_CHECKPOINT_ASYNC): one staging arena per run ----
 * A segment is one device array of a snapshot and its region of the staging arena, which holds `bytes` bytes at
 * `offset`.  B200OCL_SNAP_COPY regions hold the bytes as they are.  B200OCL_SNAP_U8 segments are fp32 replay-memory
 * rows (bytes a multiple of 4): each value v is stored as one byte u = rint(v * 255) when v is finite, 0 <= u <= 255
 * and u / 255 (IEEE division, the stream feeder's, common.cuh:u8_unit) is v bit for bit; the region keeps its fp32
 * size so that a segment with any other value can be stored as fp32 instead.  The table itself is in device memory. */
#define B200OCL_SNAP_COPY 0
#define B200OCL_SNAP_U8 1
typedef struct b200ocl_snapshot_segment {
  uint64_t ptr;    /* device address: the source (pack) or the destination (unpack); 16-byte aligned is fastest */
  uint64_t bytes;  /* bytes at ptr */
  uint64_t offset; /* byte offset of the segment's region in the staging arena */
  int32_t kind;    /* pack: B200OCL_SNAP_COPY or B200OCL_SNAP_U8; unpack: the form the region holds */
  int32_t reserved;
} b200ocl_snapshot_segment;

/* Workspace of pack and unpack: int32 counters[n_segments + 1].  After a pack, counters[s] is the number of values
 * of U8 segment s that failed the test (its region then holds the fp32 rows) and counters[n_segments] the number of
 * segments that were skipped as malformed (a region past staging_bytes, or a U8 size not a multiple of 4); after an
 * unpack, counters[n_segments] is the latter. */
size_t b200ocl_snapshot_workspace_bytes(int n_segments);
/* Copy (or encode) every segment into the staging arena: a memset of the counters, one launch that copies COPY
 * segments and encodes U8 segments while counting rejections, and one launch that overwrites the region of every U8
 * segment with a non-zero counter with its fp32 rows.  Nothing is read back. */
int b200ocl_snapshot_pack(const b200ocl_snapshot_segment* table, int n_segments, void* staging, size_t staging_bytes,
                          void* workspace, size_t workspace_bytes, void* stream);
/* The inverse: one launch that copies each COPY region to its ptr and decodes each U8 region (bytes / 4 bytes) into
 * bytes / 4 fp32 values u / 255 at its ptr. */
int b200ocl_snapshot_unpack(const b200ocl_snapshot_segment* table, int n_segments, const void* staging,
                            size_t staging_bytes, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200OCL_H_ */
