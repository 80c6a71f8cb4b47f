/* fgt_b200 — C-ABI of the H100-native (sm_90a) kernels behind FGT's flow-guided-attention
 * inference path. Plain pointers and sizes only; every pointer is a DEVICE pointer unless the
 * name ends in _host. All work is enqueued on the stream passed by the caller; the library never
 * allocates or frees device memory and never synchronises unless stated.
 *
 * Every entry point returns 0 on success or a negative FGT_ERR_* code; fgt_last_error() gives the
 * message (thread-local). There is no CPU fallback: without an sm_90 device the calls fail.
 *
 * Data carried between tensor-core kernels uses the "split-bf16" format: a logical fp32 tensor is
 * stored as two bf16 planes, hi = bf16(v) and lo = bf16(v - hi), the lo plane `plane` elements
 * after the hi plane. Three bf16 wgmma MMAs (hi*hi + hi*lo + lo*hi, fp32 accumulate in registers)
 * reproduce the fp32 product to ~2^-16 relative, which is what lets the path meet the 1e-3
 * end-to-end tolerance against the fp32 reference.
 *
 * Reference interfaces replaced (paths in the original FGT project, see INTEGRATION.md for the bindings):
 *   fgt_gemm_tc      : every nn.Linear / nn.Conv2d / nn.Conv3d on the inference path —
 *                      FGT/models/model.py:33-50,206-215,95-96; transformer_base/attention_flow.py:
 *                      33-36,44-48,51-54; attention_base.py:38-41; ffn_base.py:39-46;
 *                      LAFC/models/lafc.py:23-79; RAFT/extractor.py:118-192, RAFT/update.py:6-136,
 *                      RAFT/corr.py:52-60 (all-pairs correlation matmul).
 *   fgt_attention    : Attention.forward, FGT/models/transformer_base/attention_base.py:16-22 and
 *                      attention_flow.py:16-22 (softmax(QK^T/sqrt(d))V), with the window/zone
 *                      structure of TMHSA (attention_base.py:93-99) and SWMHSA (attention_flow.py:
 *                      130-164) expressed as key-tile lists instead of permuted copies.
 */
#ifndef FGT_B200_H_
#define FGT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* fgt_stream_t; /* == cudaStream_t */

enum {
  FGT_OK = 0,
  FGT_ERR_ARG = -1,     /* bad shape / alignment / unsupported geometry */
  FGT_ERR_CUDA = -2,    /* CUDA runtime or driver call failed */
  FGT_ERR_DEVICE = -3   /* no sm_90 device / driver entry point missing */
};

enum { FGT_ACT_NONE = 0, FGT_ACT_LEAKY02 = 1, FGT_ACT_RELU = 2, FGT_ACT_SIGMOID = 3, FGT_ACT_TANH = 4,
       FGT_ACT_LEAKY001 = 5 /* nn.LeakyReLU() default slope, LAFC/models/lafc.py:138 */ };
/* aux: out = act(v) + aux | act(v) * aux | act(v + aux) | relu(act(v) + aux) |
 *      (1 - aux2) * aux + aux2 * act(v)   (the ConvGRU state update, RAFT/update.py:52,58) |
 *      GRU_ZR: the z and r gate convolutions of a ConvGRU as ONE GEMM with N = 2*C (update.py:48-49,54-55):
 *      columns [0,C) -> out_f32 = act(v) (z), columns [C,2C) -> out_hi = act(v) * aux (r*h); both outputs
 *      and aux have C channels per position (output strides describe a C-channel buffer).
 *      With out_half (mixed-precision RAFT, autocast semantics) both GRU modes round act(v) to fp16 first; GRU_ZR
 *      stores r*h as fp16, and GRU rounds each of (1 - z), (1 - z) * h, z * q and their sum to fp16. */
enum { FGT_AUX_NONE = 0, FGT_AUX_ADD = 1, FGT_AUX_MUL = 2, FGT_AUX_ADD_PRE = 3, FGT_AUX_ADD_RELU = 4,
       FGT_AUX_GRU = 5, FGT_AUX_GRU_ZR = 6 };
enum { FGT_OUT_HALF_AUTOCAST = 2 /* FgtGemmDesc.out_half: autocast's rounding points, see there */ };

int fgt_version(void);
const char* fgt_last_error(void);

/* ------------------------------------------------------------------------------------------
 * fgt_gemm_tc: implicit-GEMM convolution / linear layer on the tensor cores (wgmma).
 *
 *   D[m, n] = act(alpha * sum_{tap, seg, c} A_seg[c, x(m)+dx(tap), y(m)+dy(tap), z(m)+dz(tap)]
 *                                          * W[n, tap, seg, c]  + bias[n])   (then aux add / mul)
 *
 * A operands are split-bf16 tensors with channels contiguous (NHWC / token-major). Up to two
 * segments are concatenated along the channel axis (the reference's torch.cat before a conv, and
 * its grouped skip-concat, FGT/models/model.py:57-65). A linear layer is the 1x1x1 case with
 * DX = rows. Strided convolutions are decomposed into `stride*stride` phase views of the input so
 * that every TMA box has unit element stride; zero padding is TMA out-of-bounds fill.
 * W is pre-packed (fgt_b200/packing.py) as split-bf16 [N, k_pad] in K-iteration order, each
 * (tap, segment) block padded to a multiple of 64 channels with zeros.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const void* hi;      /* bf16 hi plane */
  long long plane;     /* element offset hi -> lo plane */
  int C, DX, DY, DZ;   /* logical extents: channels, x, y, z(images / frames) */
  long long sx, sy, sz;/* element strides of x, y, z (channel stride is 1) */
  int c_base;          /* first channel of the slice consumed (group 0) */
  int c_per_group;     /* channel advance per conv group (0 if groups == 1) */
  int c_count;         /* channels consumed per group from this segment */
} FgtASeg;

typedef struct {
  int num_segs;
  FgtASeg seg[2];
  int kx, ky, kz;            /* filter taps along x, y, z */
  int stride, dil;           /* spatial stride / dilation (x and y) */
  int pad_x, pad_y, pad_z;   /* zero padding (low side; high side implied by out extents) */
  const void* w_hi;          /* packed weights, split-bf16 [N, k_pad] */
  long long w_plane;
  int N;                     /* output channels (all groups) */
  int k_pad;                 /* packed K = kz*ky*kx * sum_seg(ceil(c_count/64)*64) */
  int groups;
  int out_w, out_h, out_z;   /* output extents along x, y, z */
  int box_w, box_h;          /* output tile = box_w x box_h positions (<=128, multiple of 8) */
  int bn;                    /* output-channel tile (multiple of 16, <= 256, divides N/groups if groups>1); a
                                request wider than 128 runs as bn/t tiles of t channels, t the widest multiple
                                of 16 <= 128 dividing bn, so tiles never straddle a group boundary */
  /* epilogue */
  const float* bias;         /* [N] or NULL */
  float alpha;               /* scale applied to the accumulator before bias */
  int act;                   /* FGT_ACT_* */
  const float* aux;          /* fp32 tensor addressed like the output, or NULL */
  int aux_mode;              /* FGT_AUX_* */
  float* out_f32;            /* fp32 output or NULL */
  void* out_hi;              /* split-bf16 output (hi plane) or NULL */
  long long out_plane;
  long long os_z, os_y, os_x, os_c; /* output element strides for (z, y, x, channel) */
  const int* rowmap;         /* linear mode only (out_h == out_z == 1): row -> output row, <0 = drop */
  int lin_batch;             /* linear mode: if >0, z = row / lin_batch, x = row % lin_batch */
  const float* aux2;         /* second fp32 operand (FGT_AUX_GRU: the update gate z), addressed like the output */
  int terms;                 /* 0 / 3: split-bf16 product hi*hi + hi*lo + lo*hi (fp32-grade, 3 MMAs per K step);
                                1: the A segments and W are single-plane fp16 tensors (`hi` points at fp16 data, the
                                plane offsets are ignored), one MMA per K step — for layers whose error budget allows */
  int out_half;              /* 1: out_hi receives ONE plane of fp16 (the input format of a terms == 1 layer). With
                                out_f32 as well (mixed-precision RAFT, autocast semantics), the value is rounded to
                                fp16 before the activation and again after it, and out_f32 receives that fp16 value.
                                FGT_OUT_HALF_AUTOCAST (terms == 1 only; out_hi optional): every tensor the layer makes
                                under autocast is fp16 (mixed-precision LAFC) — the conv output is rounded before a
                                pre-activation add and the activation, the activation's output before FGT_AUX_ADD, and
                                the result; out_f32 alone (an fp32-only output) then also holds fp16 values */
} FgtGemmDesc;

int fgt_gemm_tc(const FgtGemmDesc* desc, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * fgt_attention: fused softmax(Q K^T * scale) V (flash-style, scores never leave the SM).
 * Q, K, V: split-bf16 row-major [batch, rows, heads*128] with their own leading dimensions, so one
 * fused QKV projection buffer [rows, 3*heads*128] can feed all three (V is consumed as an MN-major
 * wgmma B operand; no transposed copy). Output: split-bf16 [batch, Lq, heads*128].
 *   mode 0 (dense)   : every query row attends to keys [0, Lk)            (TMHSA zones)
 *   mode 1 (windowed): query tile i (=two 64-token windows) attends to its own two 64-key tiles
 *                      (block-diagonal) plus the shared keys [glob_start, glob_start+glob_count)
 *                      (SWMHSA local window + pooled global tokens)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const void* q_hi; long long q_plane; long long q_batch_stride; int q_ld;
  const void* k_hi; long long k_plane; long long k_batch_stride; int k_ld;
  const void* v_hi; long long v_plane; long long v_batch_stride; int v_ld;
  void* out_hi; long long out_plane; long long out_batch_stride; int out_ld;
  int batches, heads, head_dim; /* head_dim must be 128 */
  int Lq;                       /* query rows per batch */
  int Lk;                       /* dense: valid keys per batch */
  int Lk_rows;                  /* addressable key rows per batch (>= Lk; windowed: local + global rows) */
  float scale;                  /* 1/sqrt(head_dim) */
  int mode;
  int glob_start, glob_count;   /* windowed mode */
  const int* out_rowmap;        /* optional [batches * Lq]: query row -> row of a [rows, out_ld] output buffer (< 0 = drop);
                                   out_batch_stride is ignored then. Undoes the zone / window regrouping in the store. */
  int f16;                      /* 1: Q, K, V and the output are single-plane fp16 (every plane offset 0; one fp16 wgmma
                                   per K step for Q K^T and P V, scores and softmax in fp32); 0: split-bf16 */
} FgtAttnDesc;

int fgt_attention(const FgtAttnDesc* desc, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * HBM-bound helpers (coalesced / vectorised CUDA-core kernels). "split" outputs are split-bf16.
 * ------------------------------------------------------------------------------------------ */

/* NCHW fp32 (src0 channels then src1 channels) -> NHWC split with `cpad` channels (zeros beyond
 * c0+c1) and `pad` pixels of REPLICATION padding on each side. Replaces torch.cat + view at
 * FGT/models/model.py:253-258 and nn.ReplicationPad2d at model.py:207. */
int fgt_pack_nchw(const float* src0, int c0, const float* src1, int c1, int n, int H, int W, int pad, int cpad,
                  void* out_hi, long long out_plane, fgt_stream_t stream);

/* im2col of NCHW fp32 inputs (src0 channels then src1 channels) for the tiny-channel first layers:
 * output row (n, oy, ox) holds the k x k neighbourhood, channel = (ky*k+kx)*cin + c, zero-padded to
 * `cpad` (>= k*k*cin) channels; borders are zero (replicate=0) or clamped (replicate=1, i.e.
 * nn.ReplicationPad2d(pad) followed by an unpadded conv). Feeds fgt_gemm_tc as a K=cpad linear layer.
 * Replaces the input side of nn.Conv2d at FGT/models/model.py:34 and model.py:207-208. */
int fgt_im2col_nchw(const float* src0, int c0, const float* src1, int c1, int n, int H, int W, int k, int stride,
                    int pad, int replicate, int OH, int OW, int cpad, float scale, float shift, void* out_hi,
                    long long out_plane, fgt_stream_t stream); /* in-bounds values become v*scale + shift */

/* LayerNorm over the channel concatenation [a ; b] of fp32 rows. gamma/beta may be NULL (statistics
 * only: the affine is then folded into the consuming Linear at weight-pack time). Destination row of work item d is
 * (d / rows_per_batch) * dst_batch_rows + dst_row0 + d % rows_per_batch; its source row is
 * gather[d] (or d when gather == NULL); gather[d] < 0 writes a zero row (the reference's F.pad).
 * Replaces nn.LayerNorm at model.py:126,128,147 and attention_flow.py:142-143,154 together with the
 * window / zone partition copies at attention_flow.py:132-133,150-153, attention_base.py:93-98. */
/* Mixed precision: fgt_rownorm, fgt_swin_prep, fgt_fold, fgt_fold_unfold and fgt_dwconv3x3_res write their 16-bit
 * output as single-plane fp16 rows when its plane offset is 0 (split-bf16 otherwise); fgt_conv_tail reads fp16
 * activations and weights when both plane offsets are 0. */
int fgt_rownorm(const float* a, int ca, int lda, const float* b, int cb, int ldb, const int* gather,
                int rows_per_batch, long long total_rows, int dst_batch_rows, int dst_row0, const float* gamma,
                const float* beta, void* out_hi, long long out_plane, float eps, fgt_stream_t stream);

/* Same, with the normalised rows stored to n_out (<= 8) destination buffers of identical layout
 * (out_his_host: HOST array of device pointers, local or peer-mapped). With the peers' K/V-input
 * buffers as destinations this is LayerNorm fused with the all-gather of frame-sharded TMHSA
 * (attention_base.py:84-98 across ranks): P2P stores over NVLink, followed by fgt_peer_barrier. */
int fgt_rownorm_bcast(const float* a, int ca, int lda, const float* b, int cb, int ldb, const int* gather,
                      int rows_per_batch, long long total_rows, int dst_batch_rows, int dst_row0, const float* gamma,
                      const float* beta, void* const* out_his_host, int n_out, long long out_plane, float eps,
                      fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Region fill / flow diffusion (tool/utils/region_fill.py:7-138 with factor = 1, called per flow channel by
 * diffusion(), tool/video_inpainting.py:44-52): for B images [B,H,W] fp64 and hole masks (uint8, non-zero =
 * hole) solve, inside each mask, the discrete Laplace equation with the surrounding image values as
 * boundary data and zero flux at the image border — batched matrix-free conjugate gradients in fp64
 * instead of the reference's per-image sparse direct solve.
 *   fgt_regionfill_init  : x = 0, r = p0 = right-hand side (region_fill.py:69-112), rr[0..B) = <r,r>
 *   fgt_regionfill_iters : CG iterations k0 .. k0+iters-1; rr / pap are zero-initialised arrays of
 *                          (max_iters+1)*B doubles (iteration k uses rr[k*B+b], pap[k*B+b], writes rr[(k+1)*B+b]);
 *                          the host reads rr to decide convergence
 *   fgt_regionfill_finish: out = x inside the mask, img outside (region_fill.py:15-16)
 * All arrays are caller-owned device memory. */
int fgt_regionfill_init(const double* img, const unsigned char* mask, int B, int H, int W, double* x, double* r,
                        double* p0, double* rr, fgt_stream_t stream);
int fgt_regionfill_iters(const unsigned char* mask, int B, int H, int W, double* x, double* r, double* p0, double* p1,
                         double* ap, double* rr, double* pap, int k0, int iters, fgt_stream_t stream);
int fgt_regionfill_finish(const double* img, const unsigned char* mask, long long total, const double* x, double* out,
                          fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Gradient-domain (Poisson) blending (tool/utils/Poisson_blend_img.py:19-270: Poisson_blend_img, solvePoisson,
 * constructEquation; called per frame at tool/video_inpainting.py:645-656): F frames x 3 channels solved together,
 * matrix-free, by LSQR with scipy's recurrences and stopping tests (the reference calls
 * scipy.sparse.linalg.lsqr with default tolerances, so its answer is the iterate at which that rule fires).
 * All vectors fp64, channels-last; caller-owned, ZERO-INITIALISED device memory unless noted:
 *   trg [F,H,W,3], gx [F,H,W-1,3], gy [F,H-1,W,3] (forward differences); hole / gmask / edge uint8 [F,H,W]
 *   (gmask, edge may be NULL = all zero); code uint8 [F,H,W]; u [F,4,H*W,3]; v, w, x [F,H*W,3];
 *   bb, aa, ww: (max_iters + chunk + 2) * 3F per-iteration sums (slot k*3F + s); state [2, 3F, 16] (ping-pong by iteration
 *   parity; per system s = 3*frame + channel: [12] = stopped, [13] = scipy's istop, [14] = itn).
 *   fgt_poisson_setup   : equation codes, u = b, bb[0] = |b|^2 (constructEquation :176-266); appends the pixels
 *                         that own equations to list [F,H*W] uint32 (pixel index | code << 24; zero-initialised, H*W <
 *                         2^24) and counts them in cnt [F] (zero-initialised) — the host reads max(cnt) once and
 *                         passes it as max_cnt, so the iteration kernels launch threads for those pixels only
 *   fgt_poisson_iters   : the next `iters` values of the iteration index k, which lives on the device (kctr: 2 int32,
 *                         zero-initialised): k = 0 finishes the set-up (v = A^T u / alfa, w = v), k >= 1 is LSQR
 *                         iteration k; two kernels per k; systems that have stopped stay frozen
 *   fgt_poisson_graph_* : the same `iters` kernel pairs captured once into an executable CUDA graph (a host-side driver
 *                         object, the only thing this library ever creates; destroy it with _graph_destroy) and
 *                         replayed with _graph_launch — every replay continues at the device-side k
 *   fgt_poisson_unfilled: the two raster sweeps of the connectivity check (:139-172) -> clr [2,F,H,W]
 *   fgt_poisson_finish  : out = hole ? float64(float32(x)) : trg (:29,40-44); unf = hole & !clr[0] & !clr[1]
 *                         (unf / clr may be NULL)
 *   fgt_poisson_advance_host: HOST-ONLY — runs the scalar recurrence of one iteration (the same
 *                         __host__ __device__ function the kernels call) on 16-double host states; step_out_host
 *                         = {t1, t2, vscale, alfa*uscale, skip_all, skip_u}. For tests of the stopping logic. */
int fgt_poisson_setup(const double* trg, const double* gx, const double* gy, const unsigned char* hole,
                      const unsigned char* gmask, const unsigned char* edge, int F, int H, int W, unsigned char* code,
                      double* u, double* bb, unsigned* list, int* cnt, fgt_stream_t stream);
int fgt_poisson_iters(const unsigned* list, int max_cnt, int F, int H, int W, double* u, double* v, double* w, double* x,
                      double* bb, double* aa, double* ww, double* state, int* kctr, int iters, double atol, double btol,
                      double conlim, int iter_lim, fgt_stream_t stream);
int fgt_poisson_graph_create(const unsigned* list, int max_cnt, int F, int H, int W, double* u, double* v, double* w,
                             double* x, double* bb, double* aa, double* ww, double* state, int* kctr, int iters,
                             double atol, double btol, double conlim, int iter_lim, void** exec_out);
int fgt_poisson_graph_launch(void* exec, fgt_stream_t stream);
int fgt_poisson_graph_destroy(void* exec);
int fgt_poisson_unfilled(const unsigned char* hole, const unsigned char* gmask, int F, int H, int W, unsigned char* clr,
                         fgt_stream_t stream);
int fgt_poisson_finish(const double* trg, const unsigned char* hole, const double* x, int F, int H, int W, double* out,
                       const unsigned char* clr, unsigned char* unf, fgt_stream_t stream);
int fgt_poisson_advance_host(const double* prev_host, double* cur_host, double* step_out_host, int k, double bbk,
                             double aak, double wwk, double atol, double btol, double conlim, int iter_lim);

/* ------------------------------------------------------------------------------------------
 * The FGT stage's window loop around Model.forward (tool/video_inpainting.py:686-745), device-resident instead of
 * one host round trip per window and frame. Clip tensors: frames [N,3,H,W] float in [0,1] (np2tensor(frameBlends),
 * :691), masks [N,H,W] uint8 (:692-694), flows [N,2,H,W] float (completed forward flows, last one repeated, :702-707).
 *   fgt_plane_max     : out[i] = max over plane i of x [planes, plane_size]   (norm_flows :402-407: per frame & channel)
 *   fgt_window_gather : model inputs of one window — ids [t] (device int32) are neighbour + reference frame ids (:711-717):
 *                       out_frames [t,3,H,W] = (frames*2-1)*(1-mask) (:695,:721), out_flows [t,2,H,W] = flows/fmax,
 *                       out_masks [t,1,H,W]
 *   fgt_window_compose: filled [t,3,H,W] = Model.forward output; for the first k (= neighbour) frames
 *                       comp[id] = u8((out+1)/2*255)*mask + u8(frame*255)*(1-mask) (:725-733), stored if first[i] else
 *                       averaged 0.5/0.5 with the stored value (:734-741); comp [N,H,W,3] float
 *   fgt_comp_to_u8    : the final astype(uint8) (:745)
 * Same IEEE single-precision operations in the same order as the reference: bit-identical given the same model output. */
int fgt_plane_max(const float* x, int planes, long long plane_size, float* out, fgt_stream_t stream);
int fgt_window_gather(const float* frames, const unsigned char* masks, const float* flows, const float* fmax,
                      const int* ids, int t, int H, int W, float* out_frames, float* out_flows, float* out_masks,
                      fgt_stream_t stream);
int fgt_window_compose(const float* filled, const float* frames, const unsigned char* masks, const int* ids,
                       const unsigned char* first, int k, int H, int W, float* comp, fgt_stream_t stream);
int fgt_comp_to_u8(const float* comp, long long total, unsigned char* out, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * The tensor glue of FGT's validation (FGT/networks/network.py:258-352, Network._validate; fgt_b200/validate.py):
 *   fgt_valid_flow_scale : resized flows [B,H,W,2] float in place, u = u / pre_w * w, v = v / pre_h * h (read_flows)
 *   fgt_valid_inputs     : frames uint8 [t,H,W,3] and masks uint8 [t,H,W] (0 / non-zero) -> out_frames [t,3,H,W] =
 *                          x / 127.5 - 1, out_masked = out_frames * (1 - mask), out_masks [t,1,H,W] float 0 / 1
 *   fgt_valid_norm_flows : out = flows / fmax per plane of plane_size values (norm_flows: signed max, fgt_plane_max)
 *   fgt_valid_score      : comp = filled * m + frames * (1 - m); comp_u8 and frames_u8 [t,H,W,3] =
 *                          uint8(clip((x + 1) / 2 * 255, 0, 255)) of comp and of frames (metrics_calc)
 * Same IEEE single-precision operations in the same order as the reference: bit-identical given the same inputs. */
int fgt_valid_flow_scale(float* flow, long long pixels, float pre_w, float w, float pre_h, float h, fgt_stream_t stream);
int fgt_valid_inputs(const unsigned char* frames, const unsigned char* masks, int t, int H, int W, float* out_frames,
                     float* out_masked, float* out_masks, fgt_stream_t stream);
int fgt_valid_norm_flows(const float* flows, const float* fmax, int planes, long long plane_size, float* out,
                         fgt_stream_t stream);
int fgt_valid_score(const float* filled, const float* frames, const float* masks, int t, int H, int W,
                    unsigned char* comp_u8, unsigned char* frames_u8, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Forward flow splatting (LAFC/models/utils/flow_warp.py:4-94, flow_prop / warp / sample_one): feat [B,C,H,W] is
 * scattered along flow [B,2,H,W] (channel 0: column shift, channel 1: row shift, as in the reference) to the four
 * integer neighbours of each target with weights exp(-d^2); out [B,C,H,W] = accumulated features / accumulated weight
 * where the latter is positive; wsum [B,H,W] is workspace (both are zeroed by the call). backward != 0 negates the
 * integer shifts (mode='backward'). */
int fgt_flow_splat(const float* feat, const float* flow, int B, int C, int H, int W, int backward, float* out,
                   float* wsum, fgt_stream_t stream);
/* HOST-ONLY test hook: targets (row ti, column tj), weights and in-image flags of the four neighbours source pixel
 * (i, j) is scattered to — the __host__ __device__ function the kernel calls. x = row shift, y = column shift. */
int fgt_flow_splat_targets_host(float x, float y, int i, int j, int H, int W, int backward, int* ti_host, int* tj_host,
                                float* wt_host, int* ok_host);

/* ------------------------------------------------------------------------------------------
 * Peer memory for the multi-GPU exchange (no reference counterpart: the reference's inference is
 * single-device, SURVEY §8e). One process per GPU; buffers are cudaMalloc'ed here (IPC-capable,
 * zero-initialised), exported as 64-byte CUDA IPC handles that the host side exchanges over its
 * process group, and imported by the peers (peer access enabled lazily).
 * fgt_peer_barrier: device-side barrier among n ranks on `stream` — flags_host[q] is (a mapping of)
 * rank q's flag array of n uint64 (zero-initialised); epoch_ctr is a local device uint64 that the
 * kernel increments, so the call is CUDA-graph replayable. Release/acquire at system scope: all
 * peer stores issued by earlier kernels on `stream` are visible to the peers' kernels that follow
 * their barrier. Spins at most ~10 s, then traps (a lost rank must not hang the GPU). */
int fgt_peer_alloc(size_t bytes, void** ptr);
int fgt_peer_free(void* ptr);
int fgt_peer_export(void* ptr, unsigned char handle[64]);
int fgt_peer_import(const unsigned char handle[64], void** ptr);
int fgt_peer_unimport(void* ptr);
int fgt_peer_barrier(void* const* flags_host, int n, int rank, void* epoch_ctr, fgt_stream_t stream);

/* Depthwise k x k, stride k convolution (+bias) of the token grid [bt,h,w,ca+cb], zero-padded to
 * (gh*k, gw*k) -> fp32 [bt, gh*gw, ca+cb]. weight is the torch layout [C,1,k,k].
 * Replaces global_extract_k / global_extract_v, attention_flow.py:135,145. */
int fgt_dwpool(const float* a, int ca, const float* b, int cb, int bt, int h, int w, int k, int gh, int gw,
               const float* weight, const float* bias, float* out, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Mask / resize glue of the driver on the device (SURVEY 8f rank 3; tool/video_inpainting.py:264-268,546-561,637).
 * Masks are uint8 [B,H,W] (0 / non-zero); every call is bit-exact against the library call it replaces.
 *   fgt_binary_dilate     scipy.ndimage.binary_dilation(m, iterations=n): n passes of the 3x3 cross, border 0;
 *                         `tmp` is a second [B,H,W] scratch buffer, the result lands in `out`.
 *   fgt_fill_holes_*      scipy.ndimage.binary_fill_holes(m): init zeroes `reach`; each pass propagates "background
 *                         connected to the border" along whole rows and columns and sets *changed (device int) when
 *                         anything moved — the caller repeats until it stays 0; finish writes out = !reach.
 *   fgt_resize_nearest_u8 cv2.resize(..., INTER_NEAREST) on [B,H,W,C] uint8.
 *   fgt_resize_bilinear_f32  cv2.resize(..., INTER_LINEAR) on float32 [B,H,W,C] (nchw = 0) — optionally scaling channel
 *                         0 / 1 of the result (the driver rescales resized flow vectors, :266-267) — or
 *                         F.interpolate(mode="bilinear", align_corners=False) on [B,C,H,W] (nchw = 1). Bit-identical
 *                         to cv2 for C = 2 (cv2's INTER_AREA when exactly 2x smaller; C = 1, 3, 4 go to IPP in cv2) and
 *                         to ATen's vectorised CPU kernel (its FMAs included) for nchw.
 * ------------------------------------------------------------------------------------------ */
int fgt_binary_dilate(const unsigned char* in, int B, int H, int W, int iterations, unsigned char* tmp, unsigned char* out,
                      fgt_stream_t stream);
int fgt_fill_holes_init(const unsigned char* fg, int B, int H, int W, unsigned char* reach, fgt_stream_t stream);
int fgt_fill_holes_pass(const unsigned char* fg, int B, int H, int W, unsigned char* reach, int* changed, int passes,
                        fgt_stream_t stream);
int fgt_fill_holes_finish(const unsigned char* reach, int B, int H, int W, unsigned char* out, fgt_stream_t stream);
int fgt_resize_nearest_u8(const unsigned char* in, int B, int H, int W, int C, int OH, int OW, unsigned char* out,
                          fgt_stream_t stream);
int fgt_resize_bilinear_f32(const float* in, int B, int H, int W, int C, int OH, int OW, int nchw, float scale_c0,
                            float scale_c1, float* out, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * cv2.inpaint(img, mask, radius, cv2.INPAINT_TELEA) on the device, byte-identical to OpenCV
 * (tool/video_inpainting.py:316-320, 591-599, 663-671). Images uint8 [B,H,W,C] with C = 1 or 3 and H, W >= 2; masks
 * uint8 [H,W] per image, non-zero = hole, `mask_stride` elements apart (0: one mask for every image, planned once).
 * The radius is rounded and clamped to [1, 100] like cv2's, and must then be 3 (the driver's): FGT_ERR_ARG otherwise.
 * Radius 3 matched cv2 4.13 on every case tried (tens of thousands of seeded images and masks up to 1280x720); radii
 * 1, 2, 4 and 6 miss by one level on roughly 1 in 1000 to 1 in 20000 small speckled masks, so they are refused.
 * An empty or whole-image mask returns the image unchanged.
 *   fgt_inpaint_telea_workspace  bytes of workspace for n_masks distinct masks (negative FGT_ERR_* on bad arguments).
 *   fgt_inpaint_telea       fgt_inpaint_telea_plan + fgt_inpaint_telea_fill; mask_stride is 0 or H*W.
 *                           `out` must not alias `images`.
 *   fgt_inpaint_telea_plan  plans n_masks masks [n,H,W] into the workspace: the fast marches (one CTA per mask, serial),
 *                           then the levels (serial per mask as well).
 *   fgt_inpaint_telea_fill  fills images [B,H,W,C] level by level (one CTA per image) from the plans in the workspace:
 *                           one plan per image, or plan 0 for every image when shared_plan != 0.
 *   fgt_inpaint_telea_host  HOST-ONLY — the same plan and fill for one image on the CPU, through the same
 *                           __host__ __device__ routines (a verification tool; nothing on the product path calls it).
 *   fgt_grad_prep_pre       the gradient preparation before TELEA (:591-594): video float32 [B,H,W,3] with the hole
 *                           (mask [B,H,W]) zeroed, times 255 in float32, truncated to uint8.
 *   fgt_grad_prep_post      after TELEA (:596-614): uint8 / 255 in float32, forward differences along x (gx) and y
 *                           (gy) with the last column / row zero, zeroed where mask_dilated [B,H,W] is set; gx, gy
 *                           float32 [B,H,W,3]. Bit-identical to numpy's float32 arithmetic.
 * ------------------------------------------------------------------------------------------ */
long long fgt_inpaint_telea_workspace(int n_masks, int H, int W);
int fgt_inpaint_telea(const unsigned char* images, const unsigned char* masks, int B, int H, int W, int C,
                      long long mask_stride, double radius, void* workspace, long long workspace_bytes,
                      unsigned char* out, fgt_stream_t stream);
int fgt_inpaint_telea_plan(const unsigned char* masks, int n_masks, int H, int W, double radius, void* workspace,
                           long long workspace_bytes, fgt_stream_t stream);
int fgt_inpaint_telea_fill(const unsigned char* images, int B, int H, int W, int C, int shared_plan, double radius,
                           const void* workspace, long long workspace_bytes, unsigned char* out, fgt_stream_t stream);
int fgt_inpaint_telea_host(const unsigned char* image_host, const unsigned char* mask_host, int H, int W, int C,
                           double radius, unsigned char* out_host);
int fgt_grad_prep_pre(const float* video, const unsigned char* mask, int B, int H, int W, unsigned char* u8,
                      fgt_stream_t stream);
int fgt_grad_prep_post(const unsigned char* u8, const unsigned char* mask_dilated, int B, int H, int W, float* gx,
                       float* gy, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Native-resolution output (definition: oracle/native_oracle.py; bit-identical to it, integer arithmetic only). The
 * pipeline's working-resolution result comp uint8 [B,cH,cW,3] is upscaled to the frames' size H x W with cv2's
 * fixed-point INTER_LINEAR and blended into the original frames uint8 [B,H,W,3] with weight c / A, where c counts the
 * pixels of the dilated hole D in the (2k+1) x (2k+1) window around the pixel (the edge replicated outside the image)
 * and A = (2k+1)^2,
 * k = ceil(max(H / cH, W / cW)). D is the hole cross-dilated r + 2k times (fgt_binary_dilate).
 *   fgt_native_workspace  bytes of workspace for the counts of n_masks masks of H x W (negative FGT_ERR_* when a size
 *                         is empty or A does not fit the uint16 count, i.e. k outside [1, 127]).
 *   fgt_native_count      c of the dilated masks [n_masks,H,W] (0 / non-zero) into the workspace: two separable box sums.
 *   fgt_native_composite  out uint8 [B,H,W,3] from comp, frames and the counts in the workspace: one count per frame, or
 *                         count 0 for every frame when shared_mask != 0. C must be 3; k must be the window of comp's
 *                         size and the frames' size; out must not alias comp or frames.
 * ------------------------------------------------------------------------------------------ */
long long fgt_native_workspace(int n_masks, int H, int W, int k);
int fgt_native_count(const unsigned char* dilated, int n_masks, int H, int W, int k, void* workspace,
                     long long workspace_bytes, fgt_stream_t stream);
int fgt_native_composite(const unsigned char* comp, int B, int cH, int cW, const unsigned char* frames, int H, int W,
                         int C, int shared_mask, int k, const void* workspace, long long workspace_bytes,
                         unsigned char* out, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Quality metrics of N result frames against N ground-truth frames, both [N,H,W,C] with C = 1 or 3 and values on the
 * 0..255 scale, as the reference defines them (FGT/metrics/psnr.py, ssim.py and the L1 / L2 errors of
 * FGT/metrics/__init__.py calculate_metrics); every input is converted to float64 first. a_dtype / b_dtype are
 * FGT_METRIC_U8 or FGT_METRIC_F32. Per frame, with d = a - b over all H*W*C values:
 *   l1 = mean|d|,  l2 = sqrt(sum d^2) / (H*W*C),  psnr = 100 if mean d^2 == 0 else 20 log10(255 / sqrt(mean d^2)),
 *   ssim = the mean over channels of the MATLAB-style SSIM of each plane: 11x11 Gaussian window (sigma 1.5, cv2's
 *          getGaussianKernel) at the (H-10) x (W-10) valid positions, C1 = (0.01*255)^2, C2 = (0.03*255)^2,
 *          sigma^2 = w*(x^2) - mu^2 as written in ssim.py.
 * H and W must be at least 11 (the reference returns NaN below), N * C at most 65535.
 *   fgt_metrics_workspace  bytes of workspace for N frames of H x W x C (negative FGT_ERR_* on bad sizes).
 *   fgt_metrics            out float64 [N][4] = (l1, l2, psnr, ssim); ssim_c float64 [N][C] = the per-channel SSIM
 *                          (NULL: not written). Two kernels: per-(frame, channel, 32x32 tile) partial sums into the
 *                          workspace, then a fixed-order reduction per frame, so each frame's values do not depend on
 *                          N or on the other frames.
 * ------------------------------------------------------------------------------------------ */
enum { FGT_METRIC_U8 = 0, FGT_METRIC_F32 = 1 };
long long fgt_metrics_workspace(int N, int H, int W, int C);
int fgt_metrics(const void* a, int a_dtype, const void* b, int b_dtype, int N, int H, int W, int C, void* workspace,
                long long workspace_bytes, double* out, double* ssim_c, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Flow warping error of a clip (definition: oracle/warp_error_oracle.py), built from the reference's image_warp and
 * fbConsistencyCheck (FGT/models/utils/fbConsistencyCheck.py) with grid_sample's align_corners=True convention.
 * frames [N,H,W,C] (C = 1 or 3) on the 0..255 scale, frame_dtype FGT_METRIC_U8 or FGT_METRIC_F32, I = float32(V) / 255;
 * masks uint8 [N,H,W] (non-zero = hole; NULL: none); flow_f / flow_b float32 [N-1,2,H,W], F_t: t -> t+1 and
 * B_t: t+1 -> t, in pixels, x first. Per pair t, with W_t = I_{t+1} sampled at x + F_t(x) and M_t = 1 where
 * |F + B(x+F)|^2 <= 0.01 (|F|^2 + |B(x+F)|^2) + 0.5, err = sum_c (I_t - W_t)^2 in float64:
 *   out float64 [N-1][4] = (sum M*err, sum M, sum M*hole_t*err, sum M*hole_t); E_warp of the pair is out[0] / out[1].
 * H and W at least 2, N at least 2 and N - 1 at most 65535.
 *   fgt_warp_error_workspace  bytes of workspace for N frames of H x W x C (negative FGT_ERR_* on bad sizes).
 *   fgt_warp_error            two kernels: per-(pair, 32x32 tile) partial sums into the workspace, then a fixed-order
 *                             reduction per pair (bit-reproducible). Optional maps (NULL: not written): warped float32
 *                             [N-1,H,W,C], the warped frame t+1 on the 0..1 scale; valid uint8 [N-1,H,W], M_t.
 * ------------------------------------------------------------------------------------------ */
long long fgt_warp_error_workspace(int N, int H, int W, int C);
int fgt_warp_error(const void* frames, int frame_dtype, const unsigned char* masks, const float* flow_f,
                   const float* flow_b, int N, int H, int W, int C, void* workspace, long long workspace_bytes,
                   double* out, float* warped, unsigned char* valid, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Flow colour coding of the driver's --vis_flows (RAFT/utils/flow_viz.py flow_to_image :109-132 with
 * flow_uv_to_colors :70-106 and the 55-entry Middlebury wheel of make_colorwheel :20-67): flows fp32 [B,H,W,2]
 * (8-byte aligned) -> out uint8 [B,H,W,3], RGB (bgr = 0) or BGR (bgr != 0). Each image is divided by its own maximum
 * radius + 1e-5. Every operation is rounded as numpy 2 (NEP 50) rounds the reference's: float32 up to the wheel
 * coordinate, float64 from the interpolation weight on, no contraction. The angle is atan2f, which may differ from the
 * host's float32 arctan2 by an ulp, so a few values in a million can differ by one level.
 *   fgt_flow_to_image_workspace  bytes of workspace for B flows of H x W (negative FGT_ERR_* on bad sizes).
 *   fgt_flow_to_image            two kernels: per-image maximum radius (partial maxima into the workspace; exact in any
 *                                order), then the colour pass. maxima float [B] (NULL: not written) receives each
 *                                image's maximum radius, or NaN when the image holds a NaN or Inf, where the reference
 *                                raises; such an image's output is left unwritten. B at most 65535.
 * ------------------------------------------------------------------------------------------ */
long long fgt_flow_to_image_workspace(int B, int H, int W);
int fgt_flow_to_image(const float* flow, int B, int H, int W, int bgr, void* workspace, long long workspace_bytes,
                      unsigned char* out, float* maxima, fgt_stream_t stream);

/* 3x3 convolution (zero padding 1, stride 1) with cout <= 3 output channels + bias + activation in one kernel: the
 * nine taps become the N dimension of a wgmma GEMM over the input positions (activation read once) and are summed
 * per output pixel in shared memory. x: NHWC split-bf16 [n,H,W,cin], cin a multiple of 64 (<= 256); w: split-bf16
 * [32, cin], row tap*cout + c = W[c,:,ty,tx] (zero rows up to 32); act: FGT_ACT_NONE, _LEAKY02, _RELU, _SIGMOID or
 * _TANH; out: fp32 with element strides (os_n, os_c, os_y, os_x). Replaces the decoder's final nn.Conv2d(64, 3, 3) +
 * tanh (FGT/models/model.py:185-193) and FlowHead.conv2, nn.Conv2d(256, 2, 3) (RAFT/update.py:10,14). */
int fgt_conv_tail(const void* x_hi, long long x_plane, int n, int H, int W, int cin, const void* w_hi, long long w_plane,
                  int k_pad, int cout, const float* bias, int act, float* out, long long os_n, long long os_c,
                  long long os_y, long long os_x, fgt_stream_t stream);

/* Operand preparation of SWMHSA in one launch (attention_flow.py:130-154): for every frame, the LayerNorm statistics
 * (no affine: q_norm / k_norm / v_norm are folded into the projection weights) of the window-partitioned tokens
 * [x ; f'] (d+df channels -> qkn) and x (d channels -> vn), then of the pooled global tokens (depthwise gd x gd /
 * stride gd convolution + bias of [x ; f'] with gk_* and of x with gv_*; the depthwise weights are passed TAP-MAJOR,
 * [gd*gd, C] = torch's [C,1,gd,gd] transposed, so that one tap's weights are a coalesced row).
 * Destination rows per frame: [0, nl) window rows through win_map (token index, <0 = zero row), [nl, nl + gh*gw)
 * pooled rows; R rows per frame in total. qkn / vn are split-bf16 [bt*R, d+df] / [bt*R, d]. Replaces two fgt_dwpool
 * and four fgt_rownorm launches. */
int fgt_swin_prep(const float* x, const float* fp, int d, int df, int bt, int h, int w, const int* win_map, int nl,
                  int R, int gd, int gh, int gw, const float* gk_w, const float* gk_b, const float* gv_w,
                  const float* gv_b, void* qkn_hi, long long qkn_plane, void* vn_hi, long long vn_plane, float eps,
                  fgt_stream_t stream);

/* out = x + depthwise3x3(x) + bias on the token grid (AddPosEmb.forward, model.py:75-88). */
int fgt_dwconv3x3_res(const float* x, int bt, int h, int w, int C, const float* weight, const float* bias,
                      float* out, void* out_hi, long long out_plane, fgt_stream_t stream);

/* Overlap-add fold of position-major token patches hid[bt*th*tw, (kh*kw)*C] to [bt,OH,OW,C]
 * (optionally divided by the coverage count, optionally + add). nn.Fold at ffn_base.py:57-75 and
 * model.py:103-109 (+ the skip add at model.py:279). */
int fgt_fold(const float* hid, int bt, int th, int tw, int C, int kh, int kw, int stride, int pad, int OH, int OW,
             int normalize, const float* add, float* out, void* out_hi, long long out_plane, fgt_stream_t stream);

/* fgt_fold(normalize = 1) followed by fgt_unfold(relu) in one launch, without the [bt,OH,OW,C] image round trip
 * (FusionFeedForward's fold / coverage division / unfold / ReLU, ffn_base.py:57-75,40): every entry of the hidden
 * patches becomes the rectified mean over the entries that fold onto the same pixel. hid fp32 [bt*th*tw, kh*kw*C]
 * position-major -> split-bf16 of the same shape; bit-identical to the two-launch sequence. */
int fgt_fold_unfold(const float* hid, int bt, int th, int tw, int C, int kh, int kw, int stride, int pad, int OH, int OW,
                    int relu, void* out_hi, long long out_plane, fgt_stream_t stream);

/* nn.Unfold (+ optional ReLU) of [bt,OH,OW,C] into position-major token patches (split). */
int fgt_unfold(const float* img, int bt, int th, int tw, int C, int kh, int kw, int stride, int pad, int OH,
               int OW, int relu, void* out_hi, long long out_plane, fgt_stream_t stream);

/* Nearest x2 upsampling of an NHWC split tensor (F.interpolate at network_blocks_2d.py:58-60). */
int fgt_upsample2x(const void* in_hi, long long in_plane, int n, int H, int W, int C, void* out_hi,
                   long long out_plane, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * RAFT helpers (HBM-bound). Tensors are NHWC fp32 unless noted.
 * ------------------------------------------------------------------------------------------ */

/* Per-(image, channel) sum / sum-of-squares -> stats[n][C][2] (double). nn.InstanceNorm2d statistics,
 * RAFT/extractor.py:29-33,131-132 (the normalisation itself is fgt_instnorm_act). */
int fgt_chan_stats(const float* x, int n, int HW, int C, double* stats, fgt_stream_t stream);

/* y = (x - mean) * rsqrt(var + eps) [ReLU] ; if res: y = relu(y + res). ResidualBlock.forward,
 * RAFT/extractor.py:47-56 and BasicEncoder.forward :176-178 for the instance-norm feature net.
 * out_hi receives split-bf16, or single-plane fp16 when out_plane == 0 (mixed precision; `out` then receives the same
 * fp16-rounded values). */
int fgt_instnorm_act(const float* x, const double* stats, int n, int HW, int C, float eps, int relu,
                     const float* res, float* out, void* out_hi, long long out_plane, fgt_stream_t stream);

/* 2x2 average pooling over the last two dims of [rows, h, w] (correlation pyramid, RAFT/corr.py:25-27). */
int fgt_avgpool2(const float* in, long long rows, int h, int w, float* out, fgt_stream_t stream);

/* CorrBlock.__call__ (RAFT/corr.py:29-50) + bilinear_sampler (RAFT/utils/utils.py:57-71): for each of
 * n_pix source pixels and each pyramid level l (volume level_ptrs[l] = [n_pix, h_l, w_l] fp32), the
 * (2r+1)^2 zero-padded bilinear samples around coords/2^l. Output split-bf16 [n_pix, out_pitch],
 * channel = l*(2r+1)^2 + a*(2r+1) + b with a offsetting x and b offsetting y (reference order).
 * level_ptrs_host / level_h_host / level_w_host are HOST arrays of `levels` entries.
 * out_plane == 0: the output is single-plane fp16 [n_pix, out_pitch] (mixed precision). */
int fgt_corr_lookup(const float* const* level_ptrs_host, const int* level_h_host, const int* level_w_host,
                    int levels, int radius, const float* coords, int n_pix, int out_pitch, void* out_hi,
                    long long out_plane, fgt_stream_t stream);

/* coords += delta (delta may be NULL) for n image pairs, coords/delta [n*h*w, 2]; writes
 * flow = coords - pixel grid as NCHW fp32 [n,2,h,w] and, if x_hi != NULL, as channels
 * [x_chan, x_chan+1] of the split GRU-input buffer (RAFT/raft.py:127-132); x_plane == 0: x is single-plane fp16.
 * delta_f16 = 1 rounds delta to fp16 before the add (mixed precision: the flow head's output is an fp16 tensor under
 * autocast); 0 adds it as given. */
int fgt_raft_flow_update(float* coords, const float* delta, int delta_f16, int n, int h, int w, float* flow_nchw,
                         void* x_hi, long long x_plane, int x_pitch, int x_chan, fgt_stream_t stream);

/* fp16 [n] -> split-bf16 [2][n] (hi plane at out_hi, lo plane out_plane elements later), exact for every fp16 value.
 * Mixed-precision RAFT: the feature net's fp16 output feeds the 3-term correlation GEMM. n and out_plane multiples of
 * 8, both buffers 16-byte aligned. */
int fgt_f16_to_split(const void* src, long long n, void* out_hi, long long out_plane, fgt_stream_t stream);

/* RAFT.upsample_flow (RAFT/raft.py:73-84): mask [n*h*w, 576] fp32, flow [n,2,h,w] -> up-sampled flow
 * [n, 2, 8h, 8w]. */
int fgt_convex_upsample(const float* mask, const float* flow_nchw, int n, int h, int w, float* out,
                        fgt_stream_t stream);

/* upflow8 (RAFT/utils/utils.py:80-82), the small model's upsampling: 8 * F.interpolate(flow, (8h, 8w), bilinear,
 * align_corners=True), flow [n,2,h,w] -> out [n,2,8h,8w] fp32, ATen's source-index arithmetic (scale 0 for h or w 1). */
int fgt_upflow8(const float* flow_nchw, int n, int h, int w, float* out, fgt_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Flow-guided gradient propagation (tool/get_flowNN_gradient.py:11-534, Nonlocal=False). Dense state
 * per NN slot (0 = backward-flow neighbours, 1 = forward-flow neighbours), all [N,H,W]:
 *   nn_y, nn_x (double), nn_t (int, -1 = none), have (uint8: 1 = neighbour found), cuv (double[2]).
 * mask is uint8 [N,H,W]; flows are float [H,W,2] = (u, v) of one frame pair; gradients float [N,H,W,3].
 * ------------------------------------------------------------------------------------------ */

/* One frame `t` of one pass (neighbour frame tn = t-1 for slot 0, t+1 for slot 1); `flow_step` moves
 * t -> tn, `flow_back` tn -> t. Replaces the loop bodies at get_flowNN_gradient.py:76-235 / 241-370 and
 * BFconsistCheck / FBconsistCheck / consistCheck (tool/utils/common_utils.py:187-254). */
int fgt_prop_step(const uint8_t* mask, const float* flow_step, const float* flow_back, int H, int W, int t, int tn,
                  double thres, double* nn_y, double* nn_x, int* nn_t, uint8_t* have, double* cuv,
                  fgt_stream_t stream);

/* In-place gather for source frame s (get_flowNN_gradient.py:378-435 + interp, common_utils.py:149-171):
 * cv2.remap-compatible bilinear sampling (1/32-pixel fixed-point coordinates, zero border). */
int fgt_prop_gather(const uint8_t* mask, const double* nn_y, const double* nn_x, const int* nn_t, int N, int H, int W,
                    int s, float* gx, float* gy, fgt_stream_t stream);

/* Confidence-weighted fusion of the two candidates and the still-to-fill mask (get_flowNN_gradient.py:440-532). */
int fgt_prop_fuse(const uint8_t* mask, const uint8_t* have0, const uint8_t* have1, const double* cuv0,
                  const double* cuv1, int N, int H, int W, double alpha, const float* gx_bn, const float* gy_bn,
                  const float* gx_fn, const float* gy_fn, float* gx, float* gy, uint8_t* tofill, fgt_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* FGT_B200_H_ */
