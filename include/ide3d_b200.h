/*
 * ide3d_b200 -- C-ABI of the H100-native IDE-3D hot path (libide3d_b200.so).
 *
 * Drop-in boundary.  Every entry point below replaces one pybind11/Python boundary of the
 * reference (citations are relative to the reference tree, MrTornado24/IDE-3D @ b2ee653):
 *
 *   ide3d_bias_act            torch_utils/ops/bias_act.cpp:32       (params: bias_act.h:12-31)
 *   ide3d_modconv_epilogue    torch_utils/ops/fma.py:15 + bias_act.cpp:32 fused (extension; inversion/networks.py:104-105,512)
 *   ide3d_modconv_epilogue_rgb  the same, plus the next `x * styles` and the block's ToRGB 1x1 convolution (extension; :100, :700-707)
 *   ide3d_upfirdn2d           torch_utils/ops/upfirdn2d.cpp:16      (params: upfirdn2d.h:14-40)
 *   ide3d_upfirdn2d_add       upfirdn2d + the skip-connection add (extension; inversion/networks.py:841-844)
 *   ide3d_upfirdn2d_epilogue  upfirdn2d + demodulation/noise/bias_act tail (extension; inversion/networks.py:104-105,512)
 *   ide3d_filtered_lrelu      torch_utils/ops/filtered_lrelu.cpp:16 (params: filtered_lrelu.h:14-51)
 *   ide3d_filtered_lrelu_act  torch_utils/ops/filtered_lrelu.cpp:213 (params: filtered_lrelu.h:53-68)
 *   ide3d_initial_rays        training/volumetric_rendering.py:77   get_initial_rays_trig
 *   ide3d_transform_points    training/volumetric_rendering.py:99,108  perturb_points + transform_sampled_points
 *   ide3d_sample_triplane     dnnlib/util.py:580                    sample_from_triplane
 *   ide3d_integrate           training/volumetric_rendering.py:34   fancy_integration
 *   ide3d_sample_pdf          training/volumetric_rendering.py:224  sample_pdf
 *   ide3d_mask2color          dnnlib/seg_tools.py:75                mask2color
 *   ide3d_video_frames        gen_videos.py:129-139 + layout_grid :24-38  image_seg / image_depth frames, fused
 *   ide3d_image_strips        gen_images.py:109-116  mask2color + the two save_image strips (make_grid + uint8), fused
 *   ide3d_sample_voxel        generator.synthesis.renderer.sample_voxel (call site extract_shapes.py:146)
 *   ide3d_sigma_grid          extract_shapes.py:99-150 (create_samples :74-96 + the sample_voxel loop :144-148)
 *   ide3d_raymarch_fwd        the per-frame chain the generator class runs: rays -> jitter -> world
 *                             transform -> 2x tri-plane gather -> decoder MLP -> compositing, fused.
 *   ide3d_planes_to_nhwc      layout helper for the two kernels above (no reference counterpart).
 *   ide3d_mesh_normals        render_mesh.py:36-42  smooth vertex normals (trimesh / pyrender smooth=True)
 *   ide3d_raster              render_mesh.py:44-61  shaded frames of the mesh (pyrender OffscreenRenderer)
 *   ide3d_noise_reg           inversion/training/projectors/w_projector_ide3d.py:113-122  noise regulariser (+ its gradient)
 *   ide3d_noise_normalize     inversion/training/projectors/w_projector_ide3d.py:138-142  noise renormalisation
 *   ide3d_seg_xent_fwd/_bwd   semantic-mask loss of the projector (extension): cross-entropy of the upsampled logits
 *   ide3d_seg_xent_*_ac       apps/finetune_hybrid_encoder.py:171-174  the same with align_corners=True (BiSeNet's upsampling)
 *   ide3d_lpips_fwd/_bwd      inversion/criteria/lpips/lpips.py:29-35 + utils.py:6-8  LPIPS head over all tapped layers (pivotal tuning)
 *   ide3d_feat_l1_fwd/_bwd    apps/train_hybrid_encoder.py:143-152  the VGG loss's L1 over all tapped layers (encoder training)
 *   ide3d_seg_stem            Painter/run_UI.py:290-295 + inversion/networks.py:1638-1646  one-hot mask -> stem, conv1 and skip of the
 *                             HybridEncoder's geometry branch, from the class ids through per-class tables (extension)
 *   ide3d_seg_stem_bwd        its gradients w.r.t. the three layers' weights (encoder fine-tuning)
 *   ide3d_seg_labels          the generator's class ids at image resolution (extension; the starting mask of an edit)
 *   ide3d_seg_labels_ac       dnnlib/seg_tools.py:101-117  argmax of BiSeNet's align_corners=True upsampling
 *   ide3d_knn_kth_dist        metrics/precision_recall.py:17-52  k-th nearest-neighbour distance of every manifold row
 *   ide3d_knn_within          metrics/precision_recall.py:53-60  does a probe fall inside some manifold point's radius
 *   ide3d_spectrum_accum      avg_spectra.py:161-166  average power spectrum `calc`: whitening, window, zero-padded fftn, |X|^2
 *   ide3d_spectrum_finalize   avg_spectra.py:167  the division by the image count, in the reference's [P, P] bin order
 *   ide3d_image_moments       avg_spectra.py:126-131  `stats`: sums of 1, x and x^2, as exact integers
 *   ide3d_resample_u8         dataset_tool.py:226-256  PIL.Image.resize(LANCZOS) of 8-bit L / RGB images (Pillow's ImagingResample)
 *   ide3d_style_grid          apps/style_mixing.py:100-153  the uint8 conversion and the canvas paste loop of the style-mixing grid
 *   ide3d_viz_image           viz/renderer.py:369-393  the display tail: statistics, depth normalisation, channel window, inf-norm, dB gain,
 *                             uint8 image
 *   ide3d_viz_fft             viz/renderer.py:395-406  the FFT panel: mean removal, Kaiser window, |2-D DFT|^2 over channels, roll, dB,
 *                             colormap
 *
 * Conventions
 *   - plain C: raw device pointers, sizes, strides (in ELEMENTS), a cudaStream_t passed as void*.
 *   - the caller owns every buffer; the library never allocates or frees device memory, keeps no
 *     global device state (filters/weights travel as kernel arguments or per-launch shared memory,
 *     unlike filtered_lrelu.cu:77-78), and is therefore thread- and stream-safe.
 *   - kernels run on the CURRENT device of the calling thread, on the given stream.
 *   - return value: IDE3D_OK, or a negative code; nothing is thrown across the ABI.
 *     IDE3D_UNSUPPORTED (-1) keeps the reference meaning "no specialised kernel, caller may fall
 *     back to the generic composition" (filtered_lrelu.cpp:52-56).
 *   - ide3d_last_error() returns a thread-local, human-readable message for the last failure.
 */
#ifndef IDE3D_B200_H_
#define IDE3D_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IDE3D_ABI_VERSION 1

enum ide3d_status {
    IDE3D_OK = 0,
    IDE3D_UNSUPPORTED = -1,   /* no kernel for this configuration (caller may fall back) */
    IDE3D_INVALID = -2,       /* malformed arguments (the reference raises via TORCH_CHECK) */
    IDE3D_CUDA_ERROR = -3     /* launch / runtime failure; see ide3d_last_error() */
};

enum ide3d_dtype { IDE3D_F32 = 0, IDE3D_F16 = 1, IDE3D_F64 = 2 };
/* Mixed-format code of the modulated-convolution epilogues and the skip add: IDE3D_DTYPE2(a, b) names two dtypes where
 * those entry points take one.  Which tensors are `a` and which `b` is stated at each entry point; a plain ide3d_dtype
 * keeps its meaning (every tensor of that dtype).  Accepted pairs are listed per entry point; others are IDE3D_UNSUPPORTED. */
#define IDE3D_DTYPE2(a, b) ((a) | (((b) + 1) << 4))

typedef void* ide3d_stream_t; /* cudaStream_t */

int ide3d_abi_version(void);
const char* ide3d_last_error(void);
/* number of kernel launches issued by this library since load (all threads); for bench bookkeeping */
uint64_t ide3d_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * bias_act: y = clamp(gain * act(x + b)) and its 1st/2nd-order gradient forms.
 * Mirrors bias_act(x,b,xref,yref,dy,grad,dim,act,alpha,gain,clamp) (bias_act.cpp:32); the
 * caller resolves `dim` into size_b / step_b = x.stride(dim) exactly like bias_act.cpp:70-73.
 * x, xref, yref, dy, y: [size_x] dense, same dtype/layout; b: [size_b] or NULL.
 * act: 1 linear 2 relu 3 lrelu 4 tanh 5 sigmoid 6 elu 7 selu 8 softplus 9 swish (bias_act.py:21-31)
 * clamp < 0 disables clamping. */
int ide3d_bias_act(const void* x, const void* b, const void* xref, const void* yref, const void* dy,
                   void* y, int dtype, int grad, int act, float alpha, float gain, float clamp,
                   int64_t size_x, int64_t size_b, int64_t step_b, ide3d_stream_t stream);

/* Extension (no reference plugin): the tail of an activation-scaled modulated convolution in one pass,
 *     y = bias_act(x * scale[n,c] + noise[(n),h,w], b[c], act, alpha, gain, clamp)
 * i.e. fma.fma (inversion/networks.py:104-105; torch_utils/ops/fma.py:15) followed by bias_act (:512).
 * x, y: [n, c, h*w] dense (channels_last = 0) or [n, h*w, c] dense (channels_last = 1), dtype as bias_act;
 * scale [n*c], noise [noise_batch * h*w] (noise_batch = 1 or n), b [c]: same dtype as x, each may be NULL.
 * Optional second output y2 = y * scale2[n,c] (scale2 [n*c]; y2 like y): the style modulation `x * styles` that opens
 * the NEXT modulated convolution (inversion/networks.py:100), written in the same pass; y may then be NULL.
 * dtype IDE3D_DTYPE2(IDE3D_F32, IDE3D_F16) (channels_last only): x and every operand float32, y and y2 fp16 (each value
 * computed in float32 and rounded once) -- the fp16 input of a convolution; act 1 (linear) or 3 (lrelu).
 * Forward only.  IDE3D_UNSUPPORTED when the vector width does not divide h*w (NCHW) or c (channels_last). */
int ide3d_modconv_epilogue(const void* x, const void* scale, const void* noise, const void* b, void* y,
                           const void* scale2, void* y2, int dtype, int act, float alpha, float gain, float clamp,
                           int64_t n, int64_t c, int64_t hw, int64_t noise_batch, int channels_last,
                           ide3d_stream_t stream);

/* Extension: the same epilogue (channels_last, float32) with the layers that consume it folded into the pass.
 * t = bias_act(x * scale[n,c] + noise[(n),h,w], b[c], act, alpha, gain, clamp) as above, then any subset of
 *     y   = t * yscale[n,c]  (yscale NULL: y = t)      e.g. the next block's `x * styles` of its first convolution
 *     y2  = t * scale2[n,c]                             as ide3d_modconv_epilogue
 *     rgb[n, o, h*w] = sum_c wrgb[o,c] * srgb[n,c] * t[n,h*w,c] + brgb[o]   for o < rgb_channels (1..4), dense NCHW:
 *         the block's ToRGB layer (modulated 1x1 convolution without demodulation, inversion/networks.py:700-707)
 * x, y, y2: [n, h*w, c]; scale, yscale, scale2, srgb [n*c]; wrgb [rgb_channels * c]; b [c]; brgb [rgb_channels] (may be NULL).
 * Each pixel's rgb sum runs in a fixed order without atomics (bit-identical reruns).  Forward only.
 * dtype IDE3D_F32: every tensor float32.  IDE3D_DTYPE2(IDE3D_F16, IDE3D_F16): x, y and y2 fp16, every other operand and rgb
 * float32; the arithmetic is float32 and each fp16 output is the float32 value rounded once.
 * IDE3D_UNSUPPORTED for other dtypes, and unless c % 4 == 0 and c <= 512. */
int ide3d_modconv_epilogue_rgb(const void* x, const void* scale, const void* noise, const void* b, const void* yscale,
                               void* y, const void* scale2, void* y2, const void* wrgb, const void* srgb, const void* brgb,
                               void* rgb, int64_t rgb_channels, int dtype, int act, float alpha, float gain, float clamp,
                               int64_t n, int64_t c, int64_t hw, int64_t noise_batch, ide3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * upfirdn2d: pad -> zero-upsample -> FIR -> decimate.  Field meaning = upfirdn2d_kernel_params
 * (upfirdn2d.h:14-40); sizes/strides in the reference order [W, H, C, N]; strides in elements.
 * f is float32 [f_h, f_w] with element strides f_stride_{h,w}.  flip != 0 = correlation. */
typedef struct ide3d_upfirdn2d_params {
    const void* x;
    const float* f;
    void* y;
    int dtype;
    int up_x, up_y, down_x, down_y, pad_x0, pad_y0;
    int flip;
    float gain;
    int in_w, in_h, in_c, in_n;
    int64_t in_stride_w, in_stride_h, in_stride_c, in_stride_n;
    int f_w, f_h;
    int64_t f_stride_w, f_stride_h;
    int out_w, out_h;
    int64_t out_stride_w, out_stride_h, out_stride_c, out_stride_n;
} ide3d_upfirdn2d_params;
int ide3d_upfirdn2d(const ide3d_upfirdn2d_params* p, ide3d_stream_t stream);

/* Extension (no reference plugin): the skip-connection step of a 'skip' synthesis block in one pass,
 *     y = upfirdn2d(x, f, ...) + add + bias[c]
 * i.e. upsample2d of the running image (inversion/networks.py:841) fused with the `img.add_(y)` that follows (:844) and
 * with the ToRGB bias (:707).  add: same dtype, logical shape of y, element strides add_stride_{n,h,w}, channel stride 1
 * (it may be a channel slice of a wider channels_last tensor); bias [c] or NULL.  p->dtype IDE3D_DTYPE2(IDE3D_F32, IDE3D_F16):
 * x, y and bias float32, add fp16 (the output of an fp16 convolution).  Only the channels_last patch kernel
 * implements it (x, y channels_last, C % 4 == 0, 4x4 filter, up/down in {1,2}); otherwise IDE3D_UNSUPPORTED. */
int ide3d_upfirdn2d_add(const ide3d_upfirdn2d_params* p, const void* add, int64_t add_stride_n, int64_t add_stride_h,
                        int64_t add_stride_w, const void* bias, ide3d_stream_t stream);

/* Extension (no reference plugin): upfirdn2d with the modulated-convolution tail applied to the filter output before it is
 * stored -- the up=2 SynthesisLayer is conv_transpose2d -> FIR -> x*dcoefs + noise -> bias_act (inversion/networks.py:104-105,
 * :512; conv2d_resample.py:112-126) and this runs everything after the transposed convolution in one pass:
 *     v  = clamp(gain * act(fir * scale[n,c] + noise[(n),oy,ox] + b[c]))     act: 1 linear, 3 lrelu(alpha)
 *     y  = v                      (params->y; may be NULL when only y2 is wanted)
 *     y2 = v * scale2[n,c]        (optional: the next layer's style modulation, layout of y)
 * scale, b, scale2: dtype of x, [n*c] / [c] / [n*c]; noise: dtype of x, [noise_batch, out_h, out_w] dense; any may be NULL.
 * p->dtype IDE3D_DTYPE2(IDE3D_F16, IDE3D_F16): x, y and y2 fp16; scale, noise, b, scale2, the filter and the arithmetic float32,
 * each fp16 output rounded once from the float32 value.
 * Same kernel restrictions as ide3d_upfirdn2d_add (channels_last, C % 4 == 0, 4x4 filter); otherwise IDE3D_UNSUPPORTED. */
typedef struct ide3d_fir_epilogue {
    const void *scale, *noise, *b, *scale2;
    void* y2;
    int act;
    float alpha, gain, clamp;      /* clamp < 0: off */
    int64_t noise_batch;           /* 1 or n */
} ide3d_fir_epilogue;
int ide3d_upfirdn2d_epilogue(const ide3d_upfirdn2d_params* p, const ide3d_fir_epilogue* e, ide3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * filtered_lrelu: bias -> up-FIR -> gain*lrelu*clamp (+ 2-bit sign tensor) -> down-FIR, fused.
 * Field meaning = filtered_lrelu_kernel_params (filtered_lrelu.h:14-51).  fu/fd are float32, 1-D
 * (separable, *_h == 0) or 2-D.  s is the uint8 sign tensor [N,C,s_h,s_w/4] (filtered_lrelu.cpp:82-96)
 * written when write_signs, read when read_signs, ignored when both 0.  Returns IDE3D_UNSUPPORTED
 * for configurations without a fused kernel (the caller then composes upfirdn2d +
 * ide3d_filtered_lrelu_act exactly like filtered_lrelu.py:223-229). */
typedef struct ide3d_filtered_lrelu_params {
    const void* x;
    const void* b;          /* [C] same dtype as x, or NULL */
    const float* fu;
    const float* fd;
    void* y;
    unsigned char* s;
    int dtype;
    int up, down;
    int fu_w, fu_h;         /* fu_h == 0 -> separable 1-D filter of fu_w taps */
    int fd_w, fd_h;
    int pad_x0, pad_y0;
    int flip;
    float gain, slope, clamp;
    int x_w, x_h, x_c, x_n;
    int64_t x_stride_w, x_stride_h, x_stride_c, x_stride_n;
    int y_w, y_h;
    int64_t y_stride_w, y_stride_h, y_stride_c, y_stride_n;
    int s_w, s_h;           /* sign tensor extent in ELEMENTS (s_w multiple of 4) */
    int s_ofs_x, s_ofs_y;
    int write_signs, read_signs;
} ide3d_filtered_lrelu_params;
int ide3d_filtered_lrelu(const ide3d_filtered_lrelu_params* p, ide3d_stream_t stream);

/* In-place activation + sign handling of the generic fallback (filtered_lrelu.cpp:213). */
typedef struct ide3d_filtered_lrelu_act_params {
    void* x;                /* in/out */
    unsigned char* s;
    int dtype;
    int x_w, x_h, x_c, x_n;
    int64_t x_stride_w, x_stride_h, x_stride_c, x_stride_n;
    int s_w, s_h;
    int s_ofs_x, s_ofs_y;
    float gain, slope, clamp;
    int write_signs, read_signs;
} ide3d_filtered_lrelu_act_params;
int ide3d_filtered_lrelu_act(const ide3d_filtered_lrelu_act_params* p, ide3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Volume renderer.
 * A tri-plane tensor is [N, 3*32, H, W] float32: planes (xy, yz, xz) of 32 channels each
 * (dnnlib/util.py:586-596), addressed through element strides so that both NCHW and
 * channels_last tensors are accepted.  The fused kernels take their fast path when stride_c == 1
 * (one texel = one 128-byte line per plane); otherwise convert once with ide3d_planes_to_nhwc. */
typedef struct ide3d_triplane {
    const float* data;
    int n, h, w;            /* batch, plane height, plane width */
    int64_t stride_n, stride_c, stride_h, stride_w;
} ide3d_triplane;

/* Decoder MLP, as a list of independent heads.  Each head reads the 32 texture features
 * (in_sel 0), the 32 shape features (in_sel 1) or their concatenation (in_sel 2, 64 inputs):
 *     h = softplus(W1 @ f + b1)   W1 [hidden, in] row-major
 *     o[out_offset : out_offset+out_count] = W2 @ h + b2   W2 [out_count, hidden] row-major
 * Output channels not covered by any head are 0.  Channel 51 (the last of 52) is sigma
 * (extract_shapes.py:146-147).  Fused kernels exist for:
 *     1 head : in_sel 2, out 0..52,           hidden in {64, 128}
 *     3 heads: (tex -> 0..32), (seg -> 32..51), (seg -> 51..52), hidden 64 each
 * anything else returns IDE3D_UNSUPPORTED. */
typedef struct ide3d_mlp_head {
    int in_sel, hidden, out_offset, out_count;
    const float *w1, *b1, *w2, *b2;
} ide3d_mlp_head;
typedef struct ide3d_decoder {
    int num_heads;
    ide3d_mlp_head heads[4];
} ide3d_decoder;

/* ZVALS: jitter_u holds the depth of every sample itself, [N, R, S] ascending along S (the merged coarse + importance samples of
 * a hierarchical second pass, volumetric_rendering.py:224-265): point = ray direction * z, no linspace, no jitter. */
enum ide3d_jitter { IDE3D_JITTER_NONE = 0, IDE3D_JITTER_TENSOR = 1, IDE3D_JITTER_HASH = 2, IDE3D_JITTER_ZVALS = 3 };
enum ide3d_clamp { IDE3D_CLAMP_SOFTPLUS = 0, IDE3D_CLAMP_RELU = 1 };
/* AUTO: tensor cores when the decoder / layout allows, else CUDA cores.  FP32: CUDA-core FFMA, plain fp32.
 * TC: wgmma tensor cores, every product as bf16 hi*hi + hi*lo + lo*hi with fp32 accumulation (16-bit operand
 * mantissas); IDE3D_UNSUPPORTED if the decoder shape or plane layout has no tensor-core kernel. */
enum ide3d_precision { IDE3D_PRECISION_AUTO = 0, IDE3D_PRECISION_FP32 = 1, IDE3D_PRECISION_TC = 2 };

typedef struct ide3d_raymarch_params {
    ide3d_triplane tex, seg;
    ide3d_decoder dec;
    const float* cam2world;     /* [N,16] row-major 4x4 (c[:, :16], gen_images.py:105-107) */
    int n;                      /* frames */
    int res_w, res_h;           /* neural render resolution (64 x 64) */
    int num_steps;              /* depth samples per ray */
    float fov_deg, ray_start, ray_end;
    float box_scale;            /* world -> plane grid units (2 / box_warp) */
    int jitter_mode;            /* ide3d_jitter */
    const float* jitter_u;      /* [N, R, S] uniforms in [0,1) when jitter_mode == TENSOR; sample depths when ZVALS */
    uint64_t jitter_seed;       /* when jitter_mode == HASH */
    int clamp_mode;             /* ide3d_clamp */
    int last_back, white_back;
    float max_depth;            /* 0 = off (volumetric_rendering.py:66) */
    int fill_weight;            /* fill_mode == 'weight' (:71-72) */
    float noise_std;            /* with noise != NULL: sigma += noise_std * noise (:45) */
    const float* noise;         /* [N, R, S] standard normal, or NULL */
    float* out_feat;            /* [N, R, 51]  composited colour features + semantic logits */
    float* out_depth;           /* [N, R] */
    float* out_weights;         /* [N, R, S] or NULL */
    int precision;              /* ide3d_precision: how the decoder MLP is evaluated */
    int views;                  /* frames per plane set: frame f reads plane set f / views (tex.n == seg.n == n / views);
                                   0 or 1: one plane set per frame */
    const uint64_t* jitter_seeds; /* [n] device array or NULL.  HASH jitter of frame f then uses jitter_seeds[f] and the frame-local
                                   sample index, so frame f equals a one-frame launch with jitter_seed = jitter_seeds[f] */
} ide3d_raymarch_params;
int ide3d_raymarch_fwd(const ide3d_raymarch_params* p, ide3d_stream_t stream);

/* Backward of ide3d_raymarch_fwd: what autograd derives in the reference from grid_sample (grid_sample_gradfix.py:55-61), the decoder
 * layers and fancy_integration (volumetric_rendering.py:34-74), in one kernel that recomputes the per-sample chain instead of storing it.
 * p: the forward's parameters (outputs ignored).  grad_feat [N,R,51], grad_depth [N,R] or NULL.  grad_tex / grad_seg: fp32 buffers with
 * the planes' (channels-last) strides, ZERO-INITIALISED by the caller, accumulated into with red.global.add; either may be NULL.
 * grad_params: NULL, or 12 pointers {dW1, db1, dW2, db2} x 3 heads (dense, the heads' shapes), zero-initialised, accumulated into.
 * No gradient for cam2world / jitter / noise.  IDE3D_UNSUPPORTED for decoders other than the three-head one, NCHW planes, > 256 samples. */
int ide3d_raymarch_bwd(const ide3d_raymarch_params* p, const float* grad_feat, const float* grad_depth, float* grad_tex,
                       float* grad_seg, float* const* grad_params, ide3d_stream_t stream);

/* ide3d_raymarch_bwd plus the gradient w.r.t. the camera: grad_cam2world [N,16] fp32 (row-major 4x4 per frame, like cam2world),
 * ZERO-INITIALISED by the caller and accumulated into; rows 0..2 receive dL/dM, row 3 stays 0.  The sample depths (linspace + jitter,
 * or the ZVALS tensor) do not depend on the camera.  grad_cam2world == NULL behaves exactly like ide3d_raymarch_bwd, and the other
 * arguments, the validation and the unsupported configurations are those of ide3d_raymarch_bwd; grad_tex, grad_seg and grad_params may
 * all be NULL (camera-only refinement). */
int ide3d_raymarch_bwd_cam(const ide3d_raymarch_params* p, const float* grad_feat, const float* grad_depth, float* grad_tex,
                           float* grad_seg, float* const* grad_params, float* grad_cam2world, ide3d_stream_t stream);

/* sample_voxel: decode `points` [N, P, 3] (world units) -> out [N, P, 52], or, with sigma_only,
 * out [N, P] holding channel 51 only. */
int ide3d_sample_voxel(const ide3d_triplane* tex, const ide3d_triplane* seg, const ide3d_decoder* dec,
                       const float* points, int64_t num_points, float box_scale, int sigma_only,
                       float* out, ide3d_stream_t stream);

/* sigma grid for extract_shapes: generates the points of 0.9 * create_samples(N, origin, cube) in
 * the kernel (including the float-division index quirk, extract_shapes.py:84-86) for flat voxel
 * indices [first, first + count) of every batch item and writes sigma to out [n, count]. */
int ide3d_sigma_grid(const ide3d_triplane* tex, const ide3d_triplane* seg, const ide3d_decoder* dec,
                     int grid_n, const float voxel_origin[3], float cube_length, float pre_scale,
                     float box_scale, int64_t first, int64_t count, float* out, ide3d_stream_t stream);

/* [N, C, H, W] (any strides) -> dense [N, H, W, C] float32. */
int ide3d_planes_to_nhwc(const float* src, int n, int c, int h, int w, int64_t stride_n, int64_t stride_c,
                         int64_t stride_h, int64_t stride_w, float* dst, ide3d_stream_t stream);

/* ---- stand-alone stages (the reference's free functions on materialised tensors) ---- */

/* get_initial_rays_trig: points [n,R,S,3], z_vals [n,R,S], rays_d_cam [n,R,3]. */
int ide3d_initial_rays(int n, int num_steps, float fov_deg, int res_w, int res_h, float ray_start,
                       float ray_end, float* points, float* z_vals, float* rays_d_cam,
                       ide3d_stream_t stream);

/* perturb_points + the camera transform of transform_sampled_points.  u may be NULL (no jitter).
 * In: points [n,R,S,3], z_vals [n,R,S], dirs [n,R,3], cam2world [n,16].
 * Out: points_world [n,R,S,3], z_out [n,R,S], dirs_world [n,R,3], origins [n,R,3]. */
int ide3d_transform_points(const float* points, const float* z_vals, const float* dirs, const float* u,
                           const float* cam2world, int n, int num_rays, int num_steps, float* points_world,
                           float* z_out, float* dirs_world, float* origins, ide3d_stream_t stream);

/* sample_from_triplane: coords [N, P, 3] in grid units -> out [N*P, 32]. */
int ide3d_sample_triplane(const ide3d_triplane* planes, const float* coords, int64_t num_points,
                          float* out, ide3d_stream_t stream);

/* fancy_integration on a materialised rgb_sigma [n,R,S,C] (sigma = last channel).
 * Out: rgb [n,R,C-1], depth [n,R], weights [n,R,S]. */
int ide3d_integrate(const float* rgb_sigma, const float* rays_d_cam, const float* z_vals, const float* noise,
                    float noise_std, int n, int num_rays, int num_steps, int channels, int clamp_mode,
                    int last_back, int white_back, float max_depth, int fill_weight, float* rgb,
                    float* depth, float* weights, ide3d_stream_t stream);

/* sample_pdf: bins [R, S+1], weights [R, S], u [R, n_imp] -> samples [R, n_imp]. */
int ide3d_sample_pdf(const float* bins, const float* weights, const float* u, int num_rays, int num_bins,
                     int n_importance, float eps, float* samples, ide3d_stream_t stream);

/* mask2color (dnnlib/seg_tools.py:75-82): per pixel argmax over the c semantic logits (first maximum wins, like
 * torch.argmax) and colour look-up, one pass.  masks [n, c, h, w] float32 with element strides; lut [c, 3] float32 (the
 * COLOR_MAP rows, seg_tools.py:13-32); out [n, 3, h, w] float32 dense NCHW -- or, with out_u8 != 0, uint8 (the
 * `.to(torch.uint8)` that follows in gen_videos.py:24-38 folded in). */
int ide3d_mask2color(const float* masks, int n, int c, int h, int w, int64_t stride_n, int64_t stride_c, int64_t stride_h,
                     int64_t stride_w, const float* lut, void* out, int out_u8, ide3d_stream_t stream);

/* Video frames of gen_videos.py's image_seg / image_depth modes (gen_videos.py:129-139), in the uint8 form layout_grid hands to the
 * video writer ((x * 127.5 + 128).clamp(0, 255).to(uint8), :24-38), straight from the synthesis outputs.
 *   image [n, 3, height, width] fp32, element strides (NCHW or channels-last).
 *   IDE3D_FRAMES_IMAGE_SEG:   out [n, 3, height, 2 * width]; left half the image, right half the colour of the argmax class (first
 *       maximum, NaN counts as maximal; lut [seg_c, 3] fp32, the COLOR_MAP rows) of the logits seg [n, seg_c, seg_h, seg_w] (fp32, element
 *       strides) upsampled per pixel to height x width by interpolate(mode='bilinear', align_corners=False).  The upsampled logits are not
 *       stored anywhere.
 *   IDE3D_FRAMES_IMAGE_DEPTH: out [n, 3, height, width]; per frame t = -image, ((t - min t) / (max t - min t)) * 2 - 1.  Two launches;
 *       scratch holds n * IDE3D_FRAMES_PARTIALS * 2 floats of partial minima / maxima.  A constant frame divides 0 by 0, as the
 *       reference does.
 * out is dense.  Every operation is rounded separately, as the reference's torch ops are.  Limits: n <= 65535. */
#define IDE3D_FRAMES_PARTIALS 64
enum ide3d_frames_mode { IDE3D_FRAMES_IMAGE_SEG = 1, IDE3D_FRAMES_IMAGE_DEPTH = 2 };
typedef struct ide3d_frames_params {
    const float* image;
    int n, height, width;
    int64_t image_stride_n, image_stride_c, image_stride_h, image_stride_w;
    const float* seg;           /* IMAGE_SEG only */
    int seg_c, seg_h, seg_w;
    int64_t seg_stride_n, seg_stride_c, seg_stride_h, seg_stride_w;
    const float* lut;           /* IMAGE_SEG only */
    int mode;                   /* ide3d_frames_mode */
    uint8_t* out;
    float* scratch;             /* IMAGE_DEPTH only */
} ide3d_frames_params;
int ide3d_video_frames(const ide3d_frames_params* p, ide3d_stream_t stream);

/* The two PNG strips gen_images.py writes per seed (gen_images.py:109-116), in the uint8 HWC form PIL saves, straight from the synthesis
 * outputs of its `views` yaws:
 *   image [seeds * views, 3, height, width] fp32, element strides; row s * views + j is view j of seed s.
 *   seg   [seeds * views, seg_c, seg_h, seg_w] fp32, element strides: the render-resolution logits, upsampled per pixel to height x width
 *         by interpolate(mode='bilinear', align_corners=False) and never stored.  lut [seg_c, 3] fp32 (the COLOR_MAP rows).
 *   out_image, out_seg: dense uint8 [seeds, strip_h, strip_w, 3].
 * Strip layout: torchvision's make_grid(nrow=8, padding=2, pad_value=0), one row of views (views <= 8): strip_h = height + 4,
 * strip_w = views * (width + 2) + 2, view j at row 2, column 2 + j * (width + 2), padding bytes 0; views == 1: the bare image
 * (strip_h = height, strip_w = width).
 * Image bytes: save_image(normalize=True, value_range=(-1, 1)): clamp(x, -1, 1) - (-1), / 2, * 255, + 0.5, clamp(0, 255), -> uint8, each
 * operation rounded separately; NaN gets the byte torch's device conversion writes.  Seg bytes: the COLOR_MAP bytes of the argmax class
 * (first maximum, NaN maximal) -- the save_image chain of (colour / 255 - 0.5) / 0.5 gives the colour back exactly.  Limits: seeds <= 65535. */
typedef struct ide3d_strips_params {
    const float* image;
    int seeds, views, height, width;
    int64_t image_stride_n, image_stride_c, image_stride_h, image_stride_w;
    const float* seg;
    int seg_c, seg_h, seg_w;
    int64_t seg_stride_n, seg_stride_c, seg_stride_h, seg_stride_w;
    const float* lut;
    uint8_t* out_image;
    uint8_t* out_seg;
} ide3d_strips_params;
int ide3d_image_strips(const ide3d_strips_params* p, ide3d_stream_t stream);

/* Marching cubes on a density grid (render_mesh.py:30-32 / dnnlib/geometry.py:282-286 call PyMCubes' marching_cubes on the host).
 * volume [nx, ny, nz] fp32 dense (index (x*ny + y)*nz + z); a corner is inside where value >= threshold.  Tables (device memory) come
 * from ide3d_b200/mesh.py::build_tables: ntri_table [256] int32, tri_table [256*16] int8 (edge triples, -1 terminated), edge_corner
 * [12*2] int32 (lower / upper corner of each cube edge).
 *   ide3d_mc_classify: counts[cell] = number of triangles of the cell, cell = (x*(ny-1) + y)*(nz-1) + z.
 *   ide3d_mc_emit:     offsets = inclusive scan of counts (int64); per emitted vertex k of triangle t: edge_ids[3t+k] = global id of the
 *                      cut grid edge ((lower corner flat index)*3 + axis), verts[(3t+k)*3 ..] = its position in index units. */
int ide3d_mc_classify(const float* volume, int nx, int ny, int nz, float threshold, const int* ntri_table, unsigned char* counts,
                      ide3d_stream_t stream);
int ide3d_mc_emit(const float* volume, int nx, int ny, int nz, float threshold, const signed char* tri_table, const int* edge_corner,
                  const unsigned char* counts, const int64_t* offsets, int64_t* edge_ids, float* verts, ide3d_stream_t stream);

/* Mesh rendering (render_mesh.py:36-67 draws the marching-cubes mesh with pyrender / OpenGL offscreen; this is a visibility-buffer
 * rasteriser instead, no graphics context).
 *
 * ide3d_mesh_normals: smooth vertex normals.  normals[v] = normalise(sum over the faces f of v, in adjacency order, of
 * cross(p1 - p0, p2 - p0)) -- the area-weighted face normals -- or (0, 0, 0) when the sum is zero.  vertices [V,3] fp32, triangles
 * [T,3] int32; the adjacency is CSR: the faces of vertex v are adj_faces[adj_offsets[v] .. adj_offsets[v+1]) (int32, ascending face
 * index is what ide3d_b200/mesh.py builds).  No atomics: the result is deterministic.
 *
 * ide3d_raster: F frames of one mesh in one call.  Camera: cam2world [F,16] row-major, RIGID (rotation + translation); OpenGL
 * convention (looks down -z, +y up), vertical field of view yfov_deg, aspect width / height, near plane znear, no far plane.
 * Image row 0 is the top, pixel centres at half-integers, one sample per pixel (no anti-aliasing), no culling.
 *   - screen positions are snapped to 1/256 pixel (round half to even); coverage by exact int64 edge functions with the top-left
 *     fill rule, so triangles sharing an edge cover each pixel centre on it exactly once;
 *   - a triangle is dropped when a vertex has view depth w < znear, or lies more than 16384 pixels outside the viewport (guard band);
 *   - visibility: per pixel the minimum of (bits of the fp32 view depth) << 32 | triangle index, i.e. the nearest surface, ties to the
 *     lower triangle index, independent of launch order;
 *   - shading, grey, two-sided headlight: c = base * clamp(ambient + diffuse * |n . l|, 0, 1), n the perspective-correct interpolated
 *     vertex normal (normalised), l the camera's view direction; stored as round(255 c) in all three channels.  background: 0..255.
 * Outputs: rgb uint8 [F,H,W,3]; ids int32 [F,H,W] (visible triangle, -1 for background) or NULL.
 * scratch: caller-owned device memory, 256-byte aligned, at least ide3d_raster_scratch_bytes(F, W, H, V, T) bytes (a key buffer of
 * 8 bytes per pixel, 16 bytes per frame and vertex, 8 bytes per frame and triangle); contents on entry do not matter.
 * Limits: 1 <= width, height <= 16384; V, T < 2^31; F * T < 2^32. */
typedef struct ide3d_raster_params {
    const float* vertices;      /* [V,3] */
    const int32_t* triangles;   /* [T,3] */
    const float* normals;       /* [V,3] (ide3d_mesh_normals) */
    const float* cam2world;     /* [F,16] */
    int64_t num_vertices, num_triangles;
    int num_frames, width, height;
    float yfov_deg, znear;
    float base, ambient, diffuse;
    int background;
    uint8_t* rgb;               /* [F,H,W,3] */
    int32_t* ids;               /* [F,H,W] or NULL */
    void* scratch;
    int64_t scratch_bytes;
} ide3d_raster_params;
int ide3d_mesh_normals(const float* vertices, const int32_t* triangles, int64_t num_vertices, const int32_t* adj_offsets,
                       const int32_t* adj_faces, float* normals, ide3d_stream_t stream);
/* bytes of scratch ide3d_raster needs; -1 for negative arguments */
int64_t ide3d_raster_scratch_bytes(int num_frames, int width, int height, int64_t num_vertices, int64_t num_triangles);
int ide3d_raster(const ide3d_raster_params* p, ide3d_stream_t stream);

/* Style vectors and demodulation coefficients of every modulated convolution of one synthesis call, two launches
 * (replaces per layer: FullyConnectedLayer.forward of the affine, inversion/networks.py:136-165 / :476, and the dcoefs
 * reduction of modulated_conv2d, :89-90).
 *   styles[style_off + n*in_ch + i] = ((affine_w[i,:] . ws[n, w_index, :]) * w_gain + affine_b[i] * b_gain) * out_scale
 *   dcoefs[dcoef_off + n*out_ch + o] = rsqrt(sum_i styles[n,i]^2 * wsq[o,i] + 1e-8)        (layers with wsq != NULL)
 * ws [n, num_ws, w_dim] fp32 dense; wsq[o,i] = sum over the kernel taps of weight[o,i,:,:]^2 (a constant of the weights). */
typedef struct ide3d_style_layer {
    const float* affine_w;      /* [in_ch, w_dim] */
    const float* affine_b;      /* [in_ch] or NULL */
    const float* wsq;           /* [out_ch, in_ch] or NULL (no demodulation: ToRGB) */
    float w_gain, b_gain;       /* FullyConnectedLayer runtime gains */
    float out_scale;            /* extra factor on the style (ToRGB weight_gain), 1 otherwise */
    int w_index;                /* which ws[:, w_index] feeds the layer */
    int in_ch, out_ch;
    int64_t style_off, dcoef_off;
} ide3d_style_layer;
int ide3d_style_plan(const float* ws, int n, int num_ws, int w_dim, const ide3d_style_layer* layers, int num_layers,
                     float* styles, float* dcoefs, ide3d_stream_t stream);

/* Noise regulariser of the projectors (inversion/training/projectors/w_projector_ide3d.py:113-122) over a table of `count` noise
 * buffers, each a dense fp32 [side, side] map (the SynthesisLayer.noise_const buffers).  Per buffer, at pyramid levels L = 0, 1, ...
 * (level L + 1 = avg_pool2d(level L, 2), stopping after the first level whose side is <= 8):
 *   reg = sum over buffers and levels of mean(n * roll(n, 1, W))^2 + mean(n * roll(n, 1, H))^2
 * ide3d_noise_reg writes reg to loss[0] (device).  With grad_scale (device scalar) != NULL it also writes, for every buffer,
 * grads[b] = grad_scale[0] * d reg / d bufs[b]: the sum over levels of (1/4)^L times the level-L gradient at the pixel's ancestor.
 * ide3d_noise_normalize renormalises every buffer in place (:138-142): buf -= mean(buf); buf *= rsqrt(mean(buf^2)).
 * Two launches (noise_reg) and one (noise_normalize), whatever the number of buffers; reductions run in a fixed order (no float
 * atomics), so two calls give bit-identical results.
 * scratch: device memory, 8-byte aligned, at least 128 + sum over buffers of sum_{L >= 1} (side >> L)^2 floats (the pyramid levels
 * above the buffer and one double per buffer); noise_normalize does not use it.
 * IDE3D_UNSUPPORTED for count > IDE3D_NOISE_MAX_BUFFERS or a side that is not a power of two in [1, 512]. */
#define IDE3D_NOISE_MAX_BUFFERS 64
typedef struct ide3d_noise_table {
    int count;
    int sides[IDE3D_NOISE_MAX_BUFFERS];
    float* bufs[IDE3D_NOISE_MAX_BUFFERS];
    float* grads[IDE3D_NOISE_MAX_BUFFERS];   /* noise_reg with grad_scale only */
    float* scratch;
    int64_t scratch_floats;
} ide3d_noise_table;
int ide3d_noise_reg(const ide3d_noise_table* t, float* loss, const float* grad_scale, ide3d_stream_t stream);
int ide3d_noise_normalize(const ide3d_noise_table* t, ide3d_stream_t stream);

/* Semantic-mask loss of the projector (extension): F.cross_entropy(interpolate(seg, (out_h, out_w), 'bilinear', align_corners=False),
 * mask), mean over the n * out_h * out_w pixels, without building the upsampled logits.  seg [n, classes, in_h, in_w] fp32, any
 * strides (e.g. the strided view G.synthesis(..., return_seg='raw') returns); mask uint8 [n, out_h, out_w] dense, values < classes.
 *   ide3d_seg_xent_fwd: per output pixel the bilinear logits (the rounding of ide3d_image_strips), their log-sum-exp -> lse
 *                       [n, out_h, out_w] (kept for the backward), loss[0] = mean(lse - logit[mask]).  partials: n * out_h doubles.
 *   ide3d_seg_xent_bwd: grad_seg [n, classes, in_h, in_w] dense = grad_loss[0] * the adjoint of the upsampling applied to
 *                       (softmax - onehot(mask)) / (n * out_h * out_w); every texel gathers the output pixels whose taps reach it.
 * No float atomics: both are deterministic.  Limits: classes <= 32; every tensor's element offsets fit 31 bits.
 * The mask is not validated on the device: a label >= classes is read as classes - 1 (F.cross_entropy would raise); callers check it. */
typedef struct ide3d_seg_xent_params {
    const float* seg;
    int n, classes, in_h, in_w;
    int64_t seg_stride_n, seg_stride_c, seg_stride_h, seg_stride_w;
    const uint8_t* mask;
    int out_h, out_w;
    float* lse;                 /* [n, out_h, out_w]: written by fwd, read by bwd */
    double* partials;           /* fwd: [n * out_h] */
    float* loss;                /* fwd: [1] */
    const float* grad_loss;     /* bwd: [1] */
    float* grad_seg;            /* bwd: [n, classes, in_h, in_w] */
} ide3d_seg_xent_params;
int ide3d_seg_xent_fwd(const ide3d_seg_xent_params* p, ide3d_stream_t stream);
int ide3d_seg_xent_bwd(const ide3d_seg_xent_params* p, ide3d_stream_t stream);
/* The same pair with align_corners=True (source position d * (in - 1) / (out - 1)), same parameters and limits: the cross-entropy of
 * BiSeNet's upsampled logits (inversion/BiSeNet.py:249) for encoder fine-tuning. */
int ide3d_seg_xent_fwd_ac(const ide3d_seg_xent_params* p, ide3d_stream_t stream);
int ide3d_seg_xent_bwd_ac(const ide3d_seg_xent_params* p, ide3d_stream_t stream);

/* LPIPS v0.1 head of pivotal tuning (inversion/criteria/lpips/{lpips,utils}.py, the pip `lpips` package) over every tapped layer of
 * one call.  Per layer l, sample n and pixel p, with the norm over the channels:
 *   u = x / (||x||_2 + 1e-10),  v = y / (||y||_2 + 1e-10),  value[n] = sum_l mean_p sum_c lin_l[c] * (u_c - v_c)^2
 * x, y fp32 [n, c, h, w] with any element strides (NCHW and channels_last both coalesce on their fastest axis); y may have
 * y_stride[0] = 0 (one target for every sample).
 *   ide3d_lpips_fwd: value[n] (float) and, in scratch, the per-block partial sums and the per-(sample, layer) values (double, at
 *                    scratch + ide3d_lpips_scratch_bytes - 8 * n * num_layers, sample-major).  Two launches whatever num_layers:
 *                    one CTA per (layer, sample, 256 pixels) sums its pixels in double in a fixed order, one more launch folds the
 *                    partials per sample and layer in block order, then the layers in order.  No float atomics: deterministic.
 *   ide3d_lpips_bwd: one launch.  With g_c = grad_value[n] * (2 / (h w)) * lin[c] * (u_c - v_c) and s = 1 / (||x|| + 1e-10):
 *                      grad_x_k = s g_k - (s^2 / ||x||) x_k sum_c g_c x_c        (grad_y likewise with -g_c and y)
 *                    grad_x / grad_y use their own strides and may be NULL (not wanted); grad_y is per sample (gy_stride[0] != 0
 *                    when n > 1): a broadcast target's gradient is the caller's sum over n.
 *                    At a pixel whose vector is exactly zero the gradient written is 0.  torch's autograd gives NaN there (the
 *                    derivative of sqrt at 0); 0 keeps a ReLU trunk's gradient finite, as torch's threshold_backward makes it.
 * IDE3D_UNSUPPORTED for num_layers > IDE3D_LPIPS_MAX_LAYERS; IDE3D_INVALID for null pointers, empty sizes or offsets beyond 31 bits. */
#define IDE3D_LPIPS_MAX_LAYERS 8
typedef struct ide3d_lpips_layer {
    int c, h, w;
    const float* x;
    int64_t x_stride[4];        /* n, c, h, w */
    const float* y;
    int64_t y_stride[4];
    const float* lin;           /* [c] */
    float* grad_x;              /* bwd, optional */
    int64_t gx_stride[4];
    float* grad_y;              /* bwd, optional */
    int64_t gy_stride[4];
} ide3d_lpips_layer;
typedef struct ide3d_lpips_params {
    int n, num_layers;
    ide3d_lpips_layer layers[IDE3D_LPIPS_MAX_LAYERS];
    float* value;               /* fwd: [n] */
    void* scratch;              /* fwd: ide3d_lpips_scratch_bytes(p) bytes, 8-byte aligned */
    int64_t scratch_bytes;
    const float* grad_value;    /* bwd: [n] */
} ide3d_lpips_params;
/* bytes of scratch ide3d_lpips_fwd needs for this table (negative status for a table it would refuse) */
int64_t ide3d_lpips_scratch_bytes(const ide3d_lpips_params* p);
int ide3d_lpips_fwd(const ide3d_lpips_params* p, ide3d_stream_t stream);
int ide3d_lpips_bwd(const ide3d_lpips_params* p, ide3d_stream_t stream);

/* Multi-tap L1 head of the hybrid encoder's VGG loss (apps/train_hybrid_encoder.py:143-152) over every tapped layer of one call:
 *   total = sum_l weight_l * mean |x_l - y_l|      (the mean over all n * c * h * w elements of layer l)
 * x, y fp32 [n, c, h, w] with any non-negative element strides (one target per sample).  A layer whose x, y (and grad_x) share one
 * dense layout -- NCHW or channels_last -- is read as a flat array, with 16-byte accesses when aligned.
 *   ide3d_feat_l1_fwd: value[l] = the mean of layer l (float), value[num_layers] = total.  Two launches whatever num_layers: one
 *                      CTA per 4096 elements of a layer sums them into a double partial in a fixed order, one CTA folds the partials
 *                      of each layer in block order, then the layers in order.  No float atomics: deterministic.  scratch holds
 *                      the partials (ide3d_feat_l1_scratch_bytes bytes, 8-byte aligned).
 *   ide3d_feat_l1_bwd: one launch, grad_x_l = grad_value[0] * weight_l / numel_l * sgn(x_l - y_l), 0 where x == y (torch's sgn).
 *                      grad_value is read on the device.  grad_x uses its own strides.
 * IDE3D_UNSUPPORTED for num_layers > IDE3D_FEAT_L1_MAX_LAYERS or dtype != IDE3D_F32; IDE3D_INVALID for null pointers, empty sizes
 * or negative strides. */
#define IDE3D_FEAT_L1_MAX_LAYERS 8
typedef struct ide3d_feat_l1_layer {
    int c, h, w;
    float weight;
    const float* x;
    int64_t x_stride[4];        /* n, c, h, w */
    const float* y;
    int64_t y_stride[4];
    float* grad_x;              /* bwd */
    int64_t gx_stride[4];
} ide3d_feat_l1_layer;
typedef struct ide3d_feat_l1_params {
    int n, num_layers, dtype;
    ide3d_feat_l1_layer layers[IDE3D_FEAT_L1_MAX_LAYERS];
    float* value;               /* fwd: [num_layers + 1] */
    void* scratch;              /* fwd */
    int64_t scratch_bytes;
    const float* grad_value;    /* bwd: [1] */
} ide3d_feat_l1_params;
/* bytes of scratch ide3d_feat_l1_fwd needs for this table (negative status for a table it would refuse) */
int64_t ide3d_feat_l1_scratch_bytes(const ide3d_feat_l1_params* p);
int ide3d_feat_l1_fwd(const ide3d_feat_l1_params* p, ide3d_stream_t stream);
int ide3d_feat_l1_bwd(const ide3d_feat_l1_params* p, ide3d_stream_t stream);

/* Opening of the HybridEncoder's geometry branch (inversion/networks.py:1638-1646) from a class-id mask (extension).  The branch's
 * input one_hot(mask) * 2 - 1 takes `classes` + 1 distinct values per pixel (a mask value >= classes is the all-minus-one "no class"
 * row, as mask2label_np makes it), so the 1x1 stem, block 0's 3x3 conv1 (bias, lrelu slope 0.2, gain sqrt 2, no clamp) and its
 * [4, 4] FIR-down + 1x1 skip (no bias) become per-class tables:
 *   T[k]     = wg0 (2 W0[:, k] - sum_j W0[:, j]) + b0     (no class: -wg0 sum_j W0[:, j] + b0)
 *   y1[p]    = lrelu(b1 + sum_{taps t inside the image} wg1 W1[:, :, t] @ T[m(p + t)]) * sqrt 2
 *   skip[q]  = sum_{4x4 taps a inside the image} f~[a] wgs Ws @ T[m(2q + a - 1)]        f~: f flipped, as upfirdn2d convolves
 * The zero padding of conv1 and of the FIR pads the stem's OUTPUT: out-of-image taps contribute nothing.
 * Two launches whatever n: one CTA builds the tables in double (fixed order) into `tables` (ide3d_seg_stem_scratch_bytes bytes,
 * 16-byte aligned), then one CTA per 16 x 16 tile of y1 reads them from shared memory.  No atomics: reruns are bit-identical.
 * mask uint8 [n, h, w], any element strides; w0 [c0, classes], w1 [c0, c0, 3, 3], ws [c1, c0], b0 / b1 [c0], fir [4, 4]: dense fp32.
 * Outputs fp32 channels_last, dense: y1 [n, h, w, c0], skip [n, h / 2, w / 2, c1] (16-byte aligned, as are b1 and tables).
 * IDE3D_UNSUPPORTED unless c0 is 32 or 64, c1 = 2 c0, classes <= IDE3D_SEG_STEM_MAX_CLASSES, h and w even and >= 8. */
#define IDE3D_SEG_STEM_MAX_CLASSES 31
typedef struct ide3d_seg_stem_params {
    const uint8_t* mask;
    int n, h, w;
    int64_t mask_stride_n, mask_stride_h, mask_stride_w;
    int classes, c0, c1;
    const float* w0;
    const float* b0;
    float wg0;
    const float* w1;
    const float* b1;
    float wg1;
    const float* ws;
    float wgs;
    const float* fir;
    float* tables;
    float* y1;
    float* skip;
} ide3d_seg_stem_params;
/* bytes of `tables` ide3d_seg_stem needs (IDE3D_UNSUPPORTED for a configuration it would refuse) */
int64_t ide3d_seg_stem_scratch_bytes(int classes, int c0);
int ide3d_seg_stem(const ide3d_seg_stem_params* p, ide3d_stream_t stream);

/* Backward of ide3d_seg_stem: the gradients of w0, b0, w1, b1 and ws from grad_y1 [n, h, w, c0] and grad_skip [n, h / 2, w / 2, c1]
 * (fp32 channels_last, dense; grad_y1 16-byte aligned).  `fwd` is the forward's parameter block with its tables already built (the
 * lrelu's derivative is taken at the pre-activation recomputed from them).  Outputs dense fp32, overwritten: grad_w0 [c0, classes],
 * grad_b0 [c0], grad_w1 [c0, c0, 3, 3], grad_b1 [c0], grad_ws [c1, c0].
 *   launch 1: a fixed grid of CTAs sums the per-class gradients of the conv1 and skip tables over fixed sets of 16 x 16 tiles, each
 *             bin column owned by one thread walking its tile in order, into per-CTA slices of `scratch`;
 *   launch 2: the slices are folded in block order, in double;
 *   launch 3: one CTA runs the chain to the parameters in double in a fixed order (the mirror of the forward's table launch).
 * Three launches whatever n, no float atomics: reruns are bit-identical.  scratch: ide3d_seg_stem_bwd_scratch_bytes bytes, 16-byte
 * aligned.  Limits are the forward's (IDE3D_UNSUPPORTED otherwise); everything is validated before the device is touched. */
typedef struct ide3d_seg_stem_bwd_params {
    ide3d_seg_stem_params fwd;
    const float* grad_y1;
    const float* grad_skip;
    float* grad_w0;
    float* grad_b0;
    float* grad_w1;
    float* grad_b1;
    float* grad_ws;
    void* scratch;
    int64_t scratch_bytes;
} ide3d_seg_stem_bwd_params;
/* bytes of `scratch` ide3d_seg_stem_bwd needs (IDE3D_UNSUPPORTED for a shape the forward refuses, IDE3D_INVALID for bad sizes) */
int64_t ide3d_seg_stem_bwd_scratch_bytes(int n, int h, int w, int classes, int c0);
int ide3d_seg_stem_bwd(const ide3d_seg_stem_bwd_params* p, ide3d_stream_t stream);

/* Class ids of the generator's render at image resolution (extension): out[n, y, x] = argmax_k of the logits seg [n, classes, in_h,
 * in_w] (fp32, any strides; the strided view G.synthesis(..., return_seg='raw') returns) upsampled bilinearly (align_corners=False)
 * to out_h x out_w, with the rounding and tie rule of ide3d_video_frames / ide3d_image_strips.  out uint8 [n, out_h, out_w] dense.
 * One launch; the upsampled logits are never built. */
typedef struct ide3d_seg_labels_params {
    const float* seg;
    int n, classes, in_h, in_w;
    int64_t seg_stride_n, seg_stride_c, seg_stride_h, seg_stride_w;
    int out_h, out_w;
    uint8_t* out;
} ide3d_seg_labels_params;
int ide3d_seg_labels(const ide3d_seg_labels_params* p, ide3d_stream_t stream);
/* The same with align_corners=True (source position d * (in - 1) / (out - 1)): BiSeNet's upsampling (inversion/BiSeNet.py:249). */
int ide3d_seg_labels_ac(const ide3d_seg_labels_params* p, ide3d_stream_t stream);

/* k-nearest-neighbour distances of the precision / recall metric (metrics/precision_recall.py) over fp16 feature rows, D % 8 == 0,
 * dense, 16-byte aligned.  One tensor-core GEMM main loop per call: squared distances |x|^2 + |y|^2 - 2 x.y (fp32 accumulation, norms
 * in fp32 from the same fp16 values, negative values clamped to 0) are consumed in registers; the R x C matrix is never stored.
 *   ide3d_knn_kth_dist: out[r] (fp32) = the kth smallest |rows[r] - cols[c]| over all c, 1 <= kth <= IDE3D_KNN_MAX_KTH, kth <= C.
 *                       When rows is a slice of cols the row's own (zero) distance counts, as in the reference's
 *                       kthvalue(nhood_size + 1).  scratch: ide3d_knn_kth_dist_scratch_bytes(R, C, kth) bytes, 256-byte aligned.
 *   ide3d_knn_within:   flags[q] (uint8) = 1 if some j has |probes[q] - manifold[j]|^2 <= radius[j]^2 (radius fp32 [M]), else 0.
 *                       A CTA stops once every probe it owns has a hit.  scratch: ide3d_knn_within_scratch_bytes(Q, M) bytes,
 *                       256-byte aligned.
 * IDE3D_INVALID for null pointers, kth outside [1, IDE3D_KNN_MAX_KTH] or above C, D % 8 != 0, misaligned pointers or too little
 * scratch.  All but the last are decided from the arguments alone, before any CUDA call.  The kth_dist scratch size depends on the
 * current device's SM count, so ide3d_knn_kth_dist_scratch_bytes and the scratch check of ide3d_knn_kth_dist query the device
 * (cudaGetDevice, cudaDeviceGetAttribute); nothing is launched or read on the device before every check has passed. */
#define IDE3D_KNN_MAX_KTH 16
int64_t ide3d_knn_kth_dist_scratch_bytes(int64_t R, int64_t C, int kth);
int ide3d_knn_kth_dist(const void* rows, int64_t R, const void* cols, int64_t C, int D, int kth, float* out, void* scratch,
                       int64_t scratch_bytes, ide3d_stream_t stream);
int64_t ide3d_knn_within_scratch_bytes(int64_t Q, int64_t M);
int ide3d_knn_within(const void* probes, int64_t Q, const void* manifold, int64_t M, int D, const float* radius, uint8_t* flags,
                     void* scratch, int64_t scratch_bytes, ide3d_stream_t stream);

/* Average power spectrum of avg_spectra.py `calc` (float64 throughout).  images uint8 [n, c, size, size] through strides in ELEMENTS
 * (NCHW or NHWC); lut float64 [256] with lut[v] = (v - mean) / std (the caller's whitening, as the reference computes it); window
 * float64 [size], the Kaiser window scaled by rsqrt(sum w^2).  P = size * interp.  For every image in index order
 *     spectrum[k2, k1] += mean_c |sum_{n1, n2 < size} lut[x_c[n1, n2]] (window[n1] window[n2]) w_P^{n1 k1 + n2 k2}|^2
 * over the half plane k2 <= P / 2: spectrum is the float64 accumulator [P / 2 + 1, P], k2-major, zeroed by the caller before the first
 * call.  A pruned transform: rows, then columns, of the non-zero size x size block only; no P x P buffer.  Each bin has one owner
 * that adds the images in order: no float atomics, reruns are bit-identical and any split of a sequence into calls gives the same bits.
 * scratch: ide3d_spectrum_scratch_bytes(n, c, size, interp) bytes, 16-byte aligned.
 * IDE3D_UNSUPPORTED unless size is a power of two in [16, 1024], interp is 1, 2, 4 or 8, P <= 4096 and 1 <= c <= 4 (the caller falls
 * back to the reference's arithmetic); IDE3D_INVALID for null pointers or too little scratch.  Every check runs before any launch.
 * ide3d_spectrum_finalize: out float64 [P, P] = the accumulator / count in the reference's (unshifted) bin order, the half plane
 * k2 > P / 2 mirrored from out[k1, k2] = spectrum[P - k2, (P - k1) mod P]. */
int64_t ide3d_spectrum_scratch_bytes(int n, int c, int size, int interp);
int ide3d_spectrum_accum(const uint8_t* images, int n, int c, int size, int64_t stride_n, int64_t stride_c, int64_t stride_h,
                         int64_t stride_w, const double* lut, const double* window, int interp, double* spectrum, void* scratch,
                         int64_t scratch_bytes, ide3d_stream_t stream);
int ide3d_spectrum_finalize(const double* spectrum, int size, int interp, int64_t count, double* out, ide3d_stream_t stream);

/* avg_spectra.py `stats`: moments[0] += n * c * h * w, moments[1] += sum x, moments[2] += sum x^2 over uint8 images [n, c, h, w]
 * (strides in ELEMENTS).  Exact integers at any dataset size; integer atomics, so the result does not depend on the order. */
int ide3d_image_moments(const uint8_t* images, int n, int c, int h, int w, int64_t stride_n, int64_t stride_c, int64_t stride_h,
                        int64_t stride_w, uint64_t* moments, ide3d_stream_t stream);

/* Pillow's 8-bit two-pass resampler (libImaging/Resample.c, ImagingResample for L and RGB), table-driven and bit-identical.
 * in uint8 [n, in_h, in_w, c] and out uint8 [n, out_h, out_w, c] through strides in BYTES (n, h, w; channels contiguous), so a centre
 * crop is a pointer offset and a pitch and the output may be a window of a larger canvas.  c is 1 or 3.
 * Tables, in HOST memory (the library checks them and copies them into scratch; they may be freed on return), one per axis:
 *   bounds int32 [out, 2] = (first input index, tap count) and coeffs int32 [out, ksize], PIL's normalize_coeffs_8bpc weights
 *   (22 fractional bits).  Every tap range must lie inside the input and have at most ksize taps.
 * Passes as Pillow runs them: the horizontal pass (only if out_w != in_w) computes the rows bounds_y spans, first tap of the first
 * output row to last tap of the last, into a uint8 intermediate; the vertical pass (only if out_h != in_h) reads it, or the input
 * when the horizontal pass was skipped; with both skipped the call is a copy.  Each output value is
 *     clamp((2^21 + sum_i v_i k_i) >> 22, 0, 255)                      in int32, as Pillow computes it.
 * scratch: ide3d_resample_u8_scratch_bytes(n, c, in_h, out_h, out_w, ksize_x, ksize_y) bytes, 16-byte aligned.
 * IDE3D_INVALID for null pointers, c not 1 or 3, non-positive sizes or ksizes, tables that do not fit the sizes or too little scratch,
 * all decided before any CUDA call. */
int64_t ide3d_resample_u8_scratch_bytes(int n, int c, int in_h, int out_h, int out_w, int ksize_x, int ksize_y);
int ide3d_resample_u8(const uint8_t* in, int n, int c, int in_h, int in_w, int64_t in_stride_n, int64_t in_stride_h, int64_t in_stride_w,
                      uint8_t* out, int out_h, int out_w, int64_t out_stride_n, int64_t out_stride_h, int64_t out_stride_w, int ksize_x,
                      const int32_t* bounds_x, const int32_t* coeffs_x, int ksize_y, const int32_t* bounds_y, const int32_t* coeffs_y,
                      void* scratch, int64_t scratch_bytes, ide3d_stream_t stream);

/* The style-mixing grid of style_mixing.py:139-153 as uint8 HWC canvases: grid rows first_row .. first_row + rows - 1 of a grid of
 * cols + 1 columns, each grid row height pixels tall, every canvas (cols + 1) * width pixels wide.  Slot (g, j) holds cell
 * g * (cols + 1) + j - 1 (canvas order: the column seeds, then per row seed its un-mixed image followed by its mixed cells); slot (0, 0)
 * is black.  cells fp32 [ncells * views, 3, height, width], element strides, cell-major (row k * views + v is view v of the call's k-th
 * cell); the call reads the cells of its rows only, the first being that of slot (first_row, 0), or (0, 1) for first_row 0.
 * Each byte is (x * 127.5 + 128).clamp(0, 255).to(uint8) as torch computes it on the device (style_mixing.py:101).
 * out: byte (gi, v, y, x, c) of local grid row gi at out + gi * out_stride_row + v * out_stride_view + (y * (cols + 1) * width + x) * 3
 * + c.  One launch for every view.  IDE3D_INVALID for bad sizes, a canvas wider than 2^30 bytes or taller than 262140 pixels, or null
 * pointers, decided before any CUDA call; rows == 0 is a no-op. */
int ide3d_style_grid(const float* cells, int first_row, int rows, int cols, int views, int height, int width, int64_t stride_n,
                     int64_t stride_c, int64_t stride_h, int64_t stride_w, uint8_t* out, int64_t out_stride_row, int64_t out_stride_view,
                     ide3d_stream_t stream);

/* The display tail of viz/renderer.py:369-393 for one map x [c, h, w], float32 (dtype IDE3D_F32) or float16 (IDE3D_F16, widened
 * exactly as .to(torch.float32) does), element strides.  sel = channels [base_channel, base_channel + sel_channels).
 *   stats float32 [6] (or null) = mean, unbiased std and inf-norm of x, then of sel, from float64 sums of the raw values.
 *   out: byte (y, x, j) at out + y * out_stride_h + x * out_stride_w + j * out_stride_c for j < out_channels, from selected channel
 *   min(j, sel_channels - 1), in torch's float32 operations and order: with depth, v = ((v - min x) / fl(max x - min x) - 0.5) * -2
 *   (min and max over the whole map); with normalize, v / clip(max |v| over its channel, 1e-8, 1e8); v * gain; then
 *   (v * 127.5 + 128).clamp(0, 255) -> uint8.  The bytes equal torch's on the device.
 * Two launches, deterministic: a float64 reduction into one partial per CTA, then the elementwise pass, which folds the partials in a
 * fixed order.  scratch: ide3d_viz_image_scratch_bytes(c, h, w) bytes, 16-byte aligned.  IDE3D_INVALID for bad shapes, a window outside
 * [0, c), normalize with more than 1024 selected channels, null pointers or too little scratch, decided before any launch. */
int64_t ide3d_viz_image_scratch_bytes(int c, int h, int w);
int ide3d_viz_image(const void* x, int dtype, int c, int h, int w, int64_t stride_c, int64_t stride_h, int64_t stride_w, int base_channel,
                    int sel_channels, int depth, int normalize, float gain, uint8_t* out, int out_channels, int64_t out_stride_h,
                    int64_t out_stride_w, int64_t out_stride_c, float* stats, void* scratch, int64_t scratch_bytes, ide3d_stream_t stream);

/* The FFT panel of viz/renderer.py:396-406 for a map x [c, n, n] (float32 or float16, element strides), in float64:
 *     P[k1, k2] = sum_c |DFT2((x_c - mean x_c) * window[n1] window[n2])[k1, k2]|^2,
 * rolled by n / 2 in both axes, index = clamp(floor(((10 log10(P / mean P) / range_db + 1) / 2) * (lut_size - 1) + 0.5), 0, lut_size - 1),
 * and the panel pixel (y, x) gets lut[index] (uint8 [lut_size, 3]) at out + y * out_stride_h + x * out_stride_w + j * out_stride_c.  A
 * zero bin (-inf dB) and a constant map (mean P = 0) give index 0.  window: float64 [n], torch.kaiser_window(n, periodic=False, beta).
 * The FFT is fft.cuh's radix-2 transform, rows (half plane) then columns; the channel sum and the mean run in a fixed order, so reruns
 * are bit-identical.  scratch: ide3d_viz_fft_scratch_bytes(c, h, w) bytes, 256-byte aligned.  IDE3D_UNSUPPORTED unless h == w is a
 * power of two in [4, 1024] (the caller falls back to the reference's arithmetic); IDE3D_INVALID for c < 1, null pointers or too little
 * scratch.  Every check runs before any launch. */
int64_t ide3d_viz_fft_scratch_bytes(int c, int h, int w);
int ide3d_viz_fft(const void* x, int dtype, int c, int h, int w, int64_t stride_c, int64_t stride_h, int64_t stride_w, const double* window,
                  float range_db, const uint8_t* lut, int lut_size, uint8_t* out, int64_t out_stride_h, int64_t out_stride_w,
                  int64_t out_stride_c, void* scratch, int64_t scratch_bytes, ide3d_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* IDE3D_B200_H_ */
