/*
 * vqb200.h — C ABI of libvqb200.so, the H100 (sm_90a) native layer under the
 * vqgan-training hot path (Encoder -> reg -> Decoder fwd/bwd + LPIPS/VGG + PatchD + losses).
 *
 * The reference (cloneofsimo/vqgan-training) has NO native layer: its boundary is the Python
 * surface (ae.py / utils.py / vae_trainer.py) and every device op is a PyTorch library call.
 * Each entry point below therefore cites the reference *call site(s)* whose ATen/cuDNN library
 * call it replaces (file:line into the reference tree).
 *
 * Conventions
 *   - plain pointers + sizes only; no torch / C++ types. All pointers are DEVICE pointers unless
 *     the name ends in _host. `stream` is a cudaStream_t passed as void*.
 *   - activations are NHWC bf16 with C a multiple of 8 ("internal layout"); master weights,
 *     gradients and module-boundary tensors are fp32 NCHW / OIHW (the reference's layout).
 *   - every function returns 0 on success or a negative VQB_E* code; vqb_last_error() gives a
 *     message. There is no CPU fallback: on a machine without an sm_90 device the compute entry
 *     points fail with VQB_ENODEVICE.
 */
#ifndef VQB200_H_
#define VQB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VQB_OK 0
#define VQB_EINVAL (-1)    /* bad shape / alignment / flag combination */
#define VQB_ENODEVICE (-2) /* no sm_90 device or driver entry point missing */
#define VQB_ECUDA (-3)     /* a CUDA runtime / driver call failed */

#define VQB_MAX_VIEWS 16
#define VQB_MAX_TAPS 16

/* epilogue flags of vqb_conv_gemm */
#define VQB_EPI_BIAS 1   /* += bias[c]                                                    */
#define VQB_EPI_RES 2    /* += res[pixel][c]   (bf16, same addressing as out)             */
#define VQB_EPI_RELU 4   /* max(.,0)                                                      */
#define VQB_EPI_MASK 8   /* *= (mask[pixel][c] > 0)  (bf16, same addressing as out)       */
#define VQB_EPI_STATS 16 /* accumulate per-(n,channel) sum / sum-of-squares of the bf16-rounded
                            output into stats[n][Cout][2] (fp32 atomics) for GroupNorm      */

/* A strided 4-D view [Nv][Hv][Wv][C] (channel stride 1) of an NHWC bf16 tensor. */
typedef struct VqbView {
    int64_t offset;     /* element offset from the tensor base pointer */
    int32_t Wv, Hv, Nv; /* extents */
    int32_t _pad;
    int64_t sw, sh, sn; /* strides in elements */
} VqbView;

/* One filter tap: reads view `view` at (w + dw, h + dh); out-of-range reads are zero. */
typedef struct VqbTap {
    int32_t view, dw, dh, _pad;
} VqbTap;

/*
 * Implicit-GEMM convolution  out[n,h,w,co] = epi( sum_t sum_c A_view(t)[n, h+dh_t, w+dw_t, c] * Wp[co][t][c] ).
 * Covers: 3x3 s1 p1 and 1x1 convs, their dgrad (packed transposed/rotated weights), the
 * stride-2 (0,1,0,1)-padded Downsample conv (4 parity views), its transposed dgrad (per output
 * parity class), and the non-overlapping k4s4/k2s2 PatchDiscriminator heads (one view per tap).
 * Replaces: nn.Conv2d forward + autograd dgrad at ae.py:105-117,143-154,160-167,197-199,230-232,
 * 282-284,307-309; torchvision VGG convs reached from utils.py:95-111,150-154; heads utils.py:156-185.
 */
typedef struct VqbConvDesc {
    int32_t C;       /* channels of the A tensor = K per tap (multiple of 8)     */
    int32_t Cout;    /* GEMM N                                                   */
    int32_t N, H, W; /* output pixel grid, GEMM M = N*H*W                        */
    int32_t nviews, ntaps;
    int32_t flags;   /* VQB_EPI_*                                                */
    int32_t out_f32; /* 0: out is bf16, 1: out is fp32                           */
    int32_t _pad;
    int64_t on, oh, ow, oc; /* out element address = out + n*on + h*oh + w*ow + c*oc */
    VqbView views[VQB_MAX_VIEWS];
    VqbTap taps[VQB_MAX_TAPS];
} VqbConvDesc;

int vqb_conv_gemm(const VqbConvDesc* d, const void* a, const void* w_packed /* bf16 [Cout][ntaps*C] */,
                  const float* bias, const void* res, const void* mask, void* out, float* stats, void* stream);

/*
 * Weight gradient  dWp[co][t][c] = sum_{n,h,w} dy[n,h,w,co] * X_view(t)[n, h+dh_t, w+dw_t, c]
 * as a split-K wgmma GEMM with MN-major operands. `partial` is fp32 [ksplit][Cout][ntaps*C];
 * vqb_wgrad_reduce sums the splits and writes the OIHW fp32 gradient.
 * Replaces: the wgrad half of convolution_backward for every trainable conv (autograd of the
 * call sites listed at vqb_conv_gemm).
 */
typedef struct VqbWgradDesc {
    int32_t C;       /* channels of x                       */
    int32_t Cout;    /* channels of dy                      */
    int32_t N, H, W; /* dy pixel grid                       */
    int32_t nviews, ntaps;
    int32_t ksplit;
    int64_t ld_override; /* row pitch (floats) of partial; 0 = ntaps*roundup(C,64)                     */
    int64_t col_offset;  /* first column of partial this launch writes (several launches, one buffer) */
    VqbView dy_view;     /* normally the dense view of dy                                              */
    VqbView views[VQB_MAX_VIEWS];
    VqbTap taps[VQB_MAX_TAPS];
} VqbWgradDesc;

/* 1 if vqb_conv_gemm supports VQB_EPI_STATS for this descriptor (staged epilogue, whole sub-tiles inside one image) */
int vqb_conv_stats_ok(const VqbConvDesc* d);

int vqb_wgrad_gemm(const VqbWgradDesc* d, const void* dy, const void* x, float* partial, void* stream);

/* number of fp32 columns per Cout row of the wgrad partial buffer: ntaps * roundup(C, 64) */
int vqb_wgrad_cols(int ntaps, int C);

/*
 * grad[co][ci][tap] (OIHW fp32) (+)= sum_s partial[s][co][slot*C64 + ci], slot -> tap through tapmap_dev (int32[nslots],
 * device memory). Deterministic (no atomics). Replaces the tail of aten::convolution_backward (weight gradient layout).
 */
int vqb_wgrad_reduce(const float* partial, float* grad, int ksplit, int Cout, int CoutPad, int Cin, int T, int nslots,
                     int C64, const int* tapmap_dev, int accumulate, void* stream);

/*
 * OIHW fp32 master weights -> bf16 [R][nslots][Kpad] GEMM operand (R = Cin if transpose else Cout; transpose = dgrad
 * layout; tapmap_dev selects / reorders filter taps, e.g. the 180-degree rotation of the data gradient).
 * Replaces: the per-step fp32->bf16 weight casts of torch.autocast (vae_trainer.py:453,623) and cuDNN's internal
 * filter transforms.
 */
int vqb_pack_weights(const float* w_oihw, void* out, int Cout, int Cin, int T, int nslots, const int* tapmap_dev,
                     int transpose, int Kpad, void* stream);

/*
 * Module-boundary layout conversion. y[n,h,w,c] = (x[n,c,h,w] - shift[c]) * inv_scale[c] as bf16 NHWC with Cpad
 * channels (pad = 0); shift/inv_scale may be NULL. The scaled form is LPIPS/PatchD ScalingLayer (utils.py:70-71).
 * vqb_nhwc_to_nchw is the inverse / the backward of it (gx = g * inv_scale).
 */
/* folded variants (slot -> SET of taps as a bit mask): nearest-2x upsample fused into 4 phase convs with 2x2 taps */
int vqb_pack_weights_fold(const float* w_oihw, void* out, int Cout, int Cin, int T, int nslots, const int* tapmask_dev,
                          int transpose, int Kpad, void* stream);
int vqb_wgrad_reduce_fold(const float* partial, float* grad, int ksplit, int Cout, int CoutPad, int Cin, int T,
                          int nslots, int C64, const int* tapmask_dev, void* stream);

int vqb_nchw_to_nhwc(const float* x, void* y, int N, int C, int H, int W, int Cpad, const float* shift,
                     const float* inv_scale, void* stream);
int vqb_nhwc_to_nchw(const void* g, float* gx, int N, int C, int H, int W, int Cpad, const float* inv_scale,
                     void* stream);
/* variants that write / read the interior of a zero-framed [N][H+2p][W+2p][Cpad] buffer (first-layer "fat pixel" conv:
 * three horizontally adjacent 8-channel pixels are one 24-channel K run, 3 taps instead of 9) */
int vqb_nchw_to_nhwc_pad(const float* x, void* y, int N, int C, int H, int W, int Cpad, int pad, const float* shift,
                         const float* inv_scale, void* stream);
int vqb_nhwc_to_nchw_pad(const void* g, float* gx, int N, int C, int H, int W, int Cpad, int pad,
                         const float* inv_scale, void* stream);

/*
 * FP32GroupNorm (+ swish) forward / backward on bf16 NHWC: 32 groups, biased variance, eps inside the sqrt, fp32
 * statistics (ae.py:41-53 + ae.py:13-14). mr = [N][G][2] (mean, rstd) kept for the backward.
 * fwd workspace ws: N*C*2 doubles; bwd workspace ws: N*C*2 + N*G*2 floats. `add` (optional) is summed into dx.
 * `silu` is an activation code: 0 none, 1 swish, 2 LeakyReLU(0.2) (the 3-D PatchGAN of tae_disc.py; its backward
 * recomputes the pre-activation from x, gamma, beta and mr as the swish backward does); any other value is VQB_EINVAL.
 * vqb_gn_silu_apply takes codes 0 and 1 only (its caller is the ResnetBlock recompute).
 */
int vqb_gn_silu_fwd(const void* x, void* y, const float* gamma, const float* beta, float* mr, double* ws, int N,
                    int HW, int C, int G, float eps, int silu, void* stream);
/* forward when the producing conv already accumulated chsums[N][C][2] (VQB_EPI_STATS): finalise + apply only */
int vqb_gn_silu_fwd_pre(const void* x, void* y, const float* gamma, const float* beta, float* mr, const float* chsums,
                        int N, int HW, int C, int G, float eps, int silu, void* stream);
/* the apply pass alone, with the mr = [N][G][2] (mean, rstd) of an earlier vqb_gn_silu_fwd over the same x: same kernel
 * and grid, so y is bit-identical to that call's y. Recomputes a ResnetBlock's normalised activations in its backward
 * (tae.ResnetBlock, enable_training(..., recompute=True)). x, y 16-byte aligned; gamma, beta, mr 4-byte aligned. */
int vqb_gn_silu_apply(const void* x, void* y, const float* gamma, const float* beta, const float* mr, int N, int HW,
                      int C, int G, int silu, void* stream);
/* dx_colsum (optional [C] fp32): per-channel sums of dx = bias gradient of the conv that produced x, same pass */
int vqb_gn_silu_bwd(const void* x, const void* dy, const void* add, void* dx, const float* gamma, const float* beta,
                    const float* mr, float* dgamma, float* dbeta, float* ws, int N, int HW, int C, int G, int silu,
                    float* dx_colsum, void* stream);

/*
 * LeakyReLU(0.2) over n bf16 elements (an NTHWC activation; n a positive multiple of 8, pointers 16-byte aligned):
 * forward y = x > 0 ? x : 0.2 x (rounded once); backward dx = dy * (y > 0 ? 1 : 0.2), gated on the saved forward
 * output (y > 0 exactly where x > 0, so the gradient at 0 is torch's). Validates (VQB_EINVAL), then VQB_ENODEVICE
 * without an sm_90 device. The conv_in activation of tae_disc.PatchDiscriminator3D.
 */
int vqb_leaky_relu_fwd(const void* x, void* y, int64_t n, void* stream);
int vqb_leaky_relu_bwd(const void* y, const void* dy, void* dx, int64_t n, void* stream);

/*
 * Wavelet front-end of the encoder (--use_wavelet; utils.py:229-247): F.pad(x, 2) + grouped 6x6 stride-2 conv with the
 * four fixed analysis filters filt[4][6][6] (device, fp32), fused with the NCHW fp32 -> NHWC bf16 conversion:
 * y[n][ho][wo][c*4 + band], Cpad channels (pad = 0). Input-side op, no gradient (the input is data).
 */
int vqb_wavelet_fwd(const float* x, void* y, const float* filt, int N, int C, int H, int W, int Cpad, void* stream);

/*
 * bf16 inference path (README.hf.md "How to use": `VAE(...).cuda().bfloat16()`, `vae.encoder(img)`, `vae.decoder(z)`;
 * the bf16 modules' nn.Conv2d / F.group_norm / F.scaled_dot_product_attention calls at ae.py:47-53,76-93,105-117,
 * 143-154,160-167,197-199,230-232,282-284,307-309 then run on bf16 parameters and return bf16 tensors). Every entry
 * point below validates its arguments (VQB_EINVAL) and fails with VQB_ENODEVICE without an sm_90 device.
 *
 * Weight packing from bf16 OIHW masters: the layouts of vqb_pack_weights / vqb_pack_weights_fold. The plain re-layout
 * is exact (no rounding); folded taps are summed in fp32 and rounded once, like the fp32 path. vqb_pack_weights_multi
 * takes bf16 masters through VqbPackJob.w_bf16.
 */
int vqb_pack_weights_bf16(const void* w_oihw, void* out, int Cout, int Cin, int T, int nslots, const int* tapmap_dev,
                          int transpose, int Kpad, void* stream);
int vqb_pack_weights_fold_bf16(const void* w_oihw, void* out, int Cout, int Cin, int T, int nslots,
                               const int* tapmask_dev, int transpose, int Kpad, void* stream);
/* bf16 NCHW image / latent -> bf16 NHWC (plain, or into the interior of a pre-zeroed [N][H+2pad][W+2pad][Cpad] frame for
 * the fat-pixel first-layer conv), same (x - shift) * inv_scale option as vqb_nchw_to_nhwc; no fp32 copy of the input */
int vqb_nchw_to_nhwc_bf16(const void* x, void* y, int N, int C, int H, int W, int Cpad, const float* shift,
                          const float* inv_scale, void* stream);
int vqb_nchw_to_nhwc_pad_bf16(const void* x, void* y, int N, int C, int H, int W, int Cpad, int pad,
                              const float* shift, const float* inv_scale, void* stream);
/* bf16 NHWC -> bf16 NCHW module-boundary output (a submodule called directly on an NCHW tensor); an exact copy */
int vqb_nhwc_to_nchw_bf16(const void* y, void* x, int N, int C, int H, int W, int Cpad, void* stream);
/* wavelet front-end (utils.py:229-247) of a bf16 image; filter sums in fp32 */
int vqb_wavelet_fwd_bf16(const void* x, void* y, const float* filt, int N, int C, int H, int W, int Cpad,
                         void* stream);
/* The encoder z / decoder image of a bf16 module come straight out of conv_out's epilogue as bf16 NCHW through
 * vqb_conv_gemm with out_f32 = 0 and NCHW output strides (oc = H*W): no separate conversion. */

/*
 * Video autoencoder (tae.py, TVAE), no-grad inference in fp32 or bf16 modules. Activations are NTHWC bf16 with C a
 * multiple of 8; module-boundary tensors are NCTHW (the same memory as NCHW with H' = T*H, so the NCHW <-> NHWC
 * conversions and the GroupNorm kernels above serve it unchanged, as do 1x1x1 convs through vqb_conv_gemm on the
 * [N][T*H][W][C] view). Every entry point below validates its arguments (VQB_EINVAL) and fails with VQB_ENODEVICE
 * without an sm_90 device.
 */
#define VQB_MAX_VIEWS_3D 8
#define VQB_MAX_TAPS_3D 27

/* A strided 5-D view [Nv][Tv][Hv][Wv][C] (channel stride 1) of an NTHWC bf16 tensor. */
typedef struct VqbView3d {
    int64_t offset;         /* element offset from the tensor base pointer */
    int32_t Wv, Hv, Tv, Nv; /* extents */
    int64_t sw, sh, st, sn; /* strides in elements (multiples of 8) */
} VqbView3d;

/* One filter tap: reads view `view` at (w + dw, h + dh, t + dt); out-of-range reads are zero. */
typedef struct VqbTap3d {
    int32_t view, dw, dh, dt;
} VqbTap3d;

/*
 * 5-D implicit-GEMM convolution
 *   out[n,t,h,w,co] = epi( sum_tap sum_c A_view(tap)[n, t+dt, h+dh, w+dw, c] * Wp[co][tap][c] ),
 * epi = (+ bias[co] if VQB_EPI_BIAS) (+ res[voxel][co] if VQB_EPI_RES; bf16, same addressing as out). Other VQB_EPI_*
 * flags are refused (inference takes the separate, deterministic GroupNorm statistics pass). Output stores:
 *   out_f32 = 0, oc = 1: bf16 NTHWC with any voxel strides (on, ot, oh, ow multiples of 8; the folded up-sampling
 *                        writes phase sub-grids this way);
 *   otherwise          : strided fp32 (out_f32 = 1) or bf16 at out + n*on + t*ot + h*oh + w*ow + c*oc (NCTHW module
 *                        boundary).
 * Covers the 27-tap 3x3x3 stride-1 conv, the (0,1,0,1,0,1)-padded 3x3x3 stride-2 Downsample conv (8 parity views; the
 * pad is the TMA zero fill), and one phase of the nearest-x2 up-sampling folded into its 3x3x3 conv (8 taps of
 * pre-summed weights over the low-resolution input). Replaces nn.Conv3d at tae.py:66-78 (ResnetBlock conv1 / conv2),
 * :96-104 (Downsample), :110-116 (Upsample, with the F.interpolate), :136-138 and :165-167 (Encoder conv_in /
 * conv_out), :208-210 and :233 (Decoder conv_in / conv_out). The 1x1x1 convs (tae.py:22-23 qkv / proj_out,
 * :76-78 nin_shortcut) run through vqb_conv_gemm on the [N][T*H][W][C] view.
 */
typedef struct VqbConv3dDesc {
    int32_t C;          /* channels of the A tensor = K per tap (multiple of 8)     */
    int32_t Cout;       /* GEMM N                                                   */
    int32_t N, T, H, W; /* output voxel grid, GEMM M = N*T*H*W                      */
    int32_t nviews, ntaps;
    int32_t flags;   /* VQB_EPI_BIAS | VQB_EPI_RES                               */
    int32_t out_f32; /* 0: out is bf16, 1: out is fp32                           */
    int64_t on, ot, oh, ow, oc; /* out element address = out + n*on + t*ot + h*oh + w*ow + c*oc */
    VqbView3d views[VQB_MAX_VIEWS_3D];
    VqbTap3d taps[VQB_MAX_TAPS_3D];
} VqbConv3dDesc;

int vqb_conv3d_gemm(const VqbConv3dDesc* d, const void* a, const void* w_packed /* bf16 [Cout][ntaps*C] */,
                    const float* bias, const void* res, void* out, void* stream);

/*
 * Training of tae.TVAE (opt-in through tae.enable_training; fp32 master weights). The data gradients of the 3x3x3
 * stride-1 conv (27 rotated taps over dy, transposed weights) and of the stride-2 Downsample conv (one conv of 1 to 8
 * taps per parity class of dx, written through strided voxel addressing) run through vqb_conv3d_gemm. The data gradient
 * of the folded nearest-x2 up-sampling (tae.py:110-116) is inherently 4 (offset, folded weight) terms per axis: 64 taps
 * over the 8 parity views of dy, more than VqbConv3dDesc holds. VqbConv3dDgradDesc is VqbConv3dDesc with a 64-entry tap
 * table; vqb_conv3d_dgrad_gemm runs the same rank-5 kernel with no epilogue (flags must be 0) so the 64 taps accumulate
 * in one fp32 accumulator and are rounded once. Replaces the dgrad half of autograd's convolution_backward for
 * nn.Conv3d at tae.py:110-116 (Upsample).
 */
#define VQB_MAX_TAPS_3D_DGRAD 64
typedef struct VqbConv3dDgradDesc {
    int32_t C;          /* channels of dy = K per tap (multiple of 8)               */
    int32_t Cout;       /* channels of dx written                                    */
    int32_t N, T, H, W; /* dx voxel grid                                              */
    int32_t nviews, ntaps;
    int32_t flags;   /* must be 0                                                */
    int32_t out_f32; /* 0: dx is bf16, 1: dx is fp32                             */
    int64_t on, ot, oh, ow, oc;
    VqbView3d views[VQB_MAX_VIEWS_3D];
    VqbTap3d taps[VQB_MAX_TAPS_3D_DGRAD];
} VqbConv3dDgradDesc;

int vqb_conv3d_dgrad_gemm(const VqbConv3dDgradDesc* d, const void* dy, const void* w_packed /* bf16 [Cout][ntaps*C] */,
                          void* dx, void* stream);

/*
 * Rank-5 weight gradient  dWp[co][t*C64 + c] = sum_{n,t,h,w} dy[n,t,h,w,co] * X_view(tap)[n, t+dt, h+dh, w+dw, c]:
 * the split-K wgmma GEMM of vqb_wgrad_gemm with the K walk over 64-voxel boxes [bw][bh][bt][bn] (5-D TMA loads of dy and
 * of the tap-shifted x views). Up to 27 taps over up to 8 views (the Downsample's 8 parity views; its pad is the TMA zero
 * fill). ld_override / col_offset as in VqbWgradDesc, so the eight up-sampling phases fill one partial buffer. The fp32
 * partial [ksplit][Cout][ntaps*C64] is reduced to the OIDHW gradient by vqb_wgrad_reduce (T = 27) or
 * vqb_wgrad_reduce_fold (T = 27, 64 slots). Replaces the wgrad half of convolution_backward for nn.Conv3d at
 * tae.py:66-78, :96-104, :110-116, :136-138, :165-167, :208-210, :233.
 */
typedef struct VqbWgrad3dDesc {
    int32_t C;          /* channels of x                         */
    int32_t Cout;       /* channels of dy                        */
    int32_t N, T, H, W; /* dy voxel grid                         */
    int32_t nviews, ntaps;
    int32_t ksplit, _pad;
    int64_t ld_override; /* row pitch (floats) of partial; 0 = ntaps*roundup(C,64) */
    int64_t col_offset;  /* first column of partial this launch writes            */
    VqbView3d dy_view;   /* normally the dense view of dy                          */
    VqbView3d views[VQB_MAX_VIEWS_3D];
    VqbTap3d taps[VQB_MAX_TAPS_3D];
} VqbWgrad3dDesc;

int vqb_wgrad3d_gemm(const VqbWgrad3dDesc* d, const void* dy, const void* x, float* partial, void* stream);

/*
 * Attention core of tae.AttnBlock (tae.py:26-51: 8 heads of C/8 channels, F.scaled_dot_product_attention with its
 * default scale 1/sqrt(head_dim)): qkv [N][T][3C] bf16 (q | k | v channel blocks, head h owns channels
 * h*head_dim .. of each block) -> out [N][T][C] bf16; lse [N][C/head_dim][T] fp32. head_dim is a multiple of 8 from 8
 * to 112; any other value is refused with a message naming it. vqb_attn_fwd is this with head_dim = 64.
 */
int vqb_attn_fwd_hd(const void* qkv, void* out, float* lse, int N, int T, int C, int head_dim, void* stream);
/* Its backward (autograd of F.scaled_dot_product_attention at tae.py:31-50): dqkv [N][T][3C] bf16 from qkv, out, dout
 * and lse of the forward; dvec is a workspace of lse's shape. head_dim as in the forward; vqb_attn_bwd is this with
 * 64. */
int vqb_attn_bwd_hd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec, void* dqkv,
                    int N, int T, int C, int head_dim, void* stream);

/*
 * Reparameterisation of tae.DiagonalGaussian (tae.py:259-264): z [N][2Z][S] (NCTHW, S = T*H*W; mean = channels 0..Z-1,
 * logvar = Z..2Z-1) and eps [N][Z][S] -> out [N][Z][S] = mean + exp(0.5 * max(logvar, -3)) * eps, computed in fp32 and
 * rounded once. bf16 = 1: z, eps and out are bf16, else fp32. eps is drawn by the caller (torch.randn_like(mean), the
 * reference's own call, so a seeded run consumes the same CUDA RNG stream).
 */
int vqb_gauss_reparam(const void* z, const void* eps, void* out, int N, int Z, int64_t S, int bf16, void* stream);
/* Its backward (autograd of tae.py:263-264, fp32 training): g = dL/dout [N][Z][S], z, eps fp32 -> dz [N][2Z][S] fp32 with
 * dmean = g and dlogvar = g * eps * 0.5 * exp(0.5 * logvar) where logvar >= -3, else 0 (torch's clamp backward: the
 * gradient passes at exactly -3). */
int vqb_gauss_reparam_bwd(const float* g, const float* z, const float* eps, float* dz, int N, int Z, int64_t S,
                          void* stream);

/*
 * Clip boundary of the per-frame image losses (utils.LPIPS / utils.PatchDiscriminator called on a [B][C][T][H][W] clip,
 * tae_trainer.VideoTrainer): the frames of a clip, folded into the batch in (b, t) order, as per-frame NHWC bf16 images
 * [B*Tsel][H+2pad][W+2pad][Cpad], with the (x - shift) * inv_scale of vqb_nchw_to_nhwc fused in (the same fp32 arithmetic
 * and one rounding, so each image equals vqb_nchw_to_nhwc_pad of that frame bit for bit). The clip is read through its
 * strides (channel T*H*W, frame H*W): no folded copy. frames (device, int32 [B*Tsel], optional): image i is frame
 * frames[i] of clip i / Tsel; NULL means every frame (Tsel = T). The entries of one clip must be distinct and in [0, T):
 * the caller checks that on the host (ops.ClipToFrames). pad > 0 writes the interior of a PRE-ZEROED framed buffer.
 * x is fp32 or (_bf16) bf16; shift / inv_scale both NULL or both given. The non-_pad forms are pad = 0.
 * Every entry point validates its arguments (VQB_EINVAL) and fails with VQB_ENODEVICE without an sm_90 device.
 */
int vqb_ncthw_frames_to_nhwc_pad(const float* x, void* y, int B, int C, int T, int H, int W, int Cpad, int pad,
                                 const int* frames, int Tsel, const float* shift, const float* inv_scale, void* stream);
int vqb_ncthw_frames_to_nhwc_pad_bf16(const void* x, void* y, int B, int C, int T, int H, int W, int Cpad, int pad,
                                      const int* frames, int Tsel, const float* shift, const float* inv_scale,
                                      void* stream);
int vqb_ncthw_frames_to_nhwc(const float* x, void* y, int B, int C, int T, int H, int W, int Cpad, const int* frames,
                             int Tsel, const float* shift, const float* inv_scale, void* stream);
int vqb_ncthw_frames_to_nhwc_bf16(const void* x, void* y, int B, int C, int T, int H, int W, int Cpad,
                                  const int* frames, int Tsel, const float* shift, const float* inv_scale,
                                  void* stream);
/* The backward: gx [B][C][T][H][W] fp32 = g[image of (b, t)][h][w][c] * inv_scale[c] (inv_scale may be NULL), the
 * arithmetic of vqb_nhwc_to_nchw_pad; frames not in the selection get exact zeros from the same launch. Every element
 * of gx is written exactly once. */
int vqb_nhwc_pad_frames_to_ncthw(const void* g, float* gx, int B, int C, int T, int H, int W, int Cpad, int pad,
                                 const int* frames, int Tsel, const float* inv_scale, void* stream);
int vqb_nhwc_frames_to_ncthw(const void* g, float* gx, int B, int C, int T, int H, int W, int Cpad, const int* frames,
                             int Tsel, const float* inv_scale, void* stream);

/* out[c] = sum over P pixels of x[p][c] : Conv2d bias gradient */
int vqb_colsum(const void* x, float* out, int64_t P, int C, void* stream);

/*
 * 2x2/2 max-pool of the VGG16 trunk (torchvision features[4,9,16,23]) and its backward: first-maximum tie rule of
 * ATen; relu_mask additionally gates by x > 0 (x is a post-ReLU activation); `add` (optional) is summed into dx.
 */
int vqb_maxpool2_fwd(const void* x, void* y, int N, int Ho, int Wo, int C, void* stream);
int vqb_maxpool2_bwd(const void* x, const void* dy, const void* add, void* dx, int N, int Ho, int Wo, int C,
                     int relu_mask, void* stream);

/*
 * One LPIPS layer (utils.py:44-53,134-140): out[n] += mean_p sum_c w[c] (f0/(|f0|+1e-10) - f1/(|f1|+1e-10))^2,
 * and its backward w.r.t. f0 only (frozen trunk, target branch carries no gradient), gated by f0 > 0.
 */
int vqb_lpips_tail_fwd(const void* f0, const void* f1, const float* w, float* out, int N, int HW, int C, void* stream);
int vqb_lpips_tail_bwd(const void* f0, const void* f1, const float* w, const float* g, void* df0, int N, int HW, int C,
                       void* stream);
/*
 * Train-mode variants: the nn.Dropout(0.5) in front of every lin layer (utils.py:79-89) is live in the reference's
 * training loop (LPIPS is never put in eval mode, vae_trainer.py:477). Element (n, p, c) of the squared-difference tensor
 * is kept (and scaled by 2) iff bit ((n*HW + p)*C + c) of a counter-based hash stream of `seed` is set; forward and
 * backward regenerate the same bits, and vqb_lpips_dropout_mask writes them out ([N][HW][C] bytes, 1 = keep) so that a
 * test can feed the identical mask to the reference arithmetic.
 */
int vqb_lpips_tail_fwd_dropout(const void* f0, const void* f1, const float* w, float* out, int N, int HW, int C,
                               uint64_t seed, void* stream);
int vqb_lpips_tail_bwd_dropout(const void* f0, const void* f1, const float* w, const float* g, void* df0, int N, int HW,
                               int C, uint64_t seed, void* stream);
int vqb_lpips_dropout_mask(uint64_t seed, int N, int HW, int C, uint8_t* mask, void* stream);

/*
 * Multi-head self-attention core of AttnBlock (ae.py:74-93): qkv [N][T][3C] bf16 (q | k | v channel blocks, heads of 64
 * channels) -> out [N][T][C] = softmax(q k^T / 8) v, flash-style (no T x T matrix in HBM). lse [N][C/64][T] is saved for
 * the backward; dvec is a workspace of the same shape. Replaces F.scaled_dot_product_attention + einops rearranges.
 */
int vqb_attn_fwd(const void* qkv, void* out, float* lse, int N, int T, int C, void* stream);
int vqb_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec, void* dqkv, int N,
                 int T, int C, void* stream);

/*
 * VQ codebook nearest neighbour (BASELINE.json config 4; the reference has no VQ — semantics pinned by
 * oracle/vq_oracle.py): idx[i] = argmin_j sum_c (z[i][c]-e[j][c])^2 in canonical fp32 order (bit-exact vs the oracle,
 * first index on ties), zq = e[idx], *sqerr += sum (zq - z)^2 when sqerr != NULL. Non-finite distances follow
 * np.argmin: the first NaN distance wins, and a row whose distances are all +inf gets 0, so idx is always in [0, K).
 */
int vqb_vq_argmin(const float* z, const float* e, long long* idx, float* zq, float* sqerr, int M, int K, int D,
                  void* stream);

/*
 * Optimizer step over ONE flat fp32 buffer holding every tensor of a model (each tensor padded to a multiple of 1024
 * elements): torch.optim.AdamW semantics (decoupled weight decay, bias correction) with up to VQB_ADAMW_MAX_GROUPS
 * hyper-parameter groups. chunk_group[i] (device, uint8) = group of 1024-element chunk i, 255 = skip (the owning tensor
 * received no gradient). grads are multiplied by grad_scale first. groups_host is HOST memory (read during the call).
 * Replaces: optimizer_G.step()/optimizer_D.step() = AdamW(lr groups, wd 1e-3, betas (0.9, 0.95)) at
 * vae_trainer.py:455-475 with the cosine-with-warmup learning rate of :486-490 passed in as groups_host[].lr.
 */
#define VQB_ADAMW_MAX_GROUPS 4
typedef struct VqbAdamwGroup {
    float lr, beta1, beta2, eps, weight_decay;
    int32_t step; /* 1-based step count of this group (bias correction) */
} VqbAdamwGroup;
int vqb_adamw_flat(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const uint8_t* chunk_group,
                   int64_t nchunks, int ngroups, const VqbAdamwGroup* groups_host, float grad_scale, void* stream);
/* CUDA-graph friendly form: the per-group hyper-parameters (incl. bias corrections) are read from a 28-float DEVICE
 * record at kernel run time. vqb_adamw_fill_record (host function) builds that record from groups_host into host memory;
 * the caller copies it to record_dev on the launch stream before every launch / graph replay. */
int vqb_adamw_fill_record(int ngroups, const VqbAdamwGroup* groups_host, float* record_host);
int vqb_adamw_flat_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const uint8_t* chunk_group,
                       int64_t nchunks, const float* record_dev, float grad_scale, void* stream);
/* vqb_adamw_flat_dev plus an exponential moving average of the parameters in the same pass: after the AdamW update,
 * every element of the flat buffer (chunks of group 255 and zero pads included) gets ema -= r * (ema - params), with
 * r = 1 - d_n read as one fp32 from DEVICE memory (ema_rate_dev) at kernel run time, so graph replays follow the
 * schedule without re-capture. params, exp_avg and exp_avg_sq are bit-identical to vqb_adamw_flat_dev's. ema must be
 * 16-byte aligned like the other buffers. */
int vqb_adamw_ema_flat_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, float* ema,
                           const uint8_t* chunk_group, int64_t nchunks, const float* record_dev,
                           const float* ema_rate_dev, float grad_scale, void* stream);

/*
 * Re-pack every cached bf16 GEMM operand of the fp32 OIHW master weights in one launch (after an optimizer step).
 * jobs_dev: DEVICE array of njobs descriptors; total_blocks = sum over jobs of ceil(R/8)*ceil(Kpad/64)
 * (R = Cin if transpose else Cout; one block packs an 8-row x 64-k tile for every slot; T <= 16).
 *   out[r*ld_r + (slot/sg)*ld_g + (slot%sg)*Kpad + k] = bf16(transpose ? w[k][r][.] : w[r][k][.]); fold: tapmap entries are
 *   bit masks of taps summed in fp32 (vqb_pack_weights_fold), else tap indices (vqb_pack_weights).
 * Replaces: the per-step fp32->bf16 weight casts of torch.autocast (vae_trainer.py:453,623).
 */
typedef struct VqbPackJob {
    const void* w;       /* OIHW master: fp32, or bf16 when w_bf16 = 1 */
    void* out;
    const int* tapmap;
    int32_t Cout, Cin, T, nslots, transpose, Kpad, fold, sg, ld_g, ld_r;
    int32_t first_block; /* prefix sum of the tile-block counts of the preceding jobs */
    int32_t w_bf16;      /* 1: w is a bf16 master (inference-only module; exact re-layout, folds summed in fp32) */
} VqbPackJob;
int vqb_pack_weights_multi(const VqbPackJob* jobs_dev, int njobs, int total_blocks, void* stream);

/*
 * Reconstruction metrics (DESIGN.md section 7 row 25; the reference has none): per-item PSNR and SSIM of x against y,
 * both contiguous [B][C][T][H][W] (images: T = 1), fp32 (bf16 = 0) or bf16 (bf16 = 1). An item is (b, t); psnr and ssim
 * are fp32 [B * T] in (b, t) order. Every value v is mapped to u = fminf(fmaxf((v - lo) * inv, 0), 1) with inv =
 * 1 / (hi - lo) rounded once to fp32. PSNR = 10 log10(1 / mean (u_x - u_y)^2) over the item's C*H*W values (+inf when
 * the mean is 0). SSIM (Wang et al. 2004, no padding, no downsampling) is the mean over channels and the (H-10)(W-10)
 * valid positions of the 11x11 Gaussian window (sigma 1.5, normalised), C1 = 0.01^2, C2 = 0.03^2.
 * work: fp32 scratch of work_elems >= 2 * B * T * C * ceil((H-10)/32) * ceil((W-10)/32) floats. H, W >= 11, lo < hi
 * (finite). Two launches, no atomics: results are bit-reproducible.
 */
int vqb_psnr_ssim(const void* x, const void* y, int bf16, int B, int C, int T, int H, int W, float lo, float hi,
                  float* psnr, float* ssim, float* work, int64_t work_elems, void* stream);

/*
 * Tiled encode / decode blend (DESIGN.md section 3.11, definition in section 7 row 27; the reference has none):
 * accumulates one tile [N][C][Lt][Lh][Lw] (contiguous, fp32: tile_bf16 = 0, bf16: 1) into the fp32 grid acc
 * [N][C][T][H][W] at window (t0, h0, w0). wt, wh, ww: the tile's fp32 weight tables of Lt, Lh, Lw entries. Per element,
 * p = (wt[t] * wh[h]) * ww[w] rounded in that order; where every grid coordinate is >= its axis's prev_end (the end of
 * the previous tile on that axis, or the window start) acc = p * v, otherwise acc = fmaf(p, v, acc). Where every grid
 * coordinate is < its axis's next_start (the start of the next tile on that axis, or the extent) and out_bf16 is not
 * null, out_bf16 [N][C][T][H][W] = bf16_rn(acc). Launched per tile in raster order, this writes every element without a
 * memset or atomics, and rounds each bf16 output element once. Window inside the grid, t0 <= prev_end_t <= t0 + Lt,
 * t0 <= next_start_t <= T (likewise h, w), pointers aligned to their element size; otherwise VQB_EINVAL. One launch.
 */
int vqb_tile_blend(const void* tile, int tile_bf16, float* acc, void* out_bf16, int N, int C, int T, int H, int W,
                   int Lt, int Lh, int Lw, int t0, int h0, int w0, const float* wt, const float* wh, const float* ww,
                   int prev_end_t, int prev_end_h, int prev_end_w, int next_start_t, int next_start_h,
                   int next_start_w, void* stream);

/* library / device info */
const char* vqb_last_error(void);
int vqb_version(void);
int vqb_device_ok(void); /* 1 if the current device is sm_90 and the TMA driver entry point resolved */
int vqb_kernel_launch_count(void); /* number of kernels this library launched in this process */

#ifdef __cplusplus
}
#endif
#endif /* VQB200_H_ */
