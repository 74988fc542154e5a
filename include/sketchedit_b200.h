/*
 * sketchedit_b200 -- C ABI of the H100-native SketchEdit generator forward pass.
 *
 * The reference (zengxianyu/sketchedit) has no FFI / plugin layer: its boundary for this path is the
 * Python nn.Module surface. These entry points are what a binding for that surface calls; each one
 * names the reference interface it replaces. All pointers are plain device pointers (fp32, NCHW,
 * contiguous -- the layout of the torch tensors the reference passes) unless stated otherwise; no
 * torch types cross the boundary. Every function returns 0 on success; on failure it returns non-zero
 * and se_last_error() describes why. `stream` is a cudaStream_t (pass torch's current stream).
 *
 * Kernels are sm_90a only; there is no CPU fallback.
 */
#ifndef SKETCHEDIT_B200_H
#define SKETCHEDIT_B200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct se_model se_model;

/* arithmetic / storage mode of a forward call. Value 2 (bf16 activations on the CUDA-core kernels) is retired: every entry
 * point rejects it. */
enum {
  SE_PREC_BF16_TC = 0,     /* bf16 activations + weights, wgmma tensor-core kernels, fp32 accumulation */
  SE_PREC_FP32_EXACT = 1,  /* fp32 activations + weights, CUDA-core fp32 FMA kernels (fp32 parity config) */
  SE_PREC_FP32_TC = 3      /* fp32-parity arithmetic ON the tensor cores: activations and weights as fp16 hi + fp16 lo pairs (22
                              significant bits), three wgmma products per tap (hi*hi + hi*lo + lo*hi), fp32 accumulation and exact-math
                              epilogue. The fp32 parity config (1e-3) runs here; SE_PREC_FP32_EXACT stays as its cross-check.
                              Range: pairs store 64 v, saturated at +-65000, so inputs and activations with |v| > 65000 / 64
                              (about 1015.6) are silently clamped; below 2^-9 the lo half is an fp16 subnormal (absolute
                              quantum 2^-30). */
};

/* model options == the reference's command-line flags read on the hot path
 * (reference models/networks/editline_g.py:15-23,28-31 and options/base_options.py:19) */
enum {
  SE_OPT_USE_CAM = 0,        /* --use_cam          (default 1) */
  SE_OPT_POOL_AVG = 1,       /* --pool_type avg    (default 0 = max) */
  SE_OPT_NO_MASK_CC = 2,     /* --no_mask_cc       (default 0) */
  SE_OPT_NO_MASK_COARSE = 3, /* --no_mask_coarse   (default 0) */
  SE_OPT_JOINT_TRAIN_INP = 4 /* --joint_train_inp  (default 1, as in test_celeb.sh / test_places.sh) */
};

const char* se_last_error(void);
int se_abi_version(void);

/* ---- weights: replaces nn.Module parameter ownership + util.load_network
 *      (reference util/util.py:214-225; state_dict keys "<layer>.weight" [cout,cin,k,k], "<layer>.bias" [cout]) */
int se_model_create(se_model** out);
void se_model_destroy(se_model* m);
/* net: 'M' (MDGenerator, reference models/networks/editline2_g.py:14-43) or
 *      'G' (DeepFillC2Generator, reference models/networks/editline_g.py:44-100).
 * weight / bias: HOST fp32 pointers, OIHW. Shapes are validated against the architecture table. */
int se_model_set_layer(se_model* m, char net, const char* layer, const float* weight, const float* bias, int cout, int cin,
                       int ksize);
/* uploads and packs every layer; fails if a layer of either network is missing */
int se_model_finalize(se_model* m);
int se_model_set_option(se_model* m, int option, int value);

/* ---- whole path: replaces EditLine2Model.forward(data, mode='inference')
 *      (reference models/editline2_model.py:107-133 + generate_fake :338-370).
 * image [B,3,H,W] in [-1,1], sketch [B,1,H,W] in {0,1}; H, W multiples of 8 and H/4, W/4 >= 4.
 * Outputs: composed [B,3,H,W], mask [B,1,H,W] (soft). Optional (may be NULL): coarse, fine [B,3,H,W],
 * mask_image [B,3,H,W] (netM image head, only mode='visualize' uses it), mask_bin_out [B,1,H,W].
 * mask_bin_in (optional): use this binarised mask for netG instead of (mask > 0.5). */
int se_forward_inference(se_model* m, const float* image, const float* sketch, int B, int H, int W, int precision,
                         float* composed, float* mask, float* coarse, float* fine, float* mask_image,
                         const float* mask_bin_in, float* mask_bin_out, void* stream);

/* Same forward, outputs written as ONE packed tensor [B,4,H,W] (channels 0-2 composed, channel 3 the soft mask): the
 * layout of the data-parallel output all-gather (SURVEY.md 8e: `[B/n,4,H,W]` shards), so a rank's heads write straight
 * into its slice of the gather buffer and no pack/concat pass exists. */
int se_forward_inference_packed(se_model* m, const float* image, const float* sketch, int B, int H, int W, int precision,
                                float* packed, void* stream);

/* Same forward with the host-side codecs of the reference's test flow moved onto the device: inputs as the dataset reads them
 * before ToTensor/Normalize (reference data/testimage_dataset.py:89-103: image_u8 [B,H,W,3] RGB, sketch_u8 [B,H,W] already resized
 * to the image; on device: x/255 -> (x-0.5)/0.5, sketch > 0), outputs as test.py writes them (reference test.py:25-35:
 * ((x+1)/2*255) and (mask*255) truncated to uint8, HWC, RGB->BGR): bgr_u8 [B,H,W,3], mask_u8 [B,H,W]. 4x fewer bytes each way. */
int se_forward_inference_u8(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8, int B, int H, int W,
                            int precision, unsigned char* bgr_u8, unsigned char* mask_u8, void* stream);

/* ---- the same forward on a caller-supplied edit mask instead of netM's prediction (mask revising): generate_fake
 *      (editline2_model.py:338-370) with netM's soft mask replaced by edit_mask [B,1,H,W] (any fp32 values, used as given:
 *      not clamped, not checked):
 *        mask_inpaint = (edit_mask > 0.5)        strict >, like :347
 *        coarse, fine = netG(image, image, mask_inpaint, mask_inpaint, sketch)
 *        composed     = fine * edit_mask + image * (1 - edit_mask)        soft blend with the SUPPLIED mask, like :132
 *      netM's mask branch never runs; its trunk and image decoder run only when mask_image is requested (mode='visualize').
 *      Passing the soft mask se_forward_inference returned reproduces every output of that call bit for bit.
 *      Optional (may be NULL): coarse, fine, mask_image [B,3,H,W], mask_bin_out [B,1,H,W] (= mask_inpaint). NULL inputs or
 *      composed, and the retired precision 2, are errors. */
int se_forward_with_mask(se_model* m, const float* image, const float* sketch, const float* edit_mask, int B, int H, int W,
                         int precision, float* composed, float* coarse, float* fine, float* mask_image, float* mask_bin_out,
                         void* stream);
/* uint8 form, with se_forward_inference_u8's codecs: edit_mask_u8 [B,H,W] decodes to v/255 (ToTensor), so mask_inpaint is 1
 * exactly for v >= 128, and the blend uses v/255. The mask_u8 se_forward_inference_u8 writes ((int)(m * 255), truncating)
 * decodes back to the same byte, but it is not netM's exact mask: fed back, the blend moves by up to 1/255 and pixels with
 * 0.5 < m < 128/255 leave mask_inpaint. There is no mask output (the mask used is the caller's own bytes). NULL pointers and
 * the retired precision 2 are errors. */
int se_forward_with_mask_u8(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8,
                            const unsigned char* edit_mask_u8, int B, int H, int W, int precision, unsigned char* bgr_u8,
                            void* stream);

/* ---- previewing the edit mask (mask revising in two steps): netM's mask alone, then the forward on it.
 * se_predict_mask_u8: se_forward_inference_u8's input codec, then netM's trunk and mask branch only (no image decoder, no
 * netG): mask [B,1,H,W] receives netM's fp32 soft mask and mask_u8 [B,H,W] its bytes exactly as se_forward_inference_u8
 * writes them. Either output may be NULL, not both. The soft mask is bit for bit the one netM computes inside
 * se_forward_inference_u8 on the same bytes, in every precision and whatever the batch. */
int se_predict_mask_u8(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8, int B, int H, int W,
                       int precision, float* mask, unsigned char* mask_u8, void* stream);
/* se_forward_u8_with_soft_mask: se_forward_with_mask's forward on se_forward_inference_u8's codecs: uint8 image and sketch,
 * an fp32 edit_mask [B,1,H,W] used as given (netG inpaints edit_mask > 0.5, the result is blended with edit_mask), bgr_u8
 * [B,H,W,3]. netM does not run. Given the mask of se_predict_mask_u8, bgr_u8 is se_forward_inference_u8's bit for bit;
 * unlike the mask_u8 bytes, which se_forward_with_mask_u8 decodes to a mask up to 1/255 off. NULL pointers are errors. */
int se_forward_u8_with_soft_mask(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8,
                                 const float* edit_mask, int B, int H, int W, int precision, unsigned char* bgr_u8,
                                 void* stream);

/* se_forward_u8_export: one of the three uint8 region forwards above, with the attention exported for region-edit detail
 * (se_detail_u8). The mask argument chooses it: neither edit mask is se_forward_inference_u8 (mask_u8 [B,H,W] receives its
 * mask bytes, so it must not be NULL), edit_mask_u8 is se_forward_with_mask_u8 and the fp32 edit_mask [B,1,H,W] is
 * se_forward_u8_with_soft_mask; giving both is an error, and mask_u8 is ignored with either. bgr_u8 (and mask_u8) are that
 * call's bytes bit for bit, in every precision. Two more outputs:
 *   attn [B, L, L] fp32: the softmax weights of netG's contextual attention exactly as the forward used them (bf16: the
 *        stored bf16 probabilities; fp32 tensor-core mode: the fp32 weights before their split into fp16 halves), in
 *        se_contextual_attention_forward's layout [key][query], L = (H/8 - 1) (W/8 - 1); 4 L^2 bytes per image, computed in
 *        one band of query rows: the attention's L x L workspace (bf16: 2 L^2 bytes per image, fp32_direct: 8 L^2) is then
 *        not held to se_set_attention_workspace_limit, as for every call that returns the attention map.
 *   hole_u8 [B,H,W]: the mask netG inpaints (mask_inpaint) as 0 / 1 bytes.
 * A model without the attention (SE_OPT_USE_CAM = 0) has no weights to export: the call fails. */
int se_forward_u8_export(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8, const unsigned char* edit_mask_u8,
                         const float* edit_mask, int B, int H, int W, int precision, unsigned char* bgr_u8, unsigned char* mask_u8,
                         float* attn, unsigned char* hole_u8, void* stream);

/* ---- netM: replaces MDGenerator.forward(x, guide) -> (mask1, x_stage1)  (editline2_g.py:59-94) */
int se_netM_forward(se_model* m, const float* x, const float* guide, int B, int H, int W, int precision, float* mask1,
                    float* x_stage1 /* may be NULL */, void* stream);

/* ---- netG: replaces DeepFillC2Generator.forward(x, x2, mask, mask2, guide) -> (x_stage1, x_stage2)
 *      (editline_g.py:119-221). mask / mask2 [B,1,H,W]. guide may be NULL = the reference's guide=None (an all-ones
 *      sketch channel, editline_g.py:127-130). */
int se_netG_forward(se_model* m, const float* x, const float* x2, const float* mask, const float* mask2, const float* guide,
                    int B, int H, int W, int precision, float* x_stage1, float* x_stage2, void* stream);

/* ---- operators: replace gen_conv.forward / gen_deconv.forward (reference models/networks/utils.py:25-33, 48-51)
 * for the named layer of the named net. x [B,cin,H,W] -> y [B,cout_after_gate,Ho,Wo]. */
int se_gated_conv_forward(se_model* m, char net, const char* layer, const float* x, int B, int H, int W, int precision,
                          float* y, void* stream);

/* ---- replaces ReduceContextAttentionP1.forward + ReduceContextAttentionP2.forward as netG calls them
 *      (reference models/networks/splitcam.py:57-108,147-174; editline_g.py:203-207):
 * feat [B,C,h,w] (query = key = value source), mask_s [B,1,h,w] hole fraction; out [B,C,h,w].
 * attn (optional, may be NULL) receives the softmax weights [B, L, hs*ws] like cam_1's return value. */
int se_contextual_attention_forward(const float* feat, const float* mask_s, int B, int C, int h, int w, int precision,
                                    float* out, float* attn, void* stream);

/* ---- attention workspace: the contextual attention's probabilities (and, in the fp32 modes, its logits) are L x L per
 * image (L = patches of the 1/4-resolution map). They are computed in bands of query rows through one band-sized buffer:
 * the tallest band whose buffers fit `bytes` (process-wide; every forward and se_contextual_attention_forward). Results do
 * not depend on the band split. 0 restores the default of 16 GiB; a negative value is an error. A call whose smallest band
 * does not fit fails and names the bytes it needs. Calls that return the attention map (attn != NULL) use one band. */
int se_set_attention_workspace_limit(long long bytes);

/* ---- test.py:25-27 output conversion on device: uint8 HWC BGR image + uint8 mask (truncating) */
int se_outputs_to_uint8(const float* composed, const float* mask, int B, int H, int W, unsigned char* bgr_hwc,
                        unsigned char* mask_u8, void* stream);

/* ---- Pillow-exact resize of uint8 HWC images: PIL.Image.resize(size) with its default filter (BICUBIC, no box, no
 * reducing_gap), bit for bit, for a batch of n in [0, 32] windows of their own sizes (the resize-to-a-multiple-of-8 before the
 * forward and back after it of the reference demo, demo.py:39-73, and the crops of a region edit). Image i is src_hw[2i] rows
 * of src_hw[2i+1] pixels of `channels` bytes (1 or 3), its row r at src[i] + r * src_pitch[i] (bytes, >= src_hw[2i+1] *
 * channels); src is a host array of n device pointers. It is resized to dst_hw[2i] x dst_hw[2i+1] and written with packed rows
 * at dst + dst_off[i]. Sizes are in [1, 65535]; only the destination slices are written. With src[i] at the top-left pixel
 * of a box of an h x w x C image and src_pitch[i] = w * C, image i is Image.crop(box).resize(size). Windows may overlap each
 * other; dst must not overlap any window. swap_rb (channels 3) reverses the channel order of the output (BGR <-> RGB). An axis
 * whose length does not change is not resampled; an image of unchanged size is copied. scratch holds the intermediate of
 * images resized along both axes: src_hw[2i] x dst_hw[2i+1] x channels bytes each, rounded up to 256. Query form: scratch ==
 * NULL stores the bytes it needs in *scratch_bytes and enqueues nothing (src and dst may be NULL then); otherwise
 * *scratch_bytes is the size of scratch. The coefficient tables are built on the host and cached on the device per (in, out)
 * pair: the first call with a new length pair uploads its table (a synchronous copy); later calls only enqueue the kernels on
 * `stream`. */
int se_resize_window_u8(const unsigned char* const* src, const long long* src_pitch, const int* src_hw, unsigned char* dst,
                        const long long* dst_off, const int* dst_hw, int n, int channels, int swap_rb, void* scratch,
                        long long* scratch_bytes, void* stream);
/* Pillow's reducing resize of n in [0, 32] RGB windows, bit for bit (Pillow 12.2), the resize of Image.thumbnail(size):
 *     Image.crop(box).resize((w, h), Image.BICUBIC, reducing_gap=2.0)
 * The windows, their pitches, dst, dst_off and the sizes are those of se_resize_window_u8 with 3 channels and no swap;
 * the caller applies thumbnail's size rule. For a window of iw x ih resized to w x h, fx = int(iw / w / 2) or 1, fy
 * likewise. If either is > 1 the window is first reduced to ceil(iw / fx) x ceil(ih / fy) cells, each the average of the
 * pixels it covers (right and bottom cells may be partial), per channel ((s + n / 2) * m mod 2^32) >> 24 with s the cell's
 * byte sum, n its pixel count and m = uint32(float(2^32) / float(256 n)) (Image.reduce). The reduced image is then resampled
 * bicubically over the box (0, 0, iw / fx, ih / fy), box ends in C floats; an axis is resampled when its length changes or
 * its box end is not its length, vertically first when the reduced image is more than 100 times taller than wide and its
 * height shrinks, horizontally first otherwise. A window whose size does not change is copied. fx fy must stay below 2^24.
 * scratch holds per window its reduced image (when fx or fy > 1) and the intermediate of a resample along both axes, each
 * rounded up to 256 bytes; the query form (scratch == NULL) is se_resize_window_u8's. The coefficient tables share
 * se_resize_window_u8's cache and limit, keyed by (in, box end, out): the first call with a new key uploads its table (a
 * synchronous copy); otherwise the call only enqueues work on `stream`. */
int se_resize_reducing_u8(const unsigned char* const* src, const long long* src_pitch, const int* src_hw, unsigned char* dst,
                          const long long* dst_off, const int* dst_hw, int n, void* scratch, long long* scratch_bytes,
                          void* stream);
/* Resize back and paste n >= 0 boxes in order into canvases, bit for bit as sequential Pillow pastes (a region edit: the
 * forward's results on crops of the photo, pasted back into their boxes, which may overlap, nest or repeat):
 *     for i in 0 .. n-1:  res = Image.fromarray(rgb_i).resize((w, h));  m = Image.fromarray(mask_i).resize((w, h));
 *                         canvas_i.paste(res, (x, y), m)
 * Box i's result is the src_hw[2i] x src_hw[2i+1] x 3 bytes at rgb + rgb_off[i] and its mask the src_hw[2i] x src_hw[2i+1]
 * bytes at mask + mask_off[i]; both are resized to h x w = dst_hw[2i] x dst_hw[2i+1] (each rounded to uint8, as
 * se_resize_window_u8 writes them; sizes in [1, 65535]). Its canvas is the image whose row 0 starts at canvas + canvas_off[i],
 * canvas_pitch[i] bytes per row (>= 3 (x + w)), and (y, x) = (box_yx[2i], box_yx[2i+1]) is the box's top-left pixel in it.
 * Boxes with the same canvas_off share a canvas and must give the same pitch; different canvases must not overlap in memory,
 * and no canvas may overlap rgb or mask. The blend is Pillow's, per channel:
 *     canvas = DIV255(canvas * (255 - m) + res * m),   DIV255(a) = (((a + 128) >> 8) + a + 128) >> 8,
 * so a later box blends over what an earlier one wrote. Only the pixels of the boxes are read and written. swap_rb reverses
 * the result's channel order first (the forward writes BGR).
 * feather (may be NULL: no feathering) fades each box's paste mask to 0 along chosen sides (a region edit's box edges inside
 * the photo, so the paste shows no seam there). It holds 4n ints, box i's widths (left, top, right, bottom) in box pixels,
 * each in [0, the side's length: w for left and right, h for top and bottom]. Box i's resized mask m becomes, before the blend,
 *     m' = DIV255(m * r(y, x)),   r = min(ramp(x, left), ramp(w - 1 - x, right), ramp(y, top), ramp(h - 1 - y, bottom)),
 *     ramp(d, f) = d >= f ? 255 : (255 * (d + 1)) / (f + 1)   (integer division; d = 0 on the side's edge pixel),
 * with (y, x) the pixel's place in the box. A side of width 0 keeps m; DIV255(255 * m) == m, so widths of 0 give the bytes of
 * feather == NULL, and a box whose four widths are 0 runs its arithmetic unchanged.
 * detail (may be NULL, and detail_off with it: none) adds a detail plane per box (region-edit detail): it holds at byte
 * detail_off[i] (even; a negative offset: box i has none) box i's int16 plane [h][w][3] in RGB order, as se_detail_u8 writes
 * it. Box i's resized result, after the vertical pass's rounding and the channel swap, becomes clamp(res + D, 0, 255) before
 * the blend.
 * scratch holds the intermediates of boxes whose width changes: r256(src_hw[2i] * w * 3) + r256(src_hw[2i] * w) bytes for
 * box i, r256 rounding up to 256. The scratch query (scratch == NULL; rgb, mask and canvas may be NULL then) and the
 * coefficient-table cache are those of se_resize_window_u8. */
int se_resize_composite_feather_detail_u8(const unsigned char* rgb, const long long* rgb_off, const unsigned char* mask,
                                          const long long* mask_off, const int* src_hw, unsigned char* canvas, const long long* canvas_off,
                                          const long long* canvas_pitch, const int* box_yx, const int* dst_hw, const int* feather,
                                          const short* detail, const long long* detail_off, int n, int swap_rb, void* scratch,
                                          long long* scratch_bytes, void* stream);
/* Region-edit detail (contextual residual aggregation on netG's attention weights; DESIGN.md section 7b): for n >= 0 boxes of a
 * region edit at the working size Hn x Wn (multiples of 8, >= 16), box i of box_hw[2i] x box_hw[2i+1] = bh x bw pixels:
 *   photo[i], photo_pitch[i]  the photo's box, RGB bytes, row r at photo[i] + r * photo_pitch[i] (a host array of n device pointers)
 *   low + low_off[i]          resize(resize(box, (Wn, Hn)), (bw, bh)), [bh][bw][3] (se_resize_window_u8 both ways)
 *   hole + hole_off[i]        the forward's hole_u8 [Hn][Wn] for the box
 *   attn + attn_off[i]        the forward's attn [L][L] for the box (byte offset, a multiple of 4)
 * writes the int16 plane D [bh][bw][3] at byte D + d_off[i] (even), and where agg is not NULL the fp32 aggregate A [bh][bw][3]
 * at byte agg + agg_off[i] (0 outside the hole), with u(x) = ((2x + 1) Wn) / (2 bw), v(y) likewise, the patch grid ws x hs =
 * (Wn/8 - 1) x (Hn/8 - 1), patch (py, px) covering working pixels [8py, 8py + 16) x [8px, 8px + 16), ax(px) = min{x : u(x) >= 8px}:
 *   R(x, y) = hole(v(y), u(x)) ? 0 : photo - low
 *   A(x, y) = (1/nq) sum over the nq patches q covering (v(y), u(x)) of sum_k attn[k][q] R(min(ax(k) + x - ax(q), bw - 1), likewise y)
 *   D(x, y) = hole(v(y), u(x)) ? round half away from zero (A) : 0
 * Every patch position must have an anchor, u(bw - 1) >= Wn - 16 and v(bh - 1) >= Hn - 16 (true from bw >= Wn / 32 and
 * bh >= Hn / 32): a smaller box is an error. The GEMM runs over all L query rows (M = Mp), not only those that touch the hole.
 * A is an fp32 computation within 255 (L + 8) 2^-22 of its float64 value. Boxes run in order through one scratch of the
 * largest box's need (256 B aligned): 4 Mp^2 + 8 Mp Np bytes, Mp = L rounded up to 256, Np = 3 fw fh rounded up to 256,
 * fw = ceil(16 bw / Wn) + 2, fh likewise. Query form (scratch == NULL) as se_resize_window_u8's. Only enqueues work on `stream`. */
int se_detail_u8(const unsigned char* const* photo, const long long* photo_pitch, const int* box_hw, int n, int Hn, int Wn,
                 const unsigned char* low, const long long* low_off, const unsigned char* hole, const long long* hole_off, const float* attn,
                 const long long* attn_off, short* D, const long long* d_off, float* agg, const long long* agg_off, void* scratch,
                 long long* scratch_bytes, void* stream);
/* The feather of se_resize_composite_feather_detail_u8 on masks alone, in place: image i is the hw[2i] x hw[2i+1] 'L' bytes (rows
 * packed) at img + off[i], and each of its bytes m becomes DIV255(m * r(y, x)) with the ramp r of its widths feather[4i .. 4i+3]
 * (left, top, right, bottom; each in [0, the side's length]). Sizes are in [1, 65535]; an image with four widths of 0 is not
 * touched. For a predicted mask resized back to its box this gives the mask the feathered paste used. Only enqueues the
 * kernel on `stream`. */
int se_feather_u8(unsigned char* img, const long long* off, const int* hw, const int* feather, int n, void* stream);
/* Retired entries. Each is a call of the entries above. ABI version 2 retired three resize entries of version 1:
 *   se_resize_u8(src, src_off, src_hw, dst, dst_off, dst_hw, n, channels, ...)
 *       = se_resize_window_u8 with src[i] = src + src_off[i] and src_pitch[i] = src_hw[2i+1] * channels.
 *   se_resize_paste_u8(rgb, rgb_off, mask, mask_off, src_hw, base, base_off, dst, dst_off, dst_hw, n, ...)
 *       = se_resize_composite_feather_detail_u8 with one box per canvas: canvas_off[i] = base_off[i] of canvas = base,
 *         box_yx[i] = (0, 0), canvas_pitch[i] = 3 * dst_hw[2i+1], feather = detail = detail_off = NULL, pasting in place. For a
 *         separate dst, first copy each base image to its dst slice and composite into dst.
 *   se_resize_composite_u8(...) = se_resize_composite_feather_detail_u8(...) with feather = detail = detail_off = NULL.
 * ABI version 3 retired one more:
 *   se_resize_composite_feather_u8(rgb, rgb_off, mask, mask_off, src_hw, canvas, canvas_off, canvas_pitch, box_yx, dst_hw,
 *                                  feather, n, swap_rb, scratch, scratch_bytes, stream)
 *       = se_resize_composite_feather_detail_u8 with the same arguments and detail = detail_off = NULL before n. */
/* Baseline JPEG of n in [0, 32] RGB windows, byte for byte what Pillow writes for an RGB image without info:
 *     buf = io.BytesIO();  Image.fromarray(img_i).save(buf, "JPEG", quality=quality, subsampling=subsampling, optimize=optimize)
 * quality in [1, 100]; subsampling 0 (4:4:4) or 2 (4:2:0, Pillow's default with quality 75); optimize 0 (the Annex K Huffman
 * tables, Pillow's default) or 1 (Huffman tables built for each image from its symbol counts: a smaller file of the same
 * pixels). Image i is hw[2i] rows of hw[2i+1] RGB pixels (sizes in [1, 65535]), its row r at src[i] + r * src_pitch[i]
 * (bytes, >= 3 * hw[2i+1]); src is a host array of n device pointers, and windows may overlap each other. The file (SOI,
 * JFIF APP0, two DQT, SOF0, four DHT with the Annex K or the image's tables, SOS, the entropy-coded data, EOI) goes to
 * out + out_off[i], which must hold se_jpeg_max_bytes(h, w, subsampling) bytes with either value of optimize; only its first
 * out_bytes_dev[i] bytes are written, and that count is stored in the device array out_bytes_dev[i]. No out slice may
 * overlap another or a window. scratch == NULL stores the scratch bytes the call needs in *scratch_bytes (src, out and
 * out_bytes_dev may be NULL then); optimize = 1 needs about 12 KB more per image. Every argument is checked before anything
 * is enqueued on `stream`; the call only enqueues, and never waits on the device. */
int se_jpeg_encode_opt_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n, int quality,
                          int subsampling, int optimize, unsigned char* out, const long long* out_off, long long* out_bytes_dev,
                          void* scratch, long long* scratch_bytes, void* stream);
/* se_jpeg_encode_opt_u8 with optimize = 0: the file of
 *     buf = io.BytesIO();  Image.fromarray(img_i).save(buf, "JPEG", quality=quality, subsampling=subsampling) */
int se_jpeg_encode_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n, int quality, int subsampling,
                      unsigned char* out, const long long* out_off, long long* out_bytes_dev, void* scratch, long long* scratch_bytes,
                      void* stream);
/* Host only: a true upper bound of the file se_jpeg_encode_opt_u8 writes for an h x w image with either value of optimize:
 * the 623-byte header, 208 bytes per 8x8 block (64 codes of at most 26 bits) doubled for the 0x00 after each 0xFF, and EOI.
 * Optimal tables keep codes within 16 bits and list only used symbols, so their header is no longer than the Annex K one,
 * and a block's bits stay within 208 bytes (DESIGN.md, section 7b). -1 on bad arguments. */
long long se_jpeg_max_bytes(int h, int w, int subsampling);
/* Progressive JPEG of n in [0, 32] RGB windows, byte for byte what Pillow writes for an RGB image without info:
 *     buf = io.BytesIO();  Image.fromarray(img_i).save(buf, "JPEG", quality=quality, subsampling=subsampling, progressive=True)
 * with either value of Pillow's optimize (libjpeg-turbo builds optimal tables for every progressive file). The file is SOI,
 * JFIF APP0, two DQT, SOF2, then the ten scans of jpeg_simple_progression, each after the DHT segments of the tables built
 * from its own symbol counts and its SOS, then EOI. Arguments are those of se_jpeg_encode_opt_u8 without optimize, and are
 * checked the same way; out + out_off[i] must hold se_jpeg_progressive_max_bytes(h, w, subsampling) bytes. The scratch is
 * about 2.2 times that of se_jpeg_encode_opt_u8. The call only enqueues, and never waits on the device. */
int se_jpeg_encode_progressive_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n,
                                  int quality, int subsampling, unsigned char* out, const long long* out_off,
                                  long long* out_bytes_dev, void* scratch, long long* scratch_bytes, void* stream);
/* Host only: a true upper bound of the file se_jpeg_encode_progressive_u8 writes for an h x w image: the headers of the ten
 * scans with the largest alphabets, per block the most bits each scan can spend on it (DESIGN.md, section 7b) padded per
 * scan, doubled for the 0x00 after each 0xFF, and EOI. -1 on bad arguments. */
long long se_jpeg_progressive_max_bytes(int h, int w, int subsampling);
/* JPEG of n in [0, 32] RGB windows with the caller's quantisation tables, subsampling and APP1 / APP2 segments, byte for
 * byte what Pillow writes for an RGB image:
 *     buf = io.BytesIO();  Image.fromarray(img_i).save(buf, "JPEG", qtables=T, subsampling=subsampling, optimize=optimize,
 *                                                      progressive=progressive, exif=E, icc_profile=I)
 * and so also src.save(buf, "JPEG", quality="keep", ...) of a JPEG src with T = src.quantization and subsampling
 * JpegImagePlugin.get_sampling(src) (-1 there is 2 here). qtables holds ntables in [1, 4] tables of 64 entries in [0, 255],
 * natural order (as Image.quantization gives them); an entry 0 is taken as 1, as libjpeg does, and an entry above 255 (a
 * 16-bit table, an extended-sequential file) is refused. Pillow's component -> table assignment: one table serves all three
 * components and one DQT is written; with two, Y uses table 0 and Cb, Cr table 1; with three or four, component c uses
 * table c and a fourth table is never written. subsampling 0 (4:4:4), 1 (4:2:2: 16x8 MCUs, h2v1 chroma) or 2 (4:2:0).
 * segments holds segments_len in [0, 2^30] host bytes of back-to-back APP1 (FF E1) / APP2 (FF E2) segments, each with a
 * length that matches, written after APP0 as Pillow writes its EXIF block and then its ICC_PROFILE chunks (the Python
 * engine.jpeg_app_segments builds them). progressive = 1 writes se_jpeg_encode_progressive_u8's ten scans whatever optimize
 * is. The other arguments are those of se_jpeg_encode_opt_u8 and are checked the same way; out + out_off[i] must hold
 * se_jpeg_tables_max_bytes(h, w, subsampling, ntables, progressive, segments_len) bytes, and the scratch is that of the
 * quality entries at the same subsampling. The segments are copied into each file on `stream` (from pageable host memory,
 * so the copy is done with the host bytes when the call returns). The call only enqueues. */
int se_jpeg_encode_tables_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n,
                             const unsigned short* qtables, int ntables, int subsampling, int optimize, int progressive,
                             const unsigned char* segments, long long segments_len, unsigned char* out, const long long* out_off,
                             long long* out_bytes_dev, void* scratch, long long* scratch_bytes, void* stream);
/* Host only: a true upper bound of the file se_jpeg_encode_tables_u8 writes for an h x w image: that of
 * se_jpeg_max_bytes (progressive = 0) or se_jpeg_progressive_max_bytes (1) with the header's min(ntables, 3) DQT segments and
 * segments_len bytes of APP1 / APP2 segments, and 4:2:2's 4 blocks per 16x8 MCU. Entries >= 1 keep a block within the
 * quality-100 bound. -1 on bad arguments. */
long long se_jpeg_tables_max_bytes(int h, int w, int subsampling, int ntables, int progressive, long long segments_len);
/* PNG of n in [0, 32] windows, byte for byte what OpenCV writes with no parameters (OpenCV 4.13, libpng 1.6, zlib 1.3):
 *     cv2.imencode(".png", img_i)[1]
 * where img_i is the window as BGR (channels 3) or grey (channels 1). Image i is hw[2i] rows of hw[2i+1] pixels of `channels`
 * bytes (sizes in [1, 65535]), its row r at src[i] + r * src_pitch[i] (bytes, >= channels * hw[2i+1]); src is a host array of n
 * device pointers, and windows may overlap each other. swap_rb = 1 reads BGR pixels (the forward's output, what cv2.imwrite
 * is given), 0 reads RGB; it does not affect one channel. The file (signature, IHDR, the zlib stream in IDAT chunks of 8192
 * bytes, IEND) goes to out + out_off[i], which must hold se_png_max_bytes(h, w, channels) bytes; only its first
 * out_bytes_dev[i] bytes are written, and that count is stored in the device array out_bytes_dev[i]. No out slice may overlap
 * another or a window. scratch == NULL stores the scratch bytes the call needs in *scratch_bytes (src, out and out_bytes_dev
 * may be NULL then). Every argument is checked before anything is enqueued on `stream`; the call only enqueues. */
int se_png_encode_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n, int channels, int swap_rb,
                     unsigned char* out, const long long* out_off, long long* out_bytes_dev, void* scratch, long long* scratch_bytes,
                     void* stream);
/* Host only: a true upper bound of the file se_png_encode_u8 writes for an h x w image of `channels` (1 or 3) bytes per pixel:
 * the filtered data h (1 + w c) stored, 8 bytes per possible deflate block, the zlib header and Adler-32, 12 bytes per IDAT
 * chunk, the signature, IHDR and IEND. -1 on bad arguments. */
long long se_png_max_bytes(int h, int w, int channels);
/* Pixels of n in [0, 256] non-interlaced PNG files, pixel for pixel np.asarray(Image.open(f).convert(mode)) (Pillow 12) with
 * mode "RGB" (HWC, 3 bytes) or "L". The host parses each file's container and passes its IDAT payloads concatenated into one
 * zlib stream: file i's stream is the src_len[i] bytes at device address src + src_off[i]. info[6i..6i+5] are its height and
 * width (in [1, 65535]), bit depth, colour type (0 at depth 1/2/4/8, 2 at 8, 3 at 1/2/4/8, 4 at 8, 6 at 8), palette entries
 * (1 to 256 for colour type 3, else 0) and output bytes per pixel (3 "RGB", 1 "L"); a colour type 3 file's palette (RGB
 * triples) is at src + plte_off[i] (plte_off may be NULL when no file has one). Its pixels go to the device address out[i]
 * (h w mode bytes; out is a host array of n pointers, so one call fills several buffers), and its status to the device int
 * status_dev[i]: 0 when the pixels are Pillow's, nonzero for anything doubtful (a bad zlib header or FDICT, a bad block or
 * code, an over-subscribed table, a distance reaching before the start, too few or too many bytes, a wrong Adler-32, a
 * filter type past 4, a palette index past the palette), when the pixels are undefined and the file must go to Pillow. Bytes after the Adler-32 are ignored. Every read is checked against src_len[i] and every
 * write against the file's raw size. scratch holds each file's raw filtered scanlines, h (1 + ceil(w bits / 8)) bytes
 * rounded up to 16; scratch == NULL stores the bytes the call needs in *scratch_bytes (src, out and status_dev may be NULL
 * then). Every argument is checked before anything is enqueued on `stream`; the call only enqueues. */
int se_png_decode_u8(const unsigned char* src, const long long* src_off, const long long* src_len, const int* info,
                     const long long* plte_off, int n, unsigned char* const* out, int* status_dev,
                     void* scratch, long long* scratch_bytes, void* stream);
/* se_png_decode_u8 for large files: the same files, arguments, pixels and status rule, with each file's stream inflated by
 * many warps at once instead of one. The stream is cut every chunk_bytes (>= 1) compressed bytes; each cut starts at the
 * first dynamic-Huffman block header after it, and every chunk is decoded on its own. A file is decoded only if its chunks
 * join end to start into exactly the file's raw size; otherwise (as for a stream with a false block start) its status is
 * nonzero and it must go to Pillow. A stream with few dynamic blocks decodes correctly but with little parallelism. Each
 * file's raw size, h (1 + ceil(w bits / 8)), is at most 2^31 - 1. scratch holds per file the raw filtered scanlines and 4
 * bytes per raw byte of staging (about 32 + 128 MB for a 4000x2667 RGB file), plus 48 bytes per chunk (file i has
 * src_len[i] / chunk_bytes + 1 chunks); the query works as in se_png_decode_u8. */
int se_png_split_u8(const unsigned char* src, const long long* src_off, const long long* src_len, const int* info,
                    const long long* plte_off, int n, unsigned char* const* out, int* status_dev, long long chunk_bytes,
                    void* scratch, long long* scratch_bytes, void* stream);
/* Bytes of coefficient tables the resize entries keep per device (process-wide; 0 restores the default of 256 MiB; negative is an
 * error). When a call's new tables would pass the limit, the device's cache is emptied (after a device synchronise) before the
 * call looks up any table; one call's own tables may exceed it. */
int se_resize_set_table_cache_limit(long long bytes);
/* bytes of coefficient tables currently cached for the current device */
long long se_resize_table_cache_bytes(void);
/* Host only (no device needed): the coefficient table the resize entries use for one axis of length in -> out. Returns ksize;
 * bounds [out][2] = (first input sample, number of taps), coeffs [out][ksize] = weights with 22 fractional bits, zero beyond
 * the taps. cap = ints coeffs holds (>= out * ksize). bounds == coeffs == NULL: returns ksize only. Returns -1 on error. */
int se_resize_coeffs(int in, int out, int* bounds, int* coeffs, long long cap);

/* ---- introspection for bench.py */
/* number of kernels this library launched during the most recent forward-type call on this thread */
int se_last_launch_count(void);
/* bytes of device workspace currently held by the model's arena */
long long se_workspace_bytes(se_model* m);
/* when set (default 0), every kernel launch of the forward calls is bracketed by CUDA events on its stream and
 * accounted to a kernel class (kernel + layer shape) with its algorithmic FLOPs / bytes. se_timing_report writes a
 * JSON table of the classes seen since the last se_timing_enable(1) into buf (returns the length needed, -1 on error).
 * Throughput must be measured with timing OFF; bench.py runs one separate instrumented pass for its roofline table. */
int se_timing_enable(int on);
int se_timing_report(char* buf, int cap);

/* ---- activation taps (debugging and tests; off by default, no cost when off). While on, every forward of the model runs
 * eagerly (no CUDA graph is captured or replayed) and records one tap per stage input: a device copy of the raw bytes the
 * consumer reads, in memory the model owns outside the workspace arena. Tap points: the input of every gated conv / deconv /
 * stem pair ("in:<net>.<layer>", e.g. "in:G.conv11", "in:G.conv1+wconv1"), of every head ("in:G.conv17"), of the global
 * style pooling ("in:G.pool"), and the attention's feature map and pooled mask ("in:G.cam", "in:G.cam.mask_s"); in
 * SE_PREC_FP32_TC also the fp32 map the attention reads and the fp32 result it writes ("in:G.cam.f32", "out:G.cam.f32"),
 * either side of the split-half conversions. Taps are dropped at the next forward of the model, at se_taps_enable and at se_model_destroy. */
enum {
  SE_TAP_LAYOUT = 0,   /* 0 NHWC, 1 channel-blocked [B][ld][H][W][8], 2 space-to-depth channel-blocked [B][ld][H/2][W/2][8],
                          3 packed 8-channel stem rows [B][H][Wp][8] (image at x + padl) */
  SE_TAP_DTYPE = 1,    /* 0 fp32, 1 bf16, 2 split-half fp16 pairs (64 v = hi + lo; the lo blocks follow the hi blocks:
                          ld / 2 blocks further on, per parity group (CB blocks further on) in space-to-depth, one [H][Wp][8]
                          plane further on in packed rows) */
  SE_TAP_B = 2, SE_TAP_C = 3, SE_TAP_H = 4, SE_TAP_W = 5,   /* H, W: the full-resolution size also for space-to-depth */
  SE_TAP_LD = 6,       /* NHWC: pixel pitch in elements; channel-blocked: channel blocks per image (both halves) */
  SE_TAP_CB_OFF = 7,   /* first channel block of the view (channel-blocked, space-to-depth) */
  SE_TAP_WP = 8, SE_TAP_PADL = 9,   /* packed rows: row length in pixels, zero pixels left of the image */
  SE_TAP_DESC_LEN = 10
};
int se_taps_enable(se_model* m, int on);
/* taps recorded by the model's last forward (-1: no model) */
int se_taps_count(se_model* m);
/* tap i: its name (NUL-terminated, truncated to name_cap bytes), desc[SE_TAP_DESC_LEN] and size in bytes (each may be NULL) */
int se_tap_info(se_model* m, int i, char* name, int name_cap, int* desc, long long* bytes);
/* enqueues a copy of tap i's bytes to the device pointer dst on stream */
int se_tap_copy(se_model* m, int i, void* dst, void* stream);

/* ---- launch record of the channel-blocked wgmma convolution (tests; process-wide, off by default, one host branch per
 * launch when off). While it is on, every forward and operator call runs eagerly (no CUDA graph is captured or replayed), and
 * each conv_c8_kernel launch appends one record: the label of the layer that launched it ("<net>.<layer>", e.g. "G.conv11",
 * "G.conv1+wconv1") and rec[SE_C8_REC_LEN], the plan and tile geometry the launch ran (DESIGN.md 5.1). se_c8_log_enable
 * clears the record, whether it turns it on or off. */
enum {
  SE_C8_INST = 0,          /* index of the kernel instantiation (se_c8_inst_info) */
  SE_C8_TEAMS = 1,         /* consumer teams per CTA: 1 or 2 */
  SE_C8_CLUSTER = 2,       /* CTAs per cluster: 2 (streamed weights) or 1 */
  SE_C8_GRID = 3,          /* CTAs launched */
  SE_C8_TOTAL_TILES = 4,   /* N x TILES_X x TILES_Y tiles of 16 rows x 8 columns */
  SE_C8_N = 5, SE_C8_TILES_X = 6, SE_C8_TILES_Y = 7, SE_C8_HO = 8, SE_C8_WO = 9,   /* the position grid of the launch */
  SE_C8_STEP_X = 10, SE_C8_STEP_Y = 11, SE_C8_STEP_IMG = 12,      /* the grid in mixed radix (tiles_x, tiles_y, images) */
  SE_C8_CSTEP_X = 13, SE_C8_CSTEP_Y = 14, SE_C8_CSTEP_IMG = 15,   /* teams x the grid, the same way */
  SE_C8_MODE = 16,         /* 0: one halo per tile, 1: one box per tap */
  SE_C8_CPT = 17,          /* k-steps per tap (one box per tap: > 1 when a stage holds one 64-channel chunk) */
  SE_C8_NCLS = 18,         /* fused sub-pixel classes per tile (1: none) */
  SE_C8_A_BUFS = 19, SE_C8_NUM_STAGES = 20,   /* halo ring depth, weight / tap stage ring depth */
  SE_C8_OUT_C8 = 21,       /* output layout: 0 NHWC, 1 channel-blocked, 2 space-to-depth channel-blocked */
  SE_C8_CHOFF = 22, SE_C8_LDO = 23,   /* output channel offset and pitch (channels, or channel blocks x 8) */
  SE_C8_PHANTOM = 24,      /* 1: clustered with an odd tile count (the last pair's rank 1 computes nothing) */
  SE_C8_BLK_SPLIT = 25,    /* stem pair: output blocks sent to the first tensor (0: one output tensor) */
  SE_C8_REC_LEN = 26
};
int se_c8_log_enable(int on);
/* records appended since the last se_c8_log_enable */
int se_c8_log_count(void);
/* record i: its label (NUL-terminated, truncated to name_cap bytes) and rec[SE_C8_REC_LEN] (each may be NULL) */
int se_c8_log_get(int i, char* name, int name_cap, int* rec);
/* instantiations of conv_c8_kernel (host only) */
int se_c8_inst_count(void);
enum { SE_C8_INST_NT = 0, SE_C8_INST_F16 = 1, SE_C8_INST_R64 = 2, SE_C8_INST_M64 = 3, SE_C8_INST_R32 = 4, SE_C8_INST_TEAMS = 5,
       SE_C8_INST_LEN = 6 };
/* instantiation i: info[SE_C8_INST_LEN] = GEMM N, split-half operands (1) or bf16 (0), the k-step shape (R64 units of M64
 * MMAs, R32 units of 2), and TEAMS = 2 when it also has a two-team form (1 otherwise) */
int se_c8_inst_info(int i, int* info);

#ifdef __cplusplus
}
#endif
#endif
