"""Architecture tables for the SD-v1 hot path: parameter names/shapes with the reference's state-dict keys,
and a seeded synthetic initialiser (no checkpoint is available offline).

Key layout follows the reference modules: UNetModel (ldm/modules/diffusionmodules/openaimodel.py:443-708),
SpatialTransformer (ldm/modules/attention.py:218-248), AutoencoderKL Encoder/Decoder
(ldm/modules/diffusionmodules/model.py:368-533, ldm/models/autoencoder.py:285-305) and HF CLIPTextModel
(the cond stage, ldm/modules/encoders/modules.py:137-160).

The reference zero-initialises 39 weight tensors (zero_module), which makes a random-init UNet output exact
zeros; `random_state_dict` therefore draws EVERY tensor from a seeded generator so parity is non-trivial.
"""
from __future__ import annotations

from collections import OrderedDict

import torch

SD_V1_UNET = dict(image_size=32, in_channels=4, out_channels=4, model_channels=320, attention_resolutions=[4, 2, 1],
                  num_res_blocks=2, channel_mult=[1, 2, 4, 4], num_heads=8, use_spatial_transformer=True,
                  transformer_depth=1, context_dim=768, use_checkpoint=True, legacy=False)
SD_V1_VAE = dict(embed_dim=4, ddconfig=dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3,
                                             ch=128, ch_mult=[1, 2, 4, 4], num_res_blocks=2, attn_resolutions=[],
                                             dropout=0.0))
SD_V1_CLIP = dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                  num_attention_heads=12, max_position_embeddings=77, layer_norm_eps=1e-5)
# diffusers StableDiffusionSafetyChecker ("CompVis/stable-diffusion-safety-checker", scripts/txt2img.py:26-29): CLIP ViT-L/14
# vision tower + projection, 17 concept and 3 special-care embeddings
SD_V1_SAFETY = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16, image_size=224,
                    patch_size=14, projection_dim=768, layer_norm_eps=1e-5, n_concepts=17, n_special=3)
TINY_SAFETY = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, image_size=56,
                   patch_size=14, projection_dim=64, layer_norm_eps=1e-5, n_concepts=17, n_special=3)
CLIP_IMAGE_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_IMAGE_STD = (0.26862954, 0.26130258, 0.27577711)
# small configs with the same topology, for fast CPU/GPU tests (head dims stay in the kernels' supported set)
TINY_UNET = dict(image_size=16, in_channels=4, out_channels=4, model_channels=64, attention_resolutions=[2, 1],
                 num_res_blocks=1, channel_mult=[1, 2], num_heads=2, use_spatial_transformer=True,
                 transformer_depth=1, context_dim=64, use_checkpoint=False, legacy=False)
# unconditional attention-block family (openaimodel.py AttentionBlock + ResBlock with scale-shift norm / up-down):
# the LSUN-Churches LDM (models/ldm/lsun_churches256/config.yaml) and two small members for tests. The tiny ones keep
# every GroupNorm width a multiple of 32, every conv input width a multiple of 64, and head dims even, <= 128 and
# partly not multiples of 16 (8 and 24; 16 and 40).
LSUN_CHURCHES_UNET = dict(image_size=32, in_channels=4, out_channels=4, model_channels=192,
                          attention_resolutions=[1, 2, 4, 8], num_res_blocks=2, channel_mult=[1, 2, 2, 4, 4], num_heads=8,
                          use_scale_shift_norm=True, resblock_updown=True, use_spatial_transformer=False,
                          context_dim=None, legacy=True)
TINY_ATTN_UNET = dict(image_size=16, in_channels=4, out_channels=4, model_channels=64, attention_resolutions=[1, 2, 4],
                      num_res_blocks=1, channel_mult=[1, 3, 3], num_heads=8, use_scale_shift_norm=True,
                      resblock_updown=True, use_spatial_transformer=False, context_dim=None, legacy=True)
# both options off: additive-FiLM ResBlocks and conv Downsample / Upsample around AttentionBlocks
TINY_ATTN_PLAIN_UNET = dict(image_size=16, in_channels=4, out_channels=4, model_channels=64,
                            attention_resolutions=[2, 4], num_res_blocks=1, channel_mult=[1, 2, 5], num_heads=8,
                            use_scale_shift_norm=False, resblock_updown=False, use_spatial_transformer=False,
                            context_dim=None, legacy=True)
# the unconditional VQ-f4 LDMs (configs/latent-diffusion/celebahq-ldm-vq-4.yaml; ffhq- and lsun_bedrooms-ldm-vq-4 share
# the UNet and the first stage): plain ResBlocks, AttentionBlocks of num_head_channels 32 (14, 21, 28 heads of d = 32).
# Widths 224 .. 896 and the skip concats 672, 1120, 1568 are multiples of 32, not all of 64.
CELEBAHQ_UNET = dict(image_size=64, in_channels=3, out_channels=3, model_channels=224, attention_resolutions=[8, 4, 2],
                     num_res_blocks=2, channel_mult=[1, 2, 3, 4], num_head_channels=32)
# a small member for tests: widths 96 / 192 / 288, concats 288 and 480; 3 and 9 channels per GroupNorm group
TINY_VQ_UNET = dict(image_size=16, in_channels=3, out_channels=3, model_channels=96, attention_resolutions=[2, 4],
                    num_res_blocks=1, channel_mult=[1, 2, 3], num_head_channels=32)
# the class-conditional ImageNet LDM (configs/latent-diffusion/cin256-v2.yaml): the spatial-transformer UNet with
# num_heads 1 and legacy dim_head = ch, i.e. single-head attention at d = 384 / 576 / 960, cross-attention on the
# ClassEmbedder's one-token context; VQ-f4 first stage. Widths 192 .. 960 and every skip concat are multiples of 64.
CIN256_V2_UNET = dict(image_size=64, in_channels=3, out_channels=3, model_channels=192, attention_resolutions=[8, 4, 2],
                      num_res_blocks=2, channel_mult=[1, 2, 3, 5], num_heads=1, use_spatial_transformer=True,
                      transformer_depth=1, context_dim=512)
CIN256_V2_COND = dict(embed_dim=512, n_classes=1001, key="class_label")   # class 1000: the unconditional label
# a small member for tests: widths 64 / 384 / 960, single-head attention at d = 384 and 960
TINY_CIN_UNET = dict(image_size=16, in_channels=3, out_channels=3, model_channels=64, attention_resolutions=[2, 4],
                     num_res_blocks=1, channel_mult=[1, 6, 15], num_heads=1, use_spatial_transformer=True,
                     transformer_depth=1, context_dim=64)
TINY_CIN_COND = dict(embed_dim=64, n_classes=1001, key="class_label")
# the class-conditional ImageNet LDM-VQ-8 (models/ldm/cin256/config.yaml, configs/latent-diffusion/cin-ldm-vq-f8.yaml):
# spatial transformers with heads of num_head_channels 32 (8 / 16 / 32 heads at widths 256 / 512 / 1024) at every level
# of a 32x32x4 latent, cross-attention on a one-token ClassEmbedder context. n_classes stays at the reference default
# 1000, so this model has no unconditional label. The VQ-f8 first stage has AttnBlocks inside its 32x32 level (512 wide)
# as well as in the mid block.
CIN256_F8_UNET = dict(image_size=32, in_channels=4, out_channels=4, model_channels=256, attention_resolutions=[4, 2, 1],
                      num_res_blocks=2, channel_mult=[1, 2, 4], num_head_channels=32, use_spatial_transformer=True,
                      transformer_depth=1, context_dim=512)
CIN256_F8_COND = dict(embed_dim=512, n_classes=1000, key="class_label")
VQ_F8 = dict(embed_dim=4, n_embed=16384, ddconfig=dict(double_z=False, z_channels=4, resolution=256, in_channels=3, out_ch=3,
                                                        ch=128, ch_mult=[1, 2, 2, 4], num_res_blocks=2, attn_resolutions=[32],
                                                        dropout=0.0))
# small members for tests: 2 / 4 heads of d = 32 at two levels and in the middle block; a four-level (f8) first stage
# with level attention at 32x32 (128 wide: the per-image GEMM path) and at 8x8 (512 wide: the d = 512 flash kernel)
TINY_CIN_F8_UNET = dict(image_size=16, in_channels=4, out_channels=4, model_channels=64, attention_resolutions=[1, 2],
                        num_res_blocks=1, channel_mult=[1, 2], num_head_channels=32, use_spatial_transformer=True,
                        transformer_depth=1, context_dim=64)
TINY_CIN_F8_COND = dict(embed_dim=64, n_classes=1000, key="class_label")
TINY_VQ_F8 = dict(embed_dim=4, n_embed=512, ddconfig=dict(double_z=False, z_channels=4, resolution=64, in_channels=3,
                                                          out_ch=3, ch=64, ch_mult=[1, 2, 2, 8], num_res_blocks=1,
                                                          attn_resolutions=[32, 8], dropout=0.0))
# VQModelInterface first stages (models/first_stage_models/vq-f4/config.yaml) and a small member
VQ_F4 = dict(embed_dim=3, n_embed=8192, ddconfig=dict(double_z=False, z_channels=3, resolution=256, in_channels=3, out_ch=3,
                                                       ch=128, ch_mult=[1, 2, 4], num_res_blocks=2, attn_resolutions=[],
                                                       dropout=0.0))
TINY_VQ = dict(embed_dim=3, n_embed=512, ddconfig=dict(double_z=False, z_channels=3, resolution=32, in_channels=3, out_ch=3,
                                                        ch=64, ch_mult=[1, 2], num_res_blocks=1, attn_resolutions=[],
                                                        dropout=0.0))
# the LDM inpainting model (models/ldm/inpainting_big/config.yaml, scripts/inpaint.py): x_t (3 channels) concatenated
# with the VQ encoding of the masked image (3) and the resized mask (1); AttentionBlocks of 8 heads at d = 64 / 96 / 128,
# up / down ResBlocks without scale-shift norm. The first stage is VQ-f4 without mid-block attention.
INPAINTING_BIG_UNET = dict(image_size=64, in_channels=7, out_channels=3, model_channels=256,
                           attention_resolutions=[8, 4, 2], num_res_blocks=2, channel_mult=[1, 2, 3, 4], num_heads=8,
                           resblock_updown=True)
VQ_F4_NOATTN = dict(embed_dim=3, n_embed=8192, ddconfig={**VQ_F4["ddconfig"], "attn_type": "none"})
# small members for tests: heads of d = 16 and 24 at two attention levels; a VQ-f2 without mid-block attention
TINY_INPAINT_UNET = dict(image_size=16, in_channels=7, out_channels=3, model_channels=64, attention_resolutions=[2, 4],
                         num_res_blocks=1, channel_mult=[1, 2, 3], num_heads=8, resblock_updown=True)
TINY_VQ_NOATTN = dict(embed_dim=3, n_embed=512, ddconfig={**TINY_VQ["ddconfig"], "attn_type": "none"})
# the LDM super-resolution model (models/ldm/bsr_sr/config.yaml, notebook_helpers.py): x_t (3 channels) concatenated
# with the low-resolution image (3, the Identity cond stage's output at the latent size); plain ResBlocks, AttentionBlocks
# of num_head_channels 32 at ds 8 and in the middle block (20 heads at 640 channels; ds 16 is never reached). Widths
# 160 / 320 / 640 and skip concats 480 / 960 / 1280: 5, 15 and 30 channels per GroupNorm group. VQ-f4 first stage.
BSR_SR_UNET = dict(image_size=64, in_channels=6, out_channels=3, model_channels=160, attention_resolutions=[16, 8],
                   num_res_blocks=2, channel_mult=[1, 2, 2, 4], num_head_channels=32)
# small members for tests: width 160 (5 channels per group) with d = 32 heads at ds 2; a VQ-f4 (vqf 4) first stage
TINY_BSR_UNET = dict(image_size=16, in_channels=6, out_channels=3, model_channels=160, attention_resolutions=[2],
                     num_res_blocks=1, channel_mult=[1, 2], num_head_channels=32)
TINY_VQ_F4 = dict(embed_dim=3, n_embed=512, ddconfig={**TINY_VQ["ddconfig"], "ch_mult": [1, 1, 2]})
# the LDM semantic-synthesis models (models/ldm/semantic_synthesis256 and semantic_synthesis512: the same keys and
# shapes, image_size 64 / 128): x_t (3 channels) concatenated with the SpatialRescaler's 182 -> 3 channel map of the
# label map at the latent size. legacy defaults; attention_resolutions 32 / 16 / 8 are never reached (ds 1, 2, 4), so
# the only attention is the middle block's AttentionBlock of 8 heads at d = 128. Widths 128 / 512 / 1024, skip concats
# up to 2048: 4 .. 64 channels per GroupNorm group. VQ-f4 first stage.
SEMANTIC_SYNTHESIS_UNET = dict(image_size=64, in_channels=6, out_channels=3, model_channels=128,
                               attention_resolutions=[32, 16, 8], num_res_blocks=2, channel_mult=[1, 4, 8], num_heads=8)
SEMANTIC_SYNTHESIS_COND = dict(n_stages=2, in_channels=182, out_channels=3)
# small members for tests, same topology: widths 64 / 256 / 512, mid attention 8 x d 64; a 20-class rescaler
TINY_SEMANTIC_UNET = dict(image_size=16, in_channels=6, out_channels=3, model_channels=64,
                          attention_resolutions=[32, 16, 8], num_res_blocks=1, channel_mult=[1, 4, 8], num_heads=8)
TINY_SEMANTIC_COND = dict(n_stages=2, in_channels=20, out_channels=3)
TINY_VAE = dict(embed_dim=4, ddconfig=dict(double_z=True, z_channels=4, resolution=32, in_channels=3, out_ch=3,
                                           ch=64, ch_mult=[1, 2], num_res_blocks=1, attn_resolutions=[],
                                           dropout=0.0))
TINY_CLIP = dict(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=2,
                 num_attention_heads=2, max_position_embeddings=77, layer_norm_eps=1e-5)
# the LAION-400M text-to-image LDM (configs/latent-diffusion/txt2img-1p4B-eval.yaml): SD-v1's UNet with a 1280-wide
# context, cond stage BERTEmbedder(n_embed=1280, n_layer=32) (x_transformer Encoder: 8 heads of 64 whatever the width)
LAION_UNET = dict(SD_V1_UNET, context_dim=1280)
LAION_BERT = dict(n_embed=1280, n_layer=32, vocab_size=30522, max_seq_len=77)
# small members for tests: the attention's inner width stays 8 x 64 = 512
TINY_BERT = dict(n_embed=128, n_layer=2, vocab_size=1000, max_seq_len=77)
TINY_LAION_UNET = dict(TINY_UNET, context_dim=128)
# the text-conditional LDM-VQ-4 (models/ldm/text2img256/config.yaml): a 64x64x3 latent, spatial transformers with heads
# of num_head_channels 32 (12 / 18 / 30 heads at widths 384 / 576 / 960, 32² / 16² / 8² tokens) cross-attending to a
# 77-token BERTEmbedder(n_embed=640, n_layer=32) context; the VQ-f4 first stage (VQ_F4)
TEXT2IMG256_UNET = dict(image_size=64, in_channels=3, out_channels=3, model_channels=192, attention_resolutions=[8, 4, 2],
                        num_res_blocks=2, channel_mult=[1, 2, 3, 5], num_head_channels=32, use_spatial_transformer=True,
                        transformer_depth=1, context_dim=640)
TEXT2IMG256_BERT = dict(n_embed=640, n_layer=32, vocab_size=30522, max_seq_len=77)
# a small member for tests: 4 / 6 heads of d = 32 at two levels and in the middle block, on TINY_BERT's 128-wide
# context; first stage TINY_VQ_F4
TINY_TEXT2IMG256_UNET = dict(image_size=16, in_channels=3, out_channels=3, model_channels=64, attention_resolutions=[2, 4],
                             num_res_blocks=1, channel_mult=[1, 2, 3], num_head_channels=32, use_spatial_transformer=True,
                             transformer_depth=1, context_dim=128)
# the layout-to-image LDM (models/ldm/layout2img-openimages256/config.yaml): a 64x64x3 latent, spatial transformers of
# three BasicTransformerBlocks each, with heads of num_head_channels 32 (8 / 12 / 16 heads at widths 256 / 384 / 512,
# 32² / 16² / 8² tokens), cross-attending to a 92-token BERTEmbedder(n_embed=512, n_layer=16, vocab_size=8192) context
# fed token ids directly (cond_stage_key coordinates_bbox, use_tokenizer False); the VQ-f4 first stage (VQ_F4)
LAYOUT2IMG_UNET = dict(image_size=64, in_channels=3, out_channels=3, model_channels=128, attention_resolutions=[8, 4, 2],
                       num_res_blocks=2, channel_mult=[1, 2, 3, 4], num_head_channels=32, use_spatial_transformer=True,
                       transformer_depth=3, context_dim=512)
LAYOUT2IMG_BERT = dict(n_embed=512, n_layer=16, vocab_size=8192, max_seq_len=92)
# small members for tests: TINY_TEXT2IMG256_UNET with three blocks per spatial transformer, and a two-layer BERT with the
# model's 92 positions and 8192-id vocabulary; first stage TINY_VQ_F4
TINY_LAYOUT2IMG_UNET = dict(TINY_TEXT2IMG256_UNET, transformer_depth=3)
TINY_LAYOUT2IMG_BERT = dict(n_embed=128, n_layer=2, vocab_size=8192, max_seq_len=92)
# the retrieval-augmented diffusion model (configs/retrieval-augmented-diffusion/768x768.yaml, scripts/knn2img.py): a
# 48x48x16 latent, spatial transformers with heads of num_head_channels 32 (14 / 28 / 42 heads at widths 448 / 896 /
# 1344, 56 in the middle block) cross-attending to CLIP ViT-L/14's projected text embedding and its retrieved
# neighbours (768 wide, 1 + k tokens); a KL-f16 first stage (16 latent channels, five levels, AttnBlocks at 16x16).
RDM_UNET = dict(image_size=48, in_channels=16, out_channels=16, model_channels=448, attention_resolutions=[4, 2, 1],
                num_res_blocks=2, channel_mult=[1, 2, 3, 4], use_scale_shift_norm=False, resblock_updown=False,
                num_head_channels=32, use_spatial_transformer=True, transformer_depth=1, context_dim=768,
                use_checkpoint=True)
KL_F16 = dict(embed_dim=16, ddconfig=dict(double_z=True, z_channels=16, resolution=256, in_channels=3, out_ch=3, ch=128,
                                          ch_mult=[1, 1, 2, 2, 4], num_res_blocks=2, attn_resolutions=[16], dropout=0.0))
# FrozenCLIPTextEmbedder: the CLIP text tower with the text projection (transformers CLIPModel's text_projection)
CLIP_TEXT_PROJ = dict(SD_V1_CLIP, projection_dim=768)
# small members for tests: 2 / 4 heads of d = 32; a five-level (f16) KL first stage with level attention at 16x16 (128
# wide: the per-image path) and at 4x4 (512 wide: the d = 512 flash kernel); a 64-wide projected tiny CLIP
TINY_RDM_UNET = dict(image_size=16, in_channels=16, out_channels=16, model_channels=64, attention_resolutions=[1, 2],
                     num_res_blocks=1, channel_mult=[1, 2], num_head_channels=32, use_spatial_transformer=True,
                     transformer_depth=1, context_dim=64)
TINY_KL_F16 = dict(embed_dim=16, ddconfig=dict(double_z=True, z_channels=16, resolution=64, in_channels=3, out_ch=3,
                                               ch=64, ch_mult=[1, 1, 2, 2, 8], num_res_blocks=1,
                                               attn_resolutions=[16, 4], dropout=0.0))
TINY_CLIP_TEXT_PROJ = dict(TINY_CLIP, projection_dim=64)
# the standalone first stages of models/first_stage_models/*/config.yaml that no LDM uses: KL-f4 (3 latent channels),
# KL-f32 (64 latent channels, six levels, AttnBlocks at 16x16 and 8x8, 1x1 latent heads 128 -> 128 and 64 -> 64),
# VQ-f8-n256 (VQ-f8 with 256 codes) and VQ-f16 (16384 codes of width 8, five levels, AttnBlocks at 16x16)
KL_F4 = dict(embed_dim=3, ddconfig=dict(double_z=True, z_channels=3, resolution=256, in_channels=3, out_ch=3, ch=128,
                                        ch_mult=[1, 2, 4], num_res_blocks=2, attn_resolutions=[], dropout=0.0))
KL_F32 = dict(embed_dim=64, ddconfig=dict(double_z=True, z_channels=64, resolution=256, in_channels=3, out_ch=3, ch=128,
                                          ch_mult=[1, 1, 2, 2, 4, 4], num_res_blocks=2, attn_resolutions=[16, 8],
                                          dropout=0.0))
VQ_F8_N256 = dict(VQ_F8, n_embed=256)
VQ_F16 = dict(embed_dim=8, n_embed=16384, ddconfig=dict(double_z=False, z_channels=8, resolution=256, in_channels=3,
                                                         out_ch=3, ch=128, ch_mult=[1, 1, 2, 2, 4], num_res_blocks=2,
                                                         attn_resolutions=[16], dropout=0.0))
# small members for tests with the same level structure: KL-f32's six levels with level attention at 16x16 (128 wide)
# and 8x8 (256 wide) and the 128 -> 128 quant_conv; VQ-f16's five levels, attention at 16x16 and codes of width 8
FIRST_STAGES = {"kl-f4": KL_F4, "kl-f8": SD_V1_VAE, "kl-f16": KL_F16, "kl-f32": KL_F32, "vq-f4": VQ_F4,
                "vq-f4-noattn": VQ_F4_NOATTN, "vq-f8": VQ_F8, "vq-f8-n256": VQ_F8_N256, "vq-f16": VQ_F16}
TINY_KL_F4 = dict(embed_dim=3, ddconfig={**TINY_VQ_F4["ddconfig"], "double_z": True})
TINY_KL_F32 = dict(embed_dim=64, ddconfig=dict(double_z=True, z_channels=64, resolution=128, in_channels=3, out_ch=3,
                                               ch=64, ch_mult=[1, 1, 2, 2, 4, 4], num_res_blocks=1,
                                               attn_resolutions=[16, 8], dropout=0.0))
TINY_VQ_F16 = dict(embed_dim=8, n_embed=512, ddconfig=dict(double_z=False, z_channels=8, resolution=64, in_channels=3,
                                                            out_ch=3, ch=64, ch_mult=[1, 1, 2, 2, 4], num_res_blocks=1,
                                                            attn_resolutions=[16], dropout=0.0))
# FrozenClipImageEmbedder (the retriever that embeds RDM databases): the CLIP ViT-L/14 vision tower with the visual
# projection (transformers CLIPModel's visual_projection); the tiny member's 64-wide embeddings match TINY_RDM_UNET
CLIP_VISION_PROJ = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                        image_size=224, patch_size=14, projection_dim=768, layer_norm_eps=1e-5)
TINY_CLIP_VISION_PROJ = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2,
                             image_size=56, patch_size=14, projection_dim=64, layer_norm_eps=1e-5)


# ------------------------------------------------------------------------------------------------ UNet
def unet_plan(cfg):
    """Block list of UNetModel as (kind, prefix, params) tuples, in execution order.

    kinds: conv_in, res(cin, cout, ss, updown), st(ch, heads, dhead, depth), attn(ch, heads, dhead), down(ch), up(ch),
    out.
    Mirrors the constructor loops at openaimodel.py:512-686. Without a spatial transformer the attention layers are
    AttentionBlocks with `num_heads` heads of ch / num_heads channels (legacy=True passes num_head_channels=-1,
    openaimodel.py:547-549), or, when num_head_channels is set, ch / num_head_channels heads of num_head_channels
    (openaimodel.py:542-546); `ss` is use_scale_shift_norm; with resblock_updown the Downsample / Upsample layers are
    ResBlocks with updown "down" / "up" (openaimodel.py:567-582, 664-677).
    """
    mc = cfg["model_channels"]
    mult = cfg["channel_mult"]
    nrb = cfg["num_res_blocks"]
    nh = cfg.get("num_heads", -1)
    nhc = cfg.get("num_head_channels", -1)
    attn_res = set(cfg["attention_resolutions"])
    st = cfg.get("use_spatial_transformer", False)
    ss = bool(cfg.get("use_scale_shift_norm", False))
    updown = bool(cfg.get("resblock_updown", False))
    akind = "st" if st else "attn"
    depth = {"depth": cfg.get("transformer_depth", 1)} if st else {}     # BasicTransformerBlocks per SpatialTransformer

    def res(pre, cin, cout, ud=None, **kw):
        return ("res", pre, dict(cin=cin, cout=cout, ss=ss, updown=ud, **kw))

    def att(pre, ch):
        heads = nh if nhc == -1 else ch // nhc
        return (akind, pre, dict(ch=ch, heads=heads, dhead=ch // heads, **depth))

    plan = {"input": [], "middle": [], "output": []}
    plan["input"].append([("conv_in", "input_blocks.0.0", dict(cin=cfg["in_channels"], cout=mc))])
    chans = [mc]
    ch, ds, idx = mc, 1, 1
    for level, m in enumerate(mult):
        for _ in range(nrb):
            layers = [res(f"input_blocks.{idx}.0", ch, m * mc)]
            ch = m * mc
            if ds in attn_res:
                layers.append(att(f"input_blocks.{idx}.1", ch))
            plan["input"].append(layers)
            chans.append(ch)
            idx += 1
        if level != len(mult) - 1:
            plan["input"].append([res(f"input_blocks.{idx}.0", ch, ch, "down") if updown else
                                  ("down", f"input_blocks.{idx}.0", dict(ch=ch))])
            chans.append(ch)
            idx += 1
            ds *= 2
    plan["middle"] = [res("middle_block.0", ch, ch),
                      att("middle_block.1", ch),
                      res("middle_block.2", ch, ch)]
    idx = 0
    for level, m in list(enumerate(mult))[::-1]:
        for i in range(nrb + 1):
            ich = chans.pop()
            layers = [res(f"output_blocks.{idx}.0", ch + ich, mc * m, skip_ch=ich)]
            ch = mc * m
            sub = 1
            if ds in attn_res:
                layers.append(att(f"output_blocks.{idx}.{sub}", ch))
                sub += 1
            if level and i == nrb:
                layers.append(res(f"output_blocks.{idx}.{sub}", ch, ch, "up") if updown else
                              ("up", f"output_blocks.{idx}.{sub}", dict(ch=ch)))
                ds //= 2
            plan["output"].append(layers)
            idx += 1
    plan["out_ch"] = ch
    return plan


def _res_shapes(p, pre, cin, cout, temb, ss=False):
    p[f"{pre}.in_layers.0.weight"] = (cin,)
    p[f"{pre}.in_layers.0.bias"] = (cin,)
    p[f"{pre}.in_layers.2.weight"] = (cout, cin, 3, 3)
    p[f"{pre}.in_layers.2.bias"] = (cout,)
    ew = 2 * cout if ss else cout      # [scale | shift] with use_scale_shift_norm (openaimodel.py:218-224)
    p[f"{pre}.emb_layers.1.weight"] = (ew, temb)
    p[f"{pre}.emb_layers.1.bias"] = (ew,)
    p[f"{pre}.out_layers.0.weight"] = (cout,)
    p[f"{pre}.out_layers.0.bias"] = (cout,)
    p[f"{pre}.out_layers.3.weight"] = (cout, cout, 3, 3)
    p[f"{pre}.out_layers.3.bias"] = (cout,)
    if cin != cout:
        p[f"{pre}.skip_connection.weight"] = (cout, cin, 1, 1)
        p[f"{pre}.skip_connection.bias"] = (cout,)


def _st_shapes(p, pre, ch, ctx, depth=1):
    p[f"{pre}.norm.weight"] = (ch,)
    p[f"{pre}.norm.bias"] = (ch,)
    p[f"{pre}.proj_in.weight"] = (ch, ch, 1, 1)
    p[f"{pre}.proj_in.bias"] = (ch,)
    for i in range(depth):
        tb = f"{pre}.transformer_blocks.{i}"
        for a, kdim in (("attn1", ch), ("attn2", ctx)):
            p[f"{tb}.{a}.to_q.weight"] = (ch, ch)
            p[f"{tb}.{a}.to_k.weight"] = (ch, kdim)
            p[f"{tb}.{a}.to_v.weight"] = (ch, kdim)
            p[f"{tb}.{a}.to_out.0.weight"] = (ch, ch)
            p[f"{tb}.{a}.to_out.0.bias"] = (ch,)
        p[f"{tb}.ff.net.0.proj.weight"] = (8 * ch, ch)
        p[f"{tb}.ff.net.0.proj.bias"] = (8 * ch,)
        p[f"{tb}.ff.net.2.weight"] = (ch, 4 * ch)
        p[f"{tb}.ff.net.2.bias"] = (ch,)
        for n in ("norm1", "norm2", "norm3"):
            p[f"{tb}.{n}.weight"] = (ch,)
            p[f"{tb}.{n}.bias"] = (ch,)
    p[f"{pre}.proj_out.weight"] = (ch, ch, 1, 1)
    p[f"{pre}.proj_out.bias"] = (ch,)


def _attn_block_shapes(p, pre, ch):
    """AttentionBlock (openaimodel.py:278-324): GroupNorm32, qkv and proj_out are 1-d 1x1 convs."""
    p[f"{pre}.norm.weight"] = (ch,)
    p[f"{pre}.norm.bias"] = (ch,)
    p[f"{pre}.qkv.weight"] = (3 * ch, ch, 1)
    p[f"{pre}.qkv.bias"] = (3 * ch,)
    p[f"{pre}.proj_out.weight"] = (ch, ch, 1)
    p[f"{pre}.proj_out.bias"] = (ch,)


def unet_param_shapes(cfg):
    """OrderedDict key -> shape, keys exactly as UNetModel.state_dict() (686 tensors for SD v1)."""
    assert cfg.get("transformer_depth", 1) in (1, 3), "the published LDMs use transformer_depth 1 or 3"
    mc = cfg["model_channels"]
    temb = 4 * mc
    ctx = cfg.get("context_dim")
    p = OrderedDict()
    p["time_embed.0.weight"] = (temb, mc)
    p["time_embed.0.bias"] = (temb,)
    p["time_embed.2.weight"] = (temb, temb)
    p["time_embed.2.bias"] = (temb,)
    plan = unet_plan(cfg)

    def add(layers):
        for kind, pre, a in layers:
            if kind == "conv_in":
                p[f"{pre}.weight"] = (a["cout"], a["cin"], 3, 3)
                p[f"{pre}.bias"] = (a["cout"],)
            elif kind == "res":
                _res_shapes(p, pre, a["cin"], a["cout"], temb, a["ss"])
            elif kind == "st":
                _st_shapes(p, pre, a["ch"], ctx, a["depth"])
            elif kind == "attn":
                _attn_block_shapes(p, pre, a["ch"])
            elif kind == "down":
                p[f"{pre}.op.weight"] = (a["ch"], a["ch"], 3, 3)
                p[f"{pre}.op.bias"] = (a["ch"],)
            elif kind == "up":
                p[f"{pre}.conv.weight"] = (a["ch"], a["ch"], 3, 3)
                p[f"{pre}.conv.bias"] = (a["ch"],)

    for layers in plan["input"]:
        add(layers)
    add(plan["middle"])
    for layers in plan["output"]:
        add(layers)
    p["out.0.weight"] = (plan["out_ch"],)
    p["out.0.bias"] = (plan["out_ch"],)
    p["out.2.weight"] = (cfg["out_channels"], plan["out_ch"], 3, 3)
    p["out.2.bias"] = (cfg["out_channels"],)
    return p


# ------------------------------------------------------------------------------------------------ VAE
def _resnet_shapes(p, pre, cin, cout):
    p[f"{pre}.norm1.weight"] = (cin,)
    p[f"{pre}.norm1.bias"] = (cin,)
    p[f"{pre}.conv1.weight"] = (cout, cin, 3, 3)
    p[f"{pre}.conv1.bias"] = (cout,)
    p[f"{pre}.norm2.weight"] = (cout,)
    p[f"{pre}.norm2.bias"] = (cout,)
    p[f"{pre}.conv2.weight"] = (cout, cout, 3, 3)
    p[f"{pre}.conv2.bias"] = (cout,)
    if cin != cout:
        p[f"{pre}.nin_shortcut.weight"] = (cout, cin, 1, 1)
        p[f"{pre}.nin_shortcut.bias"] = (cout,)


def _attn_shapes(p, pre, c):
    p[f"{pre}.norm.weight"] = (c,)
    p[f"{pre}.norm.bias"] = (c,)
    for n in ("q", "k", "v", "proj_out"):
        p[f"{pre}.{n}.weight"] = (c, c, 1, 1)
        p[f"{pre}.{n}.bias"] = (c,)


def vae_param_shapes(cfg):
    """Keys as AutoencoderKL.state_dict() (encoder.*, decoder.*, quant_conv.*, post_quant_conv.*) — 248 tensors.
    ddconfig.attn_type "none" (make_attn, model.py:205-211: nn.Identity) drops the mid-block attention keys.
    A level whose resolution (ddconfig.resolution halved per level, independent of the input size) is in
    attn_resolutions has one AttnBlock per ResnetBlock (`encoder.down.{l}.attn.{b}`, `decoder.up.{l}.attn.{b}`)."""
    dd = cfg["ddconfig"]
    ch, mult, nrb = dd["ch"], dd["ch_mult"], dd["num_res_blocks"]
    zc = dd["z_channels"]
    attn_res = set(dd["attn_resolutions"])
    attn_type = dd.get("attn_type", "vanilla")
    if attn_type == "linear":
        raise NotImplementedError("ddconfig attn_type 'linear' (LinAttnBlock) is not supported")
    assert attn_type in ("vanilla", "none"), f"attn_type {attn_type} unknown"
    mid_attn = attn_type == "vanilla"
    if not mid_attn:        # every make_attn is nn.Identity: no level attention keys either
        attn_res = set()
    p = OrderedDict()
    # encoder (model.py:368-432)
    p["encoder.conv_in.weight"] = (ch, dd["in_channels"], 3, 3)
    p["encoder.conv_in.bias"] = (ch,)
    in_mult = [1] + list(mult)
    bi = ch
    res = dd["resolution"]
    for lvl in range(len(mult)):
        bi = ch * in_mult[lvl]
        bo = ch * mult[lvl]
        attn = OrderedDict()
        for b in range(nrb):
            _resnet_shapes(p, f"encoder.down.{lvl}.block.{b}", bi, bo)
            bi = bo
            if res in attn_res:
                _attn_shapes(attn, f"encoder.down.{lvl}.attn.{b}", bo)
        p.update(attn)                  # the level's `attn` ModuleList is registered after its `block` list
        if lvl != len(mult) - 1:
            p[f"encoder.down.{lvl}.downsample.conv.weight"] = (bi, bi, 3, 3)
            p[f"encoder.down.{lvl}.downsample.conv.bias"] = (bi,)
            res //= 2
    _resnet_shapes(p, "encoder.mid.block_1", bi, bi)
    if mid_attn:
        _attn_shapes(p, "encoder.mid.attn_1", bi)
    _resnet_shapes(p, "encoder.mid.block_2", bi, bi)
    p["encoder.norm_out.weight"] = (bi,)
    p["encoder.norm_out.bias"] = (bi,)
    zo = 2 * zc if dd["double_z"] else zc
    p["encoder.conv_out.weight"] = (zo, bi, 3, 3)
    p["encoder.conv_out.bias"] = (zo,)
    # decoder (model.py:462-533); note up.{lvl} modules are registered low-to-high
    bi = ch * mult[-1]
    p["decoder.conv_in.weight"] = (bi, zc, 3, 3)
    p["decoder.conv_in.bias"] = (bi,)
    _resnet_shapes(p, "decoder.mid.block_1", bi, bi)
    if mid_attn:
        _attn_shapes(p, "decoder.mid.attn_1", bi)
    _resnet_shapes(p, "decoder.mid.block_2", bi, bi)
    ups = OrderedDict()
    res = dd["resolution"] // 2 ** (len(mult) - 1)
    for lvl in reversed(range(len(mult))):
        q, attn = OrderedDict(), OrderedDict()
        bo = ch * mult[lvl]
        for b in range(nrb + 1):
            _resnet_shapes(q, f"decoder.up.{lvl}.block.{b}", bi, bo)
            bi = bo
            if res in attn_res:
                _attn_shapes(attn, f"decoder.up.{lvl}.attn.{b}", bo)
        q.update(attn)
        if lvl != 0:
            q[f"decoder.up.{lvl}.upsample.conv.weight"] = (bi, bi, 3, 3)
            q[f"decoder.up.{lvl}.upsample.conv.bias"] = (bi,)
            res *= 2
        ups[lvl] = q
    for lvl in range(len(mult)):
        p.update(ups[lvl])
    p["decoder.norm_out.weight"] = (bi,)
    p["decoder.norm_out.bias"] = (bi,)
    p["decoder.conv_out.weight"] = (dd["out_ch"], bi, 3, 3)
    p["decoder.conv_out.bias"] = (dd["out_ch"],)
    ed = cfg["embed_dim"]
    p["quant_conv.weight"] = (2 * ed, zo, 1, 1)
    p["quant_conv.bias"] = (2 * ed,)
    p["post_quant_conv.weight"] = (zc, ed, 1, 1)
    p["post_quant_conv.bias"] = (zc,)
    return p


def vq_param_shapes(cfg):
    """Keys as VQModelInterface.state_dict() (autoencoder.py:14-44, 264-282): encoder.* and decoder.* (double_z False),
    quantize.embedding.weight [n_embed, embed_dim], quant_conv (z -> embed) and post_quant_conv (embed -> z)."""
    dd = cfg["ddconfig"]
    assert not dd["double_z"], "VQ first stages have double_z False"
    kl = vae_param_shapes(dict(embed_dim=cfg["embed_dim"], ddconfig=dd))
    zc, ed = dd["z_channels"], cfg["embed_dim"]
    p = OrderedDict((k, v) for k, v in kl.items() if k.startswith(("encoder.", "decoder.")))
    p["quantize.embedding.weight"] = (cfg["n_embed"], ed)
    p["quant_conv.weight"] = (ed, zc, 1, 1)
    p["quant_conv.bias"] = (ed,)
    p["post_quant_conv.weight"] = (zc, ed, 1, 1)
    p["post_quant_conv.bias"] = (zc,)
    return p


def class_embedder_param_shapes(cfg):
    """Keys as ClassEmbedder.state_dict() (ldm/modules/encoders/modules.py:19-32), under `cond_stage_model.` in an
    LDM checkpoint."""
    return OrderedDict([("embedding.weight", (cfg["n_classes"], cfg["embed_dim"]))])


def spatial_rescaler_param_shapes(cfg):
    """Keys as SpatialRescaler.state_dict() (modules.py:106-134): the channel_mapper 1x1 conv when out_channels is set
    (bias only with bias=True); under `cond_stage_model.` in an LDM checkpoint."""
    p = OrderedDict()
    if cfg.get("out_channels") is not None:
        p["channel_mapper.weight"] = (cfg["out_channels"], cfg.get("in_channels", 3), 1, 1)
        if cfg.get("bias", False):
            p["channel_mapper.bias"] = (cfg["out_channels"],)
    return p


# ------------------------------------------------------------------------------------------------ CLIP
def clip_param_shapes(cfg):
    """Keys as transformers CLIPTextModel.state_dict() (`text_model.*`); in an SD checkpoint they sit under
    `cond_stage_model.transformer.` (modules.py:142)."""
    h, inter = cfg["hidden_size"], cfg["intermediate_size"]
    p = OrderedDict()
    p["text_model.embeddings.token_embedding.weight"] = (cfg["vocab_size"], h)
    p["text_model.embeddings.position_embedding.weight"] = (cfg["max_position_embeddings"], h)
    for i in range(cfg["num_hidden_layers"]):
        pre = f"text_model.encoder.layers.{i}"
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            p[f"{pre}.self_attn.{n}.weight"] = (h, h)
            p[f"{pre}.self_attn.{n}.bias"] = (h,)
        p[f"{pre}.layer_norm1.weight"] = (h,)
        p[f"{pre}.layer_norm1.bias"] = (h,)
        p[f"{pre}.mlp.fc1.weight"] = (inter, h)
        p[f"{pre}.mlp.fc1.bias"] = (inter,)
        p[f"{pre}.mlp.fc2.weight"] = (h, inter)
        p[f"{pre}.mlp.fc2.bias"] = (h,)
        p[f"{pre}.layer_norm2.weight"] = (h,)
        p[f"{pre}.layer_norm2.bias"] = (h,)
    p["text_model.final_layer_norm.weight"] = (h,)
    p["text_model.final_layer_norm.bias"] = (h,)
    return p


def clip_text_proj_param_shapes(cfg):
    """The text half of transformers CLIPModel.state_dict(): `text_model.*` and `text_projection.weight`
    [projection_dim, hidden] (no bias), for FrozenCLIPTextEmbedder."""
    p = clip_param_shapes(cfg)
    p["text_projection.weight"] = (cfg["projection_dim"], cfg["hidden_size"])
    return p


def clip_vision_proj_param_shapes(cfg):
    """The vision half of transformers CLIPModel.state_dict() (= CLIPVisionModelWithProjection's): `vision_model.*`
    and `visual_projection.weight` [projection_dim, hidden] (no bias), for FrozenClipImageEmbedder."""
    h, inter = cfg["hidden_size"], cfg["intermediate_size"]
    npos = (cfg["image_size"] // cfg["patch_size"]) ** 2 + 1
    p = OrderedDict()
    p["vision_model.embeddings.class_embedding"] = (h,)
    p["vision_model.embeddings.patch_embedding.weight"] = (h, 3, cfg["patch_size"], cfg["patch_size"])
    p["vision_model.embeddings.position_embedding.weight"] = (npos, h)
    p["vision_model.pre_layrnorm.weight"] = (h,)
    p["vision_model.pre_layrnorm.bias"] = (h,)
    for i in range(cfg["num_hidden_layers"]):
        pre = f"vision_model.encoder.layers.{i}"
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            p[f"{pre}.self_attn.{n}.weight"] = (h, h)
            p[f"{pre}.self_attn.{n}.bias"] = (h,)
        p[f"{pre}.layer_norm1.weight"] = (h,)
        p[f"{pre}.layer_norm1.bias"] = (h,)
        p[f"{pre}.mlp.fc1.weight"] = (inter, h)
        p[f"{pre}.mlp.fc1.bias"] = (inter,)
        p[f"{pre}.mlp.fc2.weight"] = (h, inter)
        p[f"{pre}.mlp.fc2.bias"] = (h,)
        p[f"{pre}.layer_norm2.weight"] = (h,)
        p[f"{pre}.layer_norm2.bias"] = (h,)
    p["vision_model.post_layernorm.weight"] = (h,)
    p["vision_model.post_layernorm.bias"] = (h,)
    p["visual_projection.weight"] = (cfg["projection_dim"], h)
    return p


def bert_param_shapes(cfg):
    """Keys as the reference BERTEmbedder.state_dict() (`transformer.*`, x_transformer.TransformerWrapper around an
    Encoder of `n_layer` ('a', 'f') pairs), to_logits included; under `cond_stage_model.` in an LDM checkpoint."""
    d, v, inner = cfg["n_embed"], cfg["vocab_size"], 8 * 64
    p = OrderedDict()
    p["transformer.token_emb.weight"] = (v, d)
    p["transformer.pos_emb.emb.weight"] = (cfg["max_seq_len"], d)
    for j in range(2 * cfg["n_layer"]):
        pre = f"transformer.attn_layers.layers.{j}"
        p[f"{pre}.0.weight"] = (d,)
        p[f"{pre}.0.bias"] = (d,)
        if j % 2 == 0:
            for n in ("to_q", "to_k", "to_v"):
                p[f"{pre}.1.{n}.weight"] = (inner, d)
            p[f"{pre}.1.to_out.weight"] = (d, inner)
            p[f"{pre}.1.to_out.bias"] = (d,)
        else:
            p[f"{pre}.1.net.0.0.weight"] = (4 * d, d)
            p[f"{pre}.1.net.0.0.bias"] = (4 * d,)
            p[f"{pre}.1.net.2.weight"] = (d, 4 * d)
            p[f"{pre}.1.net.2.bias"] = (d,)
    p["transformer.norm.weight"] = (d,)
    p["transformer.norm.bias"] = (d,)
    p["transformer.to_logits.weight"] = (v, d)
    p["transformer.to_logits.bias"] = (v,)
    return p


def safety_param_shapes(cfg):
    """Keys as diffusers StableDiffusionSafetyChecker.state_dict(): the CLIPVisionModel sits under `vision_model.`."""
    h, inter, pd = cfg["hidden_size"], cfg["intermediate_size"], cfg["projection_dim"]
    npos = (cfg["image_size"] // cfg["patch_size"]) ** 2 + 1
    v = "vision_model.vision_model"
    p = OrderedDict()
    p[f"{v}.embeddings.class_embedding"] = (h,)
    p[f"{v}.embeddings.patch_embedding.weight"] = (h, 3, cfg["patch_size"], cfg["patch_size"])
    p[f"{v}.embeddings.position_embedding.weight"] = (npos, h)
    p[f"{v}.pre_layrnorm.weight"] = (h,)
    p[f"{v}.pre_layrnorm.bias"] = (h,)
    for i in range(cfg["num_hidden_layers"]):
        pre = f"{v}.encoder.layers.{i}"
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            p[f"{pre}.self_attn.{n}.weight"] = (h, h)
            p[f"{pre}.self_attn.{n}.bias"] = (h,)
        p[f"{pre}.layer_norm1.weight"] = (h,)
        p[f"{pre}.layer_norm1.bias"] = (h,)
        p[f"{pre}.mlp.fc1.weight"] = (inter, h)
        p[f"{pre}.mlp.fc1.bias"] = (inter,)
        p[f"{pre}.mlp.fc2.weight"] = (h, inter)
        p[f"{pre}.mlp.fc2.bias"] = (h,)
        p[f"{pre}.layer_norm2.weight"] = (h,)
        p[f"{pre}.layer_norm2.bias"] = (h,)
    p[f"{v}.post_layernorm.weight"] = (h,)
    p[f"{v}.post_layernorm.bias"] = (h,)
    p["visual_projection.weight"] = (pd, h)
    p["concept_embeds"] = (cfg["n_concepts"], pd)
    p["special_care_embeds"] = (cfg["n_special"], pd)
    p["concept_embeds_weights"] = (cfg["n_concepts"],)
    p["special_care_embeds_weights"] = (cfg["n_special"],)
    return p


# ------------------------------------------------------------------------------------------------ init
def _is_norm_key(k):
    parts = k.split(".")
    if len(parts) < 2:
        return False
    leaf = parts[-2]
    if leaf.startswith("norm") or leaf.startswith("layer_norm") or leaf in ("final_layer_norm", "norm_out", "pre_layrnorm",
                                                                             "post_layernorm"):
        return True
    # BERTEmbedder LayerNorms: transformer.attn_layers.layers.{j}.0
    if len(parts) == 6 and parts[:3] == ["transformer", "attn_layers", "layers"] and parts[4] == "0":
        return True
    # UNet GroupNorms live at in_layers.0 / out_layers.0 / out.0
    return (len(parts) >= 3 and parts[-3] in ("in_layers", "out_layers") and leaf == "0") or k.startswith("out.0.")


def random_state_dict(shapes, seed, prefix="", device="cpu"):
    """Seeded synthetic weights (fp32), independent of module construction order. device="cpu" gives the values the
    golden fixtures were made with; a CUDA device draws from the device generator (fast; used by the benchmark).

    weights ~ N(0, 1/fan_in); norm gains 1 + 0.1 N(0,1); biases and norm shifts 0.1 N(0,1) (embeddings N(0, 0.02^2)
    as CLIP). Each tensor gets its own generator seeded from (seed, index) so a subset can be regenerated.
    """
    sd = OrderedDict()
    for i, (k, shape) in enumerate(shapes.items()):
        g = torch.Generator(device=device).manual_seed(seed * 1000003 + i)
        rn = lambda: torch.randn(shape, generator=g, device=device)
        if k.endswith(".bias"):
            t = 0.1 * rn()
        elif k.endswith("_embeds_weights"):      # safety-checker thresholds
            t = 0.15 + 0.05 * rn()
        elif _is_norm_key(k):
            t = 1.0 + 0.1 * rn()
        elif k.endswith("quantize.embedding.weight") or k.split(".")[-2:] == ["embedding", "weight"]:
            # VQ codebook (unit scale, or every z_q collapses towards 0) and ClassEmbedder table (nn.Embedding's N(0, 1))
            t = rn()
        elif "embedding" in k:
            t = 0.02 * rn()
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = rn() * fan_in ** -0.5
        sd[prefix + k] = t
    return sd
