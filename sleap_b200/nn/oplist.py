"""int32 op-list records consumed by ``sb_load_model`` (layout mirrored in csrc/sb_model.h)."""
import struct

import numpy as np

SB_OP_WORDS = 24
BUFFER, CONV, TCONV, POOL, UPSAMPLE, ADD, PREPROCESS, COPY = 0, 1, 2, 3, 4, 5, 6, 7
F_RELU, F_BN, F_BILINEAR, F_FUSED_POOL = 1, 2, 8, 16
F_EXPLICIT_PAD = 32      # CONV: w[16] / w[17] = top / left zero padding (otherwise TF SAME is derived from the shapes)
F_FUSED_ADD = 64         # ADD: the CONV before it carries the residual (w[20..23]) and adds it in its epilogue
F_RESIDUAL = 128         # CONV: w[20..23] = shortcut buffer / channel offset, sum buffer / channel offset of the ADD after it
# PREPROCESS modes.  IMAGENET_CAFFE: pretrained ResNet trained on colour frames; IMAGENET_CAFFE_GRAY: trained on
# grayscale frames (its Keras input has 1 channel, so colour frames are converted to gray first, then tile_channels)
PRE_PLAIN, PRE_IMAGENET_CAFFE, PRE_IMAGENET_CAFFE_GRAY = 0, 1, 2


def _rec():
    r = np.zeros((SB_OP_WORDS,), np.int32)
    r[4] = -1
    r[12:16] = -1
    r[18] = -1
    return r


def buffer_record(buf_id, stride_den, C, f32, is_input):
    r = np.zeros((SB_OP_WORDS,), np.int32)
    r[0], r[1], r[2], r[3], r[4], r[5] = BUFFER, buf_id, stride_den, C, int(bool(f32)), int(is_input)
    return r


def preprocess_record(out_buf, C, input_scale, pad_stride, mode=PRE_PLAIN):
    """``mode`` PRE_IMAGENET_CAFFE(_GRAY): after the [0, 1] scaling and zero padding, x * 255, RGB -> BGR, minus the
    ImageNet means (resnet.py imagenet_preproc_v1); _GRAY converts colour frames to gray and tiles it to 3 channels first."""
    r = _rec()
    r[0], r[1], r[6], r[8] = PREPROCESS, -1, out_buf, C
    r[16] = struct.unpack("<i", struct.pack("<f", float(input_scale)))[0]
    r[17] = int(pad_stride)
    r[19] = int(mode)
    return r


def conv_record(in_buf, in_coff, in_C, out_buf, out_coff, out_C, k, stride, relu, w_off, b_off,
                bn_scale_off=-1, bn_shift_off=-1, pool_buf=-1, pool_coff=0, pad=None, res=None):
    """``pad`` = (top, left) explicit zero padding, None = TF SAME.  ``res`` = (shortcut buf, shortcut coff, sum buf,
    sum coff): the ADD record right after this conv adds the shortcut to this conv's output into the sum slice; the
    tensor-core path does that in the conv's epilogue (the ADD record is then skipped)."""
    r = _rec()
    r[0], r[1], r[2], r[3] = CONV, in_buf, in_coff, in_C
    r[6], r[7], r[8], r[9], r[10] = out_buf, out_coff, out_C, k, stride
    r[11] = (F_RELU if relu else 0) | (F_BN if bn_scale_off >= 0 else 0) | (F_EXPLICIT_PAD if pad is not None else 0)
    r[12], r[13], r[14], r[15] = w_off, b_off, bn_scale_off, bn_shift_off
    if pad is not None:
        r[16], r[17] = int(pad[0]), int(pad[1])
    r[18], r[19] = pool_buf, pool_coff
    if res is not None:
        r[11] |= F_RESIDUAL
        r[20], r[21], r[22], r[23] = res
    return r


def tconv_record(in_buf, in_coff, in_C, out_buf, out_coff, out_C, w_off, b_off, k=3):
    r = _rec()
    r[0], r[1], r[2], r[3] = TCONV, in_buf, in_coff, in_C
    r[6], r[7], r[8], r[9], r[10] = out_buf, out_coff, out_C, int(k), 2
    r[11] = F_RELU
    r[12], r[13] = w_off, b_off
    return r


def pool_record(in_buf, in_coff, C, out_buf, out_coff, fused=False, k=2):
    """k = 2: MaxPool2D(2, 2, SAME); k = 3: ZeroPadding2D(1) + MaxPool2D(3, 2, VALID) (ResNet stem)."""
    r = _rec()
    r[0], r[1], r[2], r[3], r[6], r[7], r[8] = POOL, in_buf, in_coff, C, out_buf, out_coff, C
    r[9], r[10] = (3, 2) if k == 3 else (0, 0)
    r[11] = F_FUSED_POOL if fused else 0
    return r


def upsample_record(in_buf, in_coff, C, out_buf, out_coff, bilinear):
    r = _rec()
    r[0], r[1], r[2], r[3], r[6], r[7], r[8] = UPSAMPLE, in_buf, in_coff, C, out_buf, out_coff, C
    r[11] = F_BILINEAR if bilinear else 0
    return r


def add_record(a_buf, a_coff, b_buf, b_coff, C, out_buf, out_coff, relu=False, fused=False):
    r = _rec()
    r[0], r[1], r[2], r[3], r[4], r[5], r[6], r[7], r[8] = ADD, a_buf, a_coff, C, b_buf, b_coff, out_buf, out_coff, C
    r[11] = (F_RELU if relu else 0) | (F_FUSED_ADD if fused else 0)
    return r


def copy_record(in_buf, in_coff, C, out_buf, out_coff):
    r = _rec()
    r[0], r[1], r[2], r[3], r[6], r[7], r[8] = COPY, in_buf, in_coff, C, out_buf, out_coff, C
    return r
