"""The quantized 2-D convolution as an im2col + the linear oracle (numpy, float64 where it matters).

The reference's QConv2d forward is F.conv2d(x, w.dequantize(), bias) (optimum/quanto/nn/qconv2d.py with the weight's
qfallback): an exact sum over k = c * kh * kw + r * kw + s of x[b, c, oh * s_h - p_h + r * d_h, ow * s_w - p_w + s * d_w]
times the dequantised weight viewed as [Cout, K], plus the bias, rounded ONCE to the dtype: on the CPU the reference's
convolution adds the bias inside the sum (tests/test_qconv2d_host.py pins that on its fixture), and the sm_90a kernel
does the same.  So the conv is the linear of `quanto_oracle.linear_from_dequantized` on the im2col matrix
[M = B * Ho * Wo, K] with the bias as one more k whose activation is 1, and shares the linear's parity contract
(DESIGN 4).
"""
import numpy as np

from . import quanto_oracle as O


def out_size(h, k, stride, pad, dil):
    return (h + 2 * pad - dil * (k - 1) - 1) // stride + 1


def im2col(x, kh, kw, stride=(1, 1), padding=(0, 0), dilation=(1, 1)):
    """x [B, C, H, W] (any float dtype) -> [B * Ho * Wo, C * kh * kw] in (c, r, s) order, zeros for padding taps."""
    b, c, h, w = x.shape
    ho = out_size(h, kh, stride[0], padding[0], dilation[0])
    wo = out_size(w, kw, stride[1], padding[1], dilation[1])
    xp = np.zeros((b, c, h + 2 * padding[0], w + 2 * padding[1]), dtype=x.dtype)
    xp[:, :, padding[0]:padding[0] + h, padding[1]:padding[1] + w] = x
    cols = np.empty((b, ho, wo, c, kh, kw), dtype=x.dtype)
    for r in range(kh):
        for s in range(kw):
            r0, s0 = r * dilation[0], s * dilation[1]
            patch = xp[:, :, r0:r0 + stride[0] * (ho - 1) + 1:stride[0], s0:s0 + stride[1] * (wo - 1) + 1:stride[1]]
            cols[:, :, :, :, r, s] = patch.transpose(0, 2, 3, 1)
    return cols.reshape(b * ho * wo, c * kh * kw), (b, ho, wo)


def conv_from_dequantized(x_f32, w_f32, bias_f32, tag, stride=(1, 1), padding=(0, 0), dilation=(1, 1)):
    """x [B, C, H, W], w [Cout, C, kh, kw] (dequantised, as float32), bias [Cout] or None -> (y_exact_f64,
    y_rounded_storage, tol, cols): y_exact = im2col(x) @ w^T + bias in float64, y_rounded its single rounding to `tag`
    and tol half an output ulp, each [B, Cout, Ho, Wo]; cols the im2col matrix [M, K] (plus a column of ones with a
    bias)."""
    cout, _, kh, kw = w_f32.shape
    cols, (b, ho, wo) = im2col(np.asarray(x_f32, np.float32), kh, kw, stride, padding, dilation)
    w2 = np.asarray(w_f32, np.float32).reshape(cout, -1)
    if bias_f32 is not None:
        cols = np.concatenate([cols, np.ones((cols.shape[0], 1), np.float32)], axis=1)
        w2 = np.concatenate([w2, np.asarray(bias_f32, np.float32).reshape(cout, 1)], axis=1)
    y64, y, tol = O.linear_from_dequantized(cols, w2, None, tag)

    def nchw(t):
        return t.reshape(b, ho, wo, cout).transpose(0, 3, 1, 2)

    return nchw(y64), nchw(y), nchw(tol), cols
