"""ORACLE - TEST INFRASTRUCTURE ONLY.  numpy restatement of the image preparation of the reference's eval loader
(datasets/general_eval.py:112-131, 210-211), the rules csrc/image_prep.cu implements:

  resize_u8(img, H, W, pad_rows)   <- np.pad(img, ((pad, pad), (0, 0), (0, 0)), 'edge') + cv2.resize(img, (W, H)), uint8
  normalize(u8, mean, std)          <- transforms.ToTensor() + transforms.Normalize(mean, std), fp32
  fusion_colour(u8)                 <- test.py:287-292 (img * std + mean, clip(img * 255), astype(uint8)) read back as
                                       read_img does (float32 / 255), before the JPEG encode

The resize is cv2's INTER_LINEAR for uint8 at the bit level: coefficients from the double scale rounded to float, 11-bit
fixed-point weights, and the vertical pass of cv2's SIMD path (VResizeLinearVec_32s8u), which drops 4 bits of each
horizontal sum before a 16-bit high multiply.  The textbook (S0 b0 + S1 b1 + 2^21) >> 22 differs from it by one in
about 30 % of pixels.
"""
import numpy as np

MEAN = np.array([0.485, 0.456, 0.406], dtype=np.float32)
STD = np.array([0.229, 0.224, 0.225], dtype=np.float32)
COEF = 2048   # INTER_RESIZE_COEF_SCALE


def _axis(n_out, n_in):
    """source index and fraction per output coordinate, before clamping: (sx int64 [n_out], fx float32 [n_out])"""
    scale = 1.0 / (float(n_out) / n_in)
    d = np.arange(n_out, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    return s, f


def _weights(f):
    a0 = np.rint((np.float32(1.0) - f) * np.float32(COEF)).astype(np.int64)
    a1 = np.rint(f * np.float32(COEF)).astype(np.int64)
    return a0, a1


def resize_coefficients(h, w, H, W):
    """(x0, x1, a0, a1) per output column and (y0, y1, b0, b1) per output row of an h x w -> H x W resize"""
    sx, fx = _axis(W, w)
    lo = sx < 0
    fx[lo], sx[lo] = 0, 0
    hi = sx >= w - 1
    fx[hi], sx[hi] = 0, w - 1
    x1 = np.minimum(sx + 1, w - 1)
    a0, a1 = _weights(fx)
    sy, fy = _axis(H, h)            # rows: the fraction is kept, both rows are clamped
    y0, y1 = np.clip(sy, 0, h - 1), np.clip(sy + 1, 0, h - 1)
    b0, b1 = _weights(fy)
    return (sx, x1, a0, a1), (y0, y1, b0, b1)


def resize_u8(img, H, W, pad_rows=0):
    """uint8 [h,w,C] -> uint8 [H,W,C]: edge-pad pad_rows rows top and bottom, then cv2.resize(img, (W, H))"""
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim != 3:
        raise ValueError(f"resize_u8: expected uint8 [h,w,C], got {img.dtype} {img.shape}")
    if pad_rows:
        img = np.pad(img, ((pad_rows, pad_rows), (0, 0), (0, 0)), "edge")
    h, w = img.shape[:2]
    (x0, x1, a0, a1), (y0, y1, b0, b1) = resize_coefficients(h, w, H, W)
    src = img.astype(np.int64)
    # horizontal pass: exact integer sums per source row
    S = a0[None, :, None] * src[:, x0, :] + a1[None, :, None] * src[:, x1, :]          # [h, W, C]
    S0, S1 = S[y0] >> 4, S[y1] >> 4
    out = (((S0 * b0[:, None, None]) >> 16) + ((S1 * b1[:, None, None]) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def normalize(u8):
    """uint8 [...,H,W,3] -> fp32 [...,3,H,W] = (u8 / 255 - mean) / std, each step one fp32 operation"""
    x = np.moveaxis(np.asarray(u8), -1, -3).astype(np.float32) / np.float32(255)
    shape = (3, 1, 1)
    return ((x - MEAN.reshape(shape)) / STD.reshape(shape)).astype(np.float32)


def fusion_colour(u8):
    """uint8 [...,H,W,3] -> fp32 [...,3,H,W]: trunc(clip((norm * std + mean) * 255, 0, 255)) / 255"""
    shape = (3, 1, 1)
    c = normalize(u8) * STD.reshape(shape) + MEAN.reshape(shape)
    q = np.clip(c * np.float32(255), 0, 255).astype(np.uint8)
    return q.astype(np.float32) / np.float32(255)
