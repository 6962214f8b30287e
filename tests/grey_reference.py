"""numpy model of the grey frames the reference reads: cv2.imread(path, cv2.IMREAD_GRAYSCALE) (OpenCV 4.13) of a colour 8-bit
PNG, as a function of the BGR pixels cv2.imwrite stored in it.

    grey = (9797 * R + 19234 * G + 3737 * B) >> 15

in integers: truncation, no rounding offset; the weights sum to 2^15, so white stays 255.  Alpha is ignored: a BGRA PNG read
with IMREAD_GRAYSCALE gives the grey of its BGR channels.  Each constant was settled by probing live cv2 (DESIGN 5.11);
tests/test_grey_reference_cpu.py pins the model against cv2 on all 2^24 colours.  cv2.cvtColor(COLOR_BGR2GRAY), whose weights
are 4899 / 9617 / 1868 with a rounding >> 14, differs from it by one grey level on half of the colours.
"""
import numpy as np

COEF_R, COEF_G, COEF_B = 9797, 19234, 3737
SHIFT = 15
ORDERS = ("bgr", "rgb", "bgra", "rgba")


def grey_from_bgr(bgr_u8: np.ndarray) -> np.ndarray:
    """uint8 [..., 3] (or [..., 4], alpha ignored) in BGR order -> uint8 [...]: IMREAD_GRAYSCALE of the PNG holding them."""
    bgr = np.asarray(bgr_u8)
    if bgr.dtype != np.uint8 or bgr.ndim < 1 or bgr.shape[-1] not in (3, 4):
        raise ValueError(f"bgr_u8 must be uint8 [..., 3 or 4], got {bgr.dtype} {list(bgr.shape)}")
    b, g, r = (bgr[..., c].astype(np.int32) for c in range(3))
    return ((COEF_R * r + COEF_G * g + COEF_B * b) >> SHIFT).astype(np.uint8)


def to_bgr(pixels_u8: np.ndarray, order: str) -> np.ndarray:
    """The BGR channels of pixels in one of ORDERS (alpha dropped)."""
    if order not in ORDERS:
        raise ValueError(f"order must be one of {ORDERS}, got {order!r}")
    p = np.asarray(pixels_u8)[..., :3]
    return p if order.startswith("bgr") else p[..., ::-1]


def from_bgr(bgr_u8: np.ndarray, order: str, alpha=None) -> np.ndarray:
    """BGR pixels re-laid in `order`; the 4-channel orders take `alpha` (uint8, broadcast to the pixels; 255 when None)."""
    bgr = np.asarray(bgr_u8)
    p = bgr if order.startswith("bgr") else bgr[..., ::-1]
    if order.endswith("a"):
        a = np.broadcast_to(np.uint8(255) if alpha is None else np.asarray(alpha, np.uint8), bgr.shape[:-1])
        p = np.concatenate([p, a[..., None]], axis=-1)
    return np.ascontiguousarray(p)


def every_colour_bgr() -> np.ndarray:
    """uint8 [4096, 4096, 3]: each of the 2^24 BGR colours once, colour v = (B, G, R) = (v >> 16, v >> 8 & 255, v & 255) at
    row v // 4096, column v % 4096."""
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([v >> 16, (v >> 8) & 255, v & 255], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)


def normalised(grey_u8: np.ndarray) -> np.ndarray:
    """The reference's image / 255. of the grey frame (NormalizedDataset, src/datasets/normalized_dataset.py:26-34): float32."""
    return np.asarray(grey_u8).astype(np.float32) / np.float32(255)
