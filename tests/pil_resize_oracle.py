"""Test infrastructure: numpy restatement of Pillow's 8-bit BILINEAR resize (libImaging/Resample.c), the resize behind the
reference's Resize step (transforms/utils.py:28-42), and of the ImageNet classification chain built on it.  Checked against the
installed Pillow and against the reference's outputs recorded in tests/golden/classification.pt."""
import numpy as np

PRECISION_BITS = 22


def axis_coefficients(n_in: int, n_out: int):
    """-> (first source index [n_out], fixed-point weights [n_out, taps]) of an n_in -> n_out resize (zero-padded rows)."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support, ss = fs, 1.0 / fs
    taps = int(np.ceil(support)) * 2 + 1
    first = np.zeros(n_out, np.int64)
    weights = np.zeros((n_out, taps), np.int64)
    for xx in range(n_out):
        center = (xx + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), n_in) - lo
        w = [max(0.0, 1.0 - abs((x + lo - center + 0.5) * ss)) for x in range(n)]
        total = sum(w)  # sequential, as the C loop
        w = [v / total if total != 0.0 else v for v in w]
        first[xx] = lo
        weights[xx, :n] = [int(0.5 + v * (1 << PRECISION_BITS)) for v in w]
    return first, weights


def _pass(img: np.ndarray, n_out: int, axis: int) -> np.ndarray:
    first, weights = axis_coefficients(img.shape[axis], n_out)
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    acc = np.full((n_out,) + src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(weights.shape[1]):
        idx = np.minimum(first + t, src.shape[0] - 1)  # taps past n carry weight 0
        acc += src[idx] * weights[:, t].reshape((-1,) + (1,) * (src.ndim - 1))
    return np.moveaxis(np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis)


def resize_bilinear_u8(img: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """== np.array(PIL.Image.fromarray(img).resize((out_w, out_h), PIL.Image.BILINEAR)) for uint8 H x W x C; an axis whose size
    does not change is not resampled, and the horizontal pass runs first."""
    out = img
    if out_w != img.shape[1]:
        out = _pass(out, out_w, 1)
    if out_h != img.shape[0]:
        out = _pass(out, out_h, 0)
    return out


def classification_chain(img: np.ndarray, resize: int, crop: int, reverse=False, max_value=255.0, mean=None, std=None) -> np.ndarray:
    """[ReverseImageChannels] Resize(resize) CenterCrop(crop) StandardizeImage [NormalizeImage] ImagePermute -> float32 [3, crop, crop]
    (processing.py:614-680, 260-330)."""
    if reverse:
        img = img[:, :, ::-1]
    h, w = img.shape[:2]
    s = max(resize / h, resize / w)
    if s != 1.0:
        img = resize_bilinear_u8(np.ascontiguousarray(img), int(h * s), int(w * s))
    h, w = img.shape[:2]
    top, left = (h - crop) // 2, (w - crop) // 2
    x = (img[top : top + crop, left : left + crop] / max_value).astype(np.float32)
    if mean is not None:
        x = (x - np.array(mean, np.float32)) / np.array(std, np.float32)
    return np.ascontiguousarray(x.transpose(2, 0, 1))
