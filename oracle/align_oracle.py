"""CPU oracle of the FFHQ face alignment after the landmarks (utils/shape_predictor.py:105-185), restated with the
same numpy, scipy and Pillow calls, and each stage on its own.  Also the seeded synthetic inputs of
tests/golden/align.npz (oracle/gen_golden_align.py), generated with integer numpy arithmetic only so that every machine
rebuilds the same pixels.

What the library calls compute (probed on Pillow 12.2, scipy 1.18, NumPy 2.3; csrc/hf_align.cu restates it):
* ``Image.resize(size, LANCZOS)``: per axis, scale = in / out, support = 3 max(scale, 1); output o is centred at
  (o + 0.5) scale and reads inputs int(centre - support + 0.5) .. int(centre + support + 0.5) (clamped to the image);
  weight of input i is sinc(t) sinc(t / 3) at t = (i - centre + 0.5) / max(scale, 1), normalised by their float64 sum
  and rounded half away from zero to 22-bit fixed point.  Horizontal pass first, into uint8; each output is
  (2^21 + sum k_i v_i) >> 22 clamped to 0..255.
* ``Image.transform(size, QUAD, data, BILINEAR)``: data = corners NW, SW, SE, NE -> coefficients
  (x0, (ne_x - x0) / w, (sw_x - x0) / h, (se_x - sw_x - ne_x + x0) / (w h), and the same for y) in float64; output
  pixel (x, y) samples a0 + a1 u + a2 v + a3 u v at u = x + 0.5, v = y + 0.5 (no fused multiply-add).  A sample outside
  [0, W) x [0, H) is 0; else s - 0.5 is floored to the pixel pair (indices clamped to the image, the row below
  replaced by the row itself past the bottom), interpolated in float64 along x then y, and truncated to uint8.
* ``scipy.ndimage.gaussian_filter(img, [b, b, 0])``: axis 0 then axis 1, each rounded to float32; radius
  int(4 b + 0.5); the kernel is exactly symmetric so the correlation is w0 x_i + sum_{j = r..1} w_j (x_{i-j} + x_{i+j})
  in float64 in that order; 'reflect' extends half-sample symmetrically (the edge sample repeats).
* ``np.pad(..., 'reflect')`` mirrors about the edge sample (not repeated).  Under NumPy 2 ``np.float32(x) / pad[0]``
  is float64 (pad is an int64 array), so the mask and both blend right-hand sides are float64 and each ``img +=``
  rounds to float32; ``np.median`` of an even count is the float32 mean of the two middle values.
"""
from __future__ import annotations

import numpy as np
import PIL.Image
import scipy.ndimage
import torch

OUTPUT_SIZE, TRANSFORM_SIZE = 1024, 4096

# ---- seeded synthetic inputs ------------------------------------------------------------------------------------------
# landmark template in units of the inter-ocular distance, eye midpoint at the origin, y down: jaw (0-16), brows
# (17-26), nose (27-35), eyes (36-47, six points each around the centres (-0.5, 0) / (0.5, 0)), mouth (48-67, corners
# 48 and 54 at (-/+0.4, 1.05))
_EYE = np.array([[-0.15, 0.0], [-0.07, -0.05], [0.05, -0.05], [0.15, 0.0], [0.05, 0.04], [-0.07, 0.04]])


def landmark_template() -> np.ndarray:
    t = np.linspace(-1.0, 1.0, 17)
    jaw = np.stack([0.95 * t, 0.1 + 1.35 * (1.0 - t * t) ** 0.5], 1)
    brows = np.stack([np.r_[np.linspace(-0.8, -0.2, 5), np.linspace(0.2, 0.8, 5)], np.full(10, -0.3)], 1)
    nose = np.r_[np.stack([np.zeros(4), np.linspace(0.1, 0.55, 4)], 1),
                 np.stack([np.linspace(-0.2, 0.2, 5), np.full(5, 0.65)], 1)]
    eyes = np.r_[_EYE + [-0.5, 0.0], _EYE + [0.5, 0.0]]
    a = np.linspace(0.0, 2 * np.pi, 12, endpoint=False)
    outer = np.stack([-0.4 * np.cos(a), 1.05 - 0.15 * np.sin(a)], 1)
    b = np.linspace(0.0, 2 * np.pi, 8, endpoint=False)
    inner = np.stack([-0.3 * np.cos(b), 1.05 - 0.06 * np.sin(b)], 1)
    lm = np.r_[jaw, brows, nose, eyes, outer, inner]
    assert lm.shape == (68, 2)
    return lm


def synth_landmarks(eye_mid, inter_ocular, angle_deg=0.0) -> np.ndarray:
    """Integer landmarks (as dlib returns them) of the template scaled, rotated and placed at `eye_mid`."""
    th = np.deg2rad(angle_deg)
    rot = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    pts = landmark_template() @ rot.T * inter_ocular + np.asarray(eye_mid, dtype=np.float64)
    return np.rint(pts).astype(np.int64)


def synth_image(height: int, width: int, seed: int, cell: int | None = None) -> np.ndarray:
    """Smooth uint8 [H, W, 3]: a seeded coarse grid of `cell`-pixel cells (default 3/8 of the longer side) upsampled
    with integer bilinear weights (integer arithmetic only, identical on every machine; smooth, so that the golden
    outputs compress to a few hundred kB)."""
    if cell is None:
        cell = max(64, 3 * max(height, width) // 8)
    rng = np.random.default_rng(seed)
    gh, gw = height // cell + 2, width // cell + 2
    grid = rng.integers(16, 240, size=(gh, gw, 3), dtype=np.int64)
    y, x = np.arange(height), np.arange(width)
    iy, fy = y // cell, (y % cell)[:, None, None]
    ix, fx = x // cell, (x % cell)[None, :, None]
    g00, g01 = grid[iy][:, ix], grid[iy][:, ix + 1]
    g10, g11 = grid[iy + 1][:, ix], grid[iy + 1][:, ix + 1]
    v = (g00 * (cell - fx) * (cell - fy) + g01 * fx * (cell - fy) + g10 * (cell - fx) * fy + g11 * fx * fy)
    return np.ascontiguousarray(v // (cell * cell), dtype=np.uint8)


# name -> (height, width, image seed, eye midpoint (x, y), inter-ocular px, roll in degrees, input form)
CASES = {
    "crop":         (1024, 1024, 101, (512, 470), 200, 0.0, "u8"),       # quad inside the image: crop only
    "pad":          (1024, 1024, 102, (512, 440), 420, 0.0, "u8"),       # large face: the padding branch
    "shrink":       (4800, 4800, 103, (2400, 2250), 1100, 0.0, "u8"),    # shrink = 2 before the crop
    "tilted":       (1024, 1024, 104, (260, 300), 230, 27.0, "u8"),      # rolled face by the corner, padded
    "odd":          (757, 1001, 105, (431, 350), 150, -8.0, "u8"),       # odd, non-square size
    "float_tensor": (1024, 1024, 101, (512, 470), 200, 0.0, "float"),    # the crop image as a float tensor
    "pil":          (1024, 1024, 101, (512, 470), 200, 0.0, "pil"),      # ... and as a PIL image
}


def case_input(name):
    """(what the case passes to align_face, its landmarks [68, 2] int64, the uint8 HWC image it was made from; the
    float form's PIL image is what pil_input makes of it)."""
    h, w, seed, mid, io, angle, form = CASES[name]
    img = synth_image(h, w, seed)
    lm = synth_landmarks(mid, io, angle)
    if form == "u8":
        data = torch.from_numpy(img).permute(2, 0, 1).contiguous()
    elif form == "float":
        # fractional values between the uint8 levels: ToPILImage's mul(255).byte() truncates them
        frac = np.random.default_rng(seed + 1).integers(0, 256, size=img.shape, dtype=np.int64)
        f32 = np.minimum((img.astype(np.int64) * 256 + frac).astype(np.float32) / np.float32(255 * 256), 1.0)
        data = torch.from_numpy(f32).permute(2, 0, 1).contiguous()
    else:
        data = PIL.Image.fromarray(img)
    return data, lm, img


def pil_input(data) -> PIL.Image.Image:
    """The PIL image get_landmark_from_tensors hands on (shape_predictor.py:56-60): T.ToPILImage() of a tensor."""
    from torchvision import transforms as T
    return T.ToPILImage()(data) if isinstance(data, torch.Tensor) else data


def encode_output(img_u8: np.ndarray) -> np.ndarray:
    """[H, W, 3] -> [3, H, W] row differences modulo 256, one plane per channel (lossless; the golden stores outputs
    this way because zlib compresses the small differences of a smooth image several times better)."""
    planes = np.ascontiguousarray(img_u8.transpose(2, 0, 1))
    return np.diff(planes, axis=2, prepend=np.zeros_like(planes[:, :, :1]))


def decode_output(dx_u8: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(np.cumsum(dx_u8, axis=2, dtype=np.uint8).transpose(1, 2, 0))


def golden_output(gold, name: str) -> np.ndarray:
    """The reference's uint8 output of golden case `name`."""
    twin = str(gold[f"{name}_twin"]) if f"{name}_twin" in gold.files else name
    return decode_output(gold[f"{twin}_out_dx"])


class FakeDlib:
    """Stand-in for dlib inside utils.shape_predictor: the detector finds one face in every image, the predictor
    returns the given landmark sets in turn (call k gets set k mod n)."""

    class _Rect:
        def width(self):
            return 100

        def height(self):
            return 100

    class _Point:
        def __init__(self, x, y):
            self.x, self.y = int(x), int(y)

    class _Shape:
        def __init__(self, lm):
            self._parts = [FakeDlib._Point(x, y) for x, y in lm]

        def parts(self):
            return self._parts

    def __init__(self, landmark_sets):
        self.sets = [np.asarray(lm) for lm in landmark_sets]
        self.calls = 0

    def get_frontal_face_detector(self):
        return lambda img, upsample: [FakeDlib._Rect()]

    def predictor(self, img, det):
        lm = self.sets[self.calls % len(self.sets)]
        self.calls += 1
        return FakeDlib._Shape(lm)

    def shape_predictor(self, path):
        return self.predictor


# ---- geometry (:105-179) ---------------------------------------------------------------------------------------------
def boxes(lm, size):
    """The reference's integer boxes for an image of size (w, h): {'rsize': (w, h) or None, 'crop': (x0, y0, x1, y1)
    or None, 'pad': (l, t, r, b) or None, 'quad': final [4, 2] float64, 'qsize', 'blur'}."""
    lm = np.asarray(lm)
    eye_left, eye_right = np.mean(lm[36:42], axis=0), np.mean(lm[42:48], axis=0)
    eye_avg = (eye_left + eye_right) * 0.5
    eye_to_eye = eye_right - eye_left
    mouth_avg = (lm[48:60][0] + lm[48:60][6]) * 0.5
    eye_to_mouth = mouth_avg - eye_avg
    x = eye_to_eye - np.flipud(eye_to_mouth) * [-1, 1]
    x /= np.hypot(*x)
    x *= max(np.hypot(*eye_to_eye) * 2.0, np.hypot(*eye_to_mouth) * 1.8)
    y = np.flipud(x) * [-1, 1]
    c = eye_avg + eye_to_mouth * 0.1
    quad = np.stack([c - x - y, c - x + y, c + x + y, c + x - y])
    qsize = np.hypot(*x) * 2
    size = tuple(size)
    out = {"rsize": None, "crop": None, "pad": None}
    shrink = int(np.floor(qsize / OUTPUT_SIZE * 0.5))
    if shrink > 1:
        size = (int(np.rint(float(size[0]) / shrink)), int(np.rint(float(size[1]) / shrink)))
        out["rsize"] = size
        quad /= shrink
        qsize /= shrink
    border = max(int(np.rint(qsize * 0.1)), 3)
    crop = (int(np.floor(min(quad[:, 0]))), int(np.floor(min(quad[:, 1]))), int(np.ceil(max(quad[:, 0]))),
            int(np.ceil(max(quad[:, 1]))))
    crop = (max(crop[0] - border, 0), max(crop[1] - border, 0), min(crop[2] + border, size[0]),
            min(crop[3] + border, size[1]))
    if crop[2] - crop[0] < size[0] or crop[3] - crop[1] < size[1]:
        out["crop"] = crop
        size = (crop[2] - crop[0], crop[3] - crop[1])
        quad -= crop[0:2]
    pad = (int(np.floor(min(quad[:, 0]))), int(np.floor(min(quad[:, 1]))), int(np.ceil(max(quad[:, 0]))),
           int(np.ceil(max(quad[:, 1]))))
    pad = (max(-pad[0] + border, 0), max(-pad[1] + border, 0), max(pad[2] - size[0] + border, 0),
           max(pad[3] - size[1] + border, 0))
    if max(pad) > border - 4:
        pad = np.maximum(pad, int(np.rint(qsize * 0.3)))
        out["pad"] = tuple(int(p) for p in pad)
        quad += pad[:2]
    out.update(quad=quad, qsize=float(qsize), blur=float(qsize * 0.02))
    return out


# ---- stages -----------------------------------------------------------------------------------------------------------
def resample(img_u8: np.ndarray, width: int, height: int) -> np.ndarray:
    """Image.resize((width, height), LANCZOS) (:149 with ANTIALIAS = LANCZOS, :185)."""
    return np.asarray(PIL.Image.fromarray(img_u8).resize((width, height), PIL.Image.LANCZOS))


def gaussian(x_f32: np.ndarray, sigma: float) -> np.ndarray:
    return scipy.ndimage.gaussian_filter(x_f32, [sigma, sigma, 0])


def median(x_f32: np.ndarray) -> np.ndarray:
    return np.median(x_f32, axis=(0, 1))


def pad_blend(img_u8: np.ndarray, pad, blur: float) -> np.ndarray:
    """:170-178 with pad = (left, top, right, bottom) as an int64 array, as np.maximum leaves it."""
    pad = np.asarray(pad, dtype=np.int64)
    img = np.pad(np.float32(img_u8), ((pad[1], pad[3]), (pad[0], pad[2]), (0, 0)), 'reflect')
    h, w, _ = img.shape
    y, x, _ = np.ogrid[:h, :w, :1]
    mask = np.maximum(1.0 - np.minimum(np.float32(x) / pad[0], np.float32(w - 1 - x) / pad[2]),
                      1.0 - np.minimum(np.float32(y) / pad[1], np.float32(h - 1 - y) / pad[3]))
    img += (scipy.ndimage.gaussian_filter(img, [blur, blur, 0]) - img) * np.clip(mask * 3.0 + 1.0, 0.0, 1.0)
    img += (np.median(img, axis=(0, 1)) - img) * np.clip(mask, 0.0, 1.0)
    return np.uint8(np.clip(np.rint(img), 0, 255))


def quad(img_u8: np.ndarray, data, width: int, height: int) -> np.ndarray:
    """Image.transform((width, height), QUAD, data, BILINEAR) (:182-183)."""
    return np.asarray(PIL.Image.fromarray(img_u8).transform((width, height), PIL.Image.QUAD,
                                                            np.asarray(data, dtype=np.float64).flatten(),
                                                            PIL.Image.BILINEAR))


def align(img_u8: np.ndarray, lm) -> np.ndarray:
    """:105-185 for one uint8 RGB image and its landmarks -> [1024, 1024, 3] uint8."""
    b = boxes(lm, (img_u8.shape[1], img_u8.shape[0]))
    img = img_u8
    if b["rsize"] is not None:
        img = resample(img, *b["rsize"])
    if b["crop"] is not None:
        x0, y0, x1, y1 = b["crop"]
        img = np.ascontiguousarray(img[y0:y1, x0:x1])
    if b["pad"] is not None:
        img = pad_blend(img, b["pad"], b["blur"])
    img = quad(img, b["quad"] + 0.5, TRANSFORM_SIZE, TRANSFORM_SIZE)
    return resample(img, OUTPUT_SIZE, OUTPUT_SIZE)
