"""FFHQ face alignment (utils/shape_predictor.py:80-194) with everything after the landmarks on sm_90a kernels.

    from hairfastgan_b200.face_align import align_face, align_from_landmarks
    tensors = align_face([img_tensor], predictor)                 # drop-in for utils.shape_predictor.align_face
    out_u8 = align_from_landmarks(img_u8_hwc_cuda, lm)            # [1024, 1024, 3] uint8 CUDA, own landmarks

The landmarks still come from dlib on the CPU through the reference's own ``get_landmark`` /
``get_landmark_from_tensors``.  The crop geometry is computed here in float64 numpy (restating :105-170), so the
integer shrink, crop and pad boxes are the reference's.  The image is uploaded once as uint8 HWC; the shrink, padding,
blur, blends, QUAD transform and final resize run in csrc/hf_align.cu and compute what Pillow, scipy and numpy compute
(DESIGN.md, "Face alignment").  Only 8-bit RGB images are supported: anything else raises NotImplementedError.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib

OUTPUT_SIZE = 1024          # shape_predictor.py:140
TRANSFORM_SIZE = 4096       # :142


# ---- host geometry ---------------------------------------------------------------------------------------------------
@dataclass
class Geometry:
    """The reference's crop plan for one face in an image of `size` = (width, height)."""
    quad: np.ndarray            # [4, 2] float64 corners in the coordinates of the image the QUAD transform reads
    qsize: float
    shrink: int                 # > 1: resize to rsize first
    rsize: tuple | None         # (width, height) after the shrink
    crop: tuple | None          # (x0, y0, x1, y1) in the (shrunk) image, or None when the crop keeps the whole image
    pad: tuple | None           # (left, top, right, bottom) of the padding branch, or None
    blur: float                 # Gaussian sigma of the padding branch


def geometry(lm, size) -> Geometry:
    """Restates shape_predictor.py:105-179 with the same float64 operations in the same order."""
    lm = np.asarray(lm)
    eye_left = np.mean(lm[36:42], axis=0)
    eye_right = np.mean(lm[42:48], axis=0)
    eye_avg = (eye_left + eye_right) * 0.5
    eye_to_eye = eye_right - eye_left
    mouth_avg = (lm[48] + lm[54]) * 0.5                 # outer mouth corners, lm_mouth_outer[0] and [6]
    eye_to_mouth = mouth_avg - eye_avg
    x = eye_to_eye - np.flipud(eye_to_mouth) * [-1, 1]
    x /= np.hypot(*x)
    x *= max(np.hypot(*eye_to_eye) * 2.0, np.hypot(*eye_to_mouth) * 1.8)
    y = np.flipud(x) * [-1, 1]
    c = eye_avg + eye_to_mouth * 0.1
    quad = np.stack([c - x - y, c - x + y, c + x + y, c + x - y])
    qsize = np.hypot(*x) * 2

    w, h = int(size[0]), int(size[1])
    shrink = int(np.floor(qsize / OUTPUT_SIZE * 0.5))
    rsize = None
    if shrink > 1:
        rsize = (int(np.rint(float(w) / shrink)), int(np.rint(float(h) / shrink)))
        w, h = rsize
        quad /= shrink
        qsize /= shrink

    border = max(int(np.rint(qsize * 0.1)), 3)
    crop = (int(np.floor(min(quad[:, 0]))), int(np.floor(min(quad[:, 1]))), int(np.ceil(max(quad[:, 0]))),
            int(np.ceil(max(quad[:, 1]))))
    crop = (max(crop[0] - border, 0), max(crop[1] - border, 0), min(crop[2] + border, w), min(crop[3] + border, h))
    if crop[2] - crop[0] < w or crop[3] - crop[1] < h:
        quad -= crop[0:2]
        w, h = crop[2] - crop[0], crop[3] - crop[1]
    else:
        crop = None

    pad = (int(np.floor(min(quad[:, 0]))), int(np.floor(min(quad[:, 1]))), int(np.ceil(max(quad[:, 0]))),
           int(np.ceil(max(quad[:, 1]))))
    pad = (max(-pad[0] + border, 0), max(-pad[1] + border, 0), max(pad[2] - w + border, 0), max(pad[3] - h + border, 0))
    if max(pad) > border - 4:
        pad = np.maximum(pad, int(np.rint(qsize * 0.3)))
        quad += pad[:2]
        pad = tuple(int(p) for p in pad)
    else:
        pad = None
    return Geometry(quad=quad, qsize=float(qsize), shrink=shrink, rsize=rsize, crop=crop, pad=pad,
                    blur=float(qsize * 0.02))


def gaussian_half_kernel(sigma: float, truncate: float = 4.0) -> np.ndarray:
    """scipy.ndimage's order-0 Gaussian of `sigma` (radius int(truncate sigma + 0.5), normalised by its float64 sum),
    from the centre tap outwards: [radius + 1] float64.  The kernel is exactly symmetric."""
    if sigma <= 1e-15:                                   # gaussian_filter skips such an axis
        return np.ones(1)
    radius = int(truncate * float(sigma) + 0.5)
    taps = np.arange(-radius, radius + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * taps ** 2)
    phi = phi / phi.sum()
    return np.ascontiguousarray(phi[radius:])


def quad_coefficients(data, width: int, height: int) -> np.ndarray:
    """The bilinear map Pillow's Image.transform(size, QUAD, data) samples with: data = the corners NW, SW, SE, NE;
    source (a0 + a1 u + a2 v + a3 u v, a4 + a5 u + a6 v + a7 u v) for output pixel centre (u, v)."""
    d = [np.float64(v) for v in np.asarray(data, dtype=np.float64).ravel()]
    x0, y0, sw, se, ne = d[0], d[1], d[2:4], d[4:6], d[6:8]
    sx, sy = 1.0 / width, 1.0 / height
    return np.array([x0, (ne[0] - x0) * sx, (sw[0] - x0) * sy, (se[0] - sw[0] - ne[0] + x0) * sx * sy,
                     y0, (ne[1] - y0) * sx, (sw[1] - y0) * sy, (se[1] - sw[1] - ne[1] + y0) * sx * sy],
                    dtype=np.float64)


# ---- kernels --------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=64)
def lanczos_table(in_size: int, out_size: int) -> np.ndarray:
    """Pillow's LANCZOS coefficients of one axis: [out_size, taps + 2] int32 (first input, count, 22-bit weights)."""
    taps = _lib.lib().hf_align_lanczos_taps(in_size, out_size)
    if taps < 0:
        raise ValueError(f"lanczos_table: bad sizes {in_size} -> {out_size}")
    table = np.zeros((out_size, taps + 2), dtype=np.int32)
    _lib.check(_lib.lib().hf_align_lanczos_coeffs(in_size, out_size, table.ctypes.data), "hf_align_lanczos_coeffs")
    return table


@functools.lru_cache(maxsize=64)
def _device_table(in_size: int, out_size: int, device: torch.device) -> torch.Tensor:
    return torch.from_numpy(lanczos_table(in_size, out_size)).to(device)


def _image_u8(t: torch.Tensor, what: str):
    """(pointer, height, width, pitch) of a uint8 CUDA [H, W, 3] image whose pixels are packed along each row (a crop
    window of a larger image qualifies)."""
    if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
        raise NotImplementedError(f"{what}: expected a uint8 [H, W, 3] RGB tensor, got "
                                  f"{getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))}")
    if not t.is_cuda:
        raise RuntimeError(f"{what}: the image must be on a CUDA device (no CPU fallback)")
    if t.stride(2) != 1 or t.stride(1) != 3 or t.stride(0) % 3 or t.stride(0) < 3 * t.shape[1]:
        raise ValueError(f"{what}: pixels must be packed along each row, got strides {t.stride()}")
    _lib.use_device(t.device.index)
    return t.data_ptr(), t.shape[0], t.shape[1], t.stride(0) // 3


def resample(image: torch.Tensor, width: int, height: int) -> torch.Tensor:
    """Image.resize((width, height), Image.LANCZOS) of a uint8 [H, W, 3] CUDA image."""
    ptr, H, W, pitch = _image_u8(image, "resample")
    dev = image.device
    out = torch.empty((height, width, 3), dtype=torch.uint8, device=dev)
    ws = torch.empty(max(_lib.lib().hf_align_resample_workspace_bytes(H, W, height, width), 1), dtype=torch.uint8,
                     device=dev)
    cx = _device_table(W, width, dev) if width != W else None
    cy = _device_table(H, height, dev) if height != H else None
    _lib.check(_lib.lib().hf_align_resample_u8(ptr, H, W, pitch, out.data_ptr(), height, width,
                                               cx.data_ptr() if cx is not None else None,
                                               cy.data_ptr() if cy is not None else None, ws.data_ptr(),
                                               _lib.stream_ptr()), "hf_align_resample_u8")
    return out


def pad_blend(image: torch.Tensor, pad, blur: float) -> torch.Tensor:
    """shape_predictor.py:170-178 on a uint8 [H, W, 3] CUDA image: reflect padding by pad = (left, top, right,
    bottom), the Gaussian-blur blend toward the edges, the blend toward the channel medians, rounding to uint8."""
    ptr, H, W, pitch = _image_u8(image, "pad_blend")
    pad = tuple(int(p) for p in pad)
    Hp, Wp = H + pad[1] + pad[3], W + pad[0] + pad[2]
    dev = image.device
    w = torch.from_numpy(gaussian_half_kernel(blur)).to(dev)
    out = torch.empty((Hp, Wp, 3), dtype=torch.uint8, device=dev)
    ws = torch.empty(_lib.lib().hf_align_pad_blend_workspace_bytes(Hp, Wp), dtype=torch.uint8, device=dev)
    _lib.check(_lib.lib().hf_align_pad_blend_u8(ptr, H, W, pitch, (C.c_int * 4)(*pad), w.data_ptr(), w.numel() - 1,
                                                out.data_ptr(), ws.data_ptr(), _lib.stream_ptr()),
               "hf_align_pad_blend_u8")
    return out


def gaussian(x: torch.Tensor, sigma: float) -> torch.Tensor:
    """scipy.ndimage.gaussian_filter(x, [sigma, sigma, 0]) of a float32 [H, W, 3] CUDA image."""
    if x.dtype != torch.float32 or x.dim() != 3 or x.shape[2] != 3 or not x.is_cuda:
        raise NotImplementedError("gaussian: expected a float32 [H, W, 3] CUDA tensor")
    x = x.contiguous()
    _lib.use_device(x.device.index)
    w = torch.from_numpy(gaussian_half_kernel(sigma)).to(x.device)
    y, ws = torch.empty_like(x), torch.empty_like(x)
    _lib.check(_lib.lib().hf_align_gaussian_f32(x.data_ptr(), y.data_ptr(), x.shape[0], x.shape[1], w.data_ptr(),
                                                w.numel() - 1, ws.data_ptr(), _lib.stream_ptr()),
               "hf_align_gaussian_f32")
    return y


def median(x: torch.Tensor) -> torch.Tensor:
    """np.median(x, axis=(0, 1)) of a float32 [..., 3] CUDA tensor: [3] float32."""
    if x.dtype != torch.float32 or x.shape[-1] != 3 or not x.is_cuda:
        raise NotImplementedError("median: expected a float32 [..., 3] CUDA tensor")
    x = x.contiguous()
    _lib.use_device(x.device.index)
    med = torch.empty(3, dtype=torch.float32, device=x.device)
    ws = torch.empty(_lib.lib().hf_align_median_workspace_bytes(), dtype=torch.uint8, device=x.device)
    _lib.check(_lib.lib().hf_align_median_f32(x.data_ptr(), x.numel() // 3, med.data_ptr(), ws.data_ptr(),
                                              _lib.stream_ptr()), "hf_align_median_f32")
    return med


def quad_transform(image: torch.Tensor, data, width: int, height: int) -> torch.Tensor:
    """Image.transform((width, height), Image.QUAD, data, Image.BILINEAR) of a uint8 [H, W, 3] CUDA image."""
    ptr, H, W, pitch = _image_u8(image, "quad_transform")
    coeffs = quad_coefficients(data, width, height)
    out = torch.empty((height, width, 3), dtype=torch.uint8, device=image.device)
    _lib.check(_lib.lib().hf_align_quad_u8(ptr, H, W, pitch, coeffs.ctypes.data_as(C.POINTER(C.c_double)),
                                           out.data_ptr(), width, height, _lib.stream_ptr()), "hf_align_quad_u8")
    return out


def align_from_landmarks(image: torch.Tensor, lm) -> torch.Tensor:
    """The aligned 1024^2 face of a uint8 [H, W, 3] RGB CUDA image (any strides) given its 68 dlib landmarks (x, y):
    [1024, 1024, 3] uint8 on the image's device, what shape_predictor.py:105-185 makes of the same image and
    landmarks."""
    if isinstance(image, torch.Tensor) and image.dim() == 3 and (image.stride(2) != 1 or image.stride(1) != 3):
        image = image.contiguous()                       # e.g. a CHW tensor permuted to HWC
    _image_u8(image, "align_from_landmarks")
    lm = np.asarray(lm)
    if lm.shape != (68, 2):
        raise ValueError(f"align_from_landmarks: expected [68, 2] landmarks, got {lm.shape}")
    g = geometry(lm, (image.shape[1], image.shape[0]))
    img = image
    if g.rsize is not None:
        img = resample(img, *g.rsize)
    if g.crop is not None:
        x0, y0, x1, y1 = g.crop
        img = img[y0:y1, x0:x1]
    if g.pad is not None:
        img = pad_blend(img, g.pad, g.blur)
    img = quad_transform(img, (g.quad + 0.5).flatten(), TRANSFORM_SIZE, TRANSFORM_SIZE)
    return resample(img, OUTPUT_SIZE, OUTPUT_SIZE)


# ---- drop-in for utils.shape_predictor.align_face ---------------------------------------------------------------------
def _rgb_array(img) -> np.ndarray:
    from PIL import Image
    if not isinstance(img, Image.Image) or img.mode != "RGB":
        raise NotImplementedError("align_face: only 8-bit RGB images are supported, got "
                                  + (f"a PIL image of mode {img.mode}" if isinstance(img, Image.Image)
                                     else f"{type(img).__name__}"))
    return np.asarray(img)


def align_face(data, predictor=None, is_filepath=False, return_tensors=True):
    """Drop-in for utils/shape_predictor.py:80-194: same arguments, prints and return types (CPU float tensors
    T.ToTensor()(img).clamp(0, 1), or PIL RGB images).  The landmarks come from the reference module's own
    get_landmark / get_landmark_from_tensors; the warp runs on the current CUDA device."""
    import PIL.Image
    from torchvision import transforms as T
    import utils.shape_predictor as sp

    if predictor is None:                                 # :85-94
        predictor_path = 'pretrained_models/ShapeAdaptor/shape_predictor_68_face_landmarks.dat'
        if not os.path.isfile(predictor_path):
            print("Downloading Shape Predictor")
            data_io = sp.open_url("https://drive.google.com/uc?id=1huhv8PYpNNKbGCLOaYUjOgR1pY5pmbJx")
            with open(predictor_path, 'wb') as f:
                f.write(data_io.getbuffer())
        predictor = sp.dlib.shape_predictor(predictor_path)

    if is_filepath:
        lms = sp.get_landmark(data, predictor)
        images = [PIL.Image.open(data) for _ in lms]
    else:
        if not isinstance(data, list):
            data = [data]
        images, lms = sp.get_landmark_from_tensors(data, predictor)

    if not torch.cuda.is_available():
        raise RuntimeError("align_face: hairfastgan_b200's face alignment runs on a CUDA device (no CPU fallback)")
    device = torch.device("cuda", torch.cuda.current_device())
    imgs = []
    for img, lm in zip(images, lms):
        src = torch.from_numpy(np.ascontiguousarray(_rgb_array(img))).to(device)
        out = align_from_landmarks(src, lm).cpu().numpy()
        imgs.append(PIL.Image.fromarray(out))
    if return_tensors:
        transform = T.ToTensor()
        return [transform(img).clamp(0, 1) for img in imgs]
    return imgs
