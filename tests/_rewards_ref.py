"""TEST INFRASTRUCTURE: the reference's image-symmetry and consistency rewards restated in NumPy + PIL (jannerm/ddpo
``ddpo/training/callbacks.py``; line numbers cite that file).  Model calls are replaced by a ``features`` function
(pixel values fp32 NHWC -> image features) so that a test can feed the features of any tower; the CLIPProcessor is
``clip_vision.preprocess``."""
import numpy as np
from PIL import Image, ImageOps

from ddpo_b200 import clip_vision as CV


def _pils(images):
    images = np.asarray(images)
    if images.dtype != np.uint8:
        images = (images * 255).astype(np.uint8)                 # :181 and its copies
    return [Image.fromarray(image) for image in images]


def _stack(pils):
    return np.array([np.array(img) for img in pils])


def mirror(images):                                             # :244-260
    pils = _pils(images)
    mirrored = _stack([ImageOps.mirror(img) for img in pils])
    pils = _stack(pils)
    return -((pils - mirrored) ** 2).mean(axis=(1, 2, 3))


def rotational_corr(images):                                    # :216-241
    pils = _pils(images)
    rotated = []
    for rot in (0, 180):
        rotated += [pil.rotate(rot) for pil in pils]
    output = _stack(rotated).reshape(2, len(pils), *np.asarray(rotated[0]).shape)
    scores = 0
    scores += ((output[0] - output[1]) ** 2).mean(axis=(1, 2, 3))
    scores /= 1
    return -scores


def _cov(X, Y):
    return ((X - X.mean(-1, keepdims=True)) * (Y - Y.mean(-1, keepdims=True))).sum(-1)


def mirror_corr(images, dtype=np.float32):                      # :268-292 (dtype float64: the exact value)
    pils = _pils(images)
    mirrored = _stack([ImageOps.mirror(img) for img in pils])
    pils = _stack(pils)
    n = len(pils)
    pils = (pils / 255.0).astype(dtype).reshape(n, -1)
    mirrored = (mirrored / 255.0).astype(dtype).reshape(n, -1)
    return -(_cov(pils, mirrored) / np.sqrt(_cov(pils, pils) * _cov(mirrored, mirrored)))


def angle_score(output, n):                                     # :196-211, :327-342
    output = output.reshape(-1, n, output.shape[-1])
    scores = 0
    for i in range(1, len(output)):
        numer = (output[0] * output[i]).sum(axis=-1)
        denom = np.linalg.norm(output[0], axis=-1) * np.linalg.norm(output[i], axis=-1)
        theta = np.arccos(np.clip(numer / denom, a_min=0, a_max=1))
        scores += theta * 180 / np.pi
    scores /= len(output) - 1
    return -scores


def rotational_pixels(images, size):                            # :181-188 + the processor
    pils = _pils(images)
    rotated = []
    for rot in (0, 90, 180, 270):
        rotated += [pil.rotate(rot) for pil in pils]
    return CV.preprocess(_stack(rotated), size)


def thumbnail_pixels(images, size):                             # :310-318 + the processor
    pils = _pils(images)
    downsampled = list(pils)
    for d in (4, 8, 16):
        s = (pils[0].size[0] // d, pils[0].size[1] // d)
        downsampled += [pil.resize(s) for pil in pils]
    return [CV.preprocess(np.array(img)[None], size)[0] for img in downsampled]


def rotational(images, features, size):
    return angle_score(np.asarray(features(rotational_pixels(images, size)), np.float32), len(images))


def thumbnail(images, features, size):
    return angle_score(np.asarray(features(np.stack(thumbnail_pixels(images, size))), np.float32), len(images))


def consistency(image_embeds, text_embeds, logit_scale):        # :122-140: FlaxCLIPModel's logits_per_image diagonal
    image_embeds = image_embeds / np.linalg.norm(image_embeds, axis=-1, keepdims=True)
    text_embeds = text_embeds / np.linalg.norm(text_embeds, axis=-1, keepdims=True)
    logits_per_image = np.exp(logit_scale) * image_embeds @ text_embeds.T
    return logits_per_image.diagonal()[:, None]
