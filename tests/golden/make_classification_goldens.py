"""Generates tests/golden/classification.pt by running the UNMODIFIED reference (/root/reference) on CPU through oracle/ref_shim.py:
its ImageNet processing chain (Resize -> CenterCrop -> StandardizeImage -> NormalizeImage -> ImagePermute, with PIL's resize) on
seeded images, its accuracy(output, target, topk=(1, 5)) and its classification pipeline decode (torch.max(softmax(logits), 1)) on
seeded logits.  Run once in the build container:

    python tests/golden/make_classification_goldens.py

The reference tree does not exist on the GPU box, so the output is committed.
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
# landscape, portrait, short side exactly 256 (no resize), short side 257 (scale just below 1), a large downscale, an upscale from 60 x 90,
# and two more ordinary photographs' sizes
IMAGENET_SHAPES = [(375, 500), (500, 375), (256, 340), (257, 300), (3000, 4000), (60, 90), (480, 640), (427, 640)]
SMALL_SHAPES = [(375, 500), (200, 160), (90, 60)]


def _sha(t_bf16):
    return hashlib.sha256(t_bf16.contiguous().view(torch.int16).numpy().tobytes()).hexdigest()


def golden_images():
    from super_gradients.training.processing import processing as P

    rng = np.random.RandomState(31)
    chains = {
        "imagenet": (lambda: [P.Resize(size=256), P.CenterCrop(size=224), P.StandardizeImage(), P.NormalizeImage(mean=MEAN, std=STD), P.ImagePermute()],
                     IMAGENET_SHAPES, dict(resize=256, crop=224, reverse=False, mean=MEAN, std=STD)),
        "small_reversed": (lambda: [P.ReverseImageChannels(), P.Resize(size=160), P.CenterCrop(size=128), P.StandardizeImage(max_value=255.0), P.ImagePermute()],
                           SMALL_SHAPES, dict(resize=160, crop=128, reverse=True, mean=None, std=None)),
    }  # fmt: skip
    out = {}
    for name, (mk, shapes, kw) in chains.items():
        cases = []
        for (h, w) in shapes:
            seed = int(rng.randint(0, 2**31 - 1))
            img = np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)
            steps = mk()
            resized = next(s for s in steps if type(s).__name__ == "Resize").preprocess_image(img[:, :, ::-1].copy() if kw["reverse"] else img)[0]
            pre, _ = P.ComposeProcessing(steps).preprocess_image(img)
            t = torch.from_numpy(np.ascontiguousarray(pre)).to(torch.bfloat16)  # what the model consumes (round to nearest)
            cases.append(dict(image_seed=seed, image_shape=(h, w), resized_shape=tuple(resized.shape[:2]), pre_shape=tuple(t.shape), pre_sha256=_sha(t),
                              pre_sample=t[:, ::13, ::17].clone()))  # fmt: skip
        out[name] = dict(kw=kw, cases=cases)
    return out


def golden_logits():
    from super_gradients.training.metrics.classification_metrics import accuracy
    from super_gradients.training.pipelines.pipelines import ClassificationPipeline

    g = torch.Generator().manual_seed(5)
    out = {}
    for name, (n, c) in {"imagenet": (96, 1000), "cifar": (64, 10), "five": (40, 5)}.items():
        logits = torch.randn(n, c, generator=g) * 3
        target = torch.randint(0, c, (n,), generator=g)
        hit = torch.rand(n, generator=g) < 0.4  # a share of rows whose target is the argmax or in the top five
        rank = torch.randint(0, 5, (n,), generator=g)
        target[hit] = logits.argsort(1, descending=True)[torch.arange(n), rank][hit]
        soft = torch.rand(n, c, generator=g) * 0.1
        soft[torch.arange(n), target] = 0.9  # smooth labels whose argmax is the target
        top1, top5 = accuracy(logits, target, topk=(1, 5))
        pred = ClassificationPipeline._decode_model_output(None, logits, np.zeros((n, 3, 8, 8), np.float32))
        out[name] = dict(logits=logits, target=target, soft=soft, top1_percent=float(top1), top5_percent=float(top5),
                         labels=torch.tensor([p.label for p in pred]), confidence=torch.tensor([p.confidence for p in pred], dtype=torch.float64))  # fmt: skip
    return out


def main():
    ref_shim.install()
    torch.save(dict(images=golden_images(), logits=golden_logits()), os.path.join(HERE, "classification.pt"))


if __name__ == "__main__":
    main()
