"""Generates tests/golden/imagenet_augment.pt by running the UNMODIFIED reference ImageNet train chain (/root/reference, through
oracle/ref_shim.py): RandomResizedCropAndInterpolation(224, 'random'), RandomHorizontalFlip, RandAugmentTransform('rand-m7-mstd0.5',
224, img_mean), ToTensor, Normalize on the seeded StubImageDataset of tests/imagenet_augment_cases.py (as PIL RGB images, the way
ImageFolder's loader returns them), batched by CollateMixup in batch mode, for every case of GOLDEN_CASES under random.seed /
np.random.seed / torch.manual_seed.  Per sample it records what the reference drew (the crop window, the interpolation, the flip and
the RandAugment ops it applied with their arguments, logged by wrappers that call the original functions) and the sha256 of the
uint8 image ToTensor receives; per batch the sha256 of the float32 batch rounded to bf16, image by image, the sha256 of the float32
targets and the sha256 of the python / numpy / torch RNG states after the batch.  Run once in the build container:

    python tests/golden/make_imagenet_augment_goldens.py
"""
import hashlib
import os
import pickle
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from imagenet_augment_cases import CONFIG, GOLDEN_BATCH, GOLDEN_CASES, GOLDEN_MIX, IMG_MEAN, IMG_STD, SIZE, StubImageDataset  # noqa: E402
from oracle import ref_shim  # noqa: E402


def sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def rng_states():
    return {"python": sha(pickle.dumps(random.getstate())), "numpy": sha(pickle.dumps(np.random.get_state())), "torch": sha(torch.get_rng_state().numpy().tobytes())}


def main():
    ref_shim.install()
    import PIL
    import torchvision.transforms as TT
    import torchvision.transforms.functional as TF
    from PIL import Image
    from super_gradients.training.datasets import auto_augment
    from super_gradients.training.datasets.datasets_utils import RandomResizedCropAndInterpolation
    from super_gradients.training.datasets.mixup import CollateMixup

    log = {}
    resized_crop, hflip = TF.resized_crop, TF.hflip

    def rec_resized_crop(img, i, j, h, w, size, interpolation, *a, **kw):
        log["crop"], log["interpolation"] = (i, j, h, w), str(interpolation).split(".")[-1].lower()
        return resized_crop(img, i, j, h, w, size, interpolation, *a, **kw)

    def rec_hflip(img):
        log["flip"] = True
        return hflip(img)

    TF.resized_crop, TF.hflip = rec_resized_crop, rec_hflip
    crop = RandomResizedCropAndInterpolation(size=SIZE, interpolation="random")
    ra = auto_augment.rand_augment_transform(CONFIG, crop_size=SIZE, img_mean=IMG_MEAN)
    for k, op in enumerate(ra.ops):
        def wrap(fn, name):
            def rec(img, *args, **kw):
                log["ops"].append((name, tuple(float(x) for x in args)))
                return fn(img, *args, **kw)
            return rec
        op.aug_fn = wrap(op.aug_fn, auto_augment._RAND_TRANSFORMS[k])
    flip, to_tensor, normalize = TT.RandomHorizontalFlip(), TT.ToTensor(), TT.Normalize(mean=IMG_MEAN, std=IMG_STD)

    out = {"pillow": PIL.__version__, "torch": torch.__version__, "numpy": np.__version__, "cases": {}}
    stub = StubImageDataset(length=GOLDEN_BATCH)
    for case in GOLDEN_CASES:
        name, seed = case
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        samples, batch = [], []
        for i in range(len(stub)):
            arr, label = stub[i]
            log.clear()
            log.update(flip=False, ops=[])
            img = ra(flip(crop(Image.fromarray(arr))))
            u8 = np.asarray(img)
            samples.append(dict(crop=log["crop"], interpolation=log["interpolation"], flip=log["flip"], ops=list(log["ops"]), u8_sha256=sha(u8.tobytes())))
            batch.append((normalize(to_tensor(img)), label))
        x, target = CollateMixup(**GOLDEN_MIX[name])(batch)
        assert x.dtype == torch.float32 and x.shape == (GOLDEN_BATCH, 3, SIZE, SIZE)
        bf = x.bfloat16().view(torch.int16).numpy()
        out["cases"][case] = dict(samples=samples, input_sha256=[sha(bf[i].tobytes()) for i in range(len(bf))], target_sha256=sha(target.numpy().tobytes()),
                                  labels=[b[1] for b in batch], rng=rng_states(), first_input=x[0, :, ::16, ::16].clone())  # fmt: skip
        print(case, "mixed" if not torch.equal(x[0], batch[0][0]) else "unmixed", flush=True)
    TF.resized_crop, TF.hflip = resized_crop, hflip
    torch.save(out, os.path.join(HERE, "imagenet_augment.pt"))


if __name__ == "__main__":
    main()
