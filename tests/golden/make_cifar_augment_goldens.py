"""Generates tests/golden/cifar_augment.pt by running the UNMODIFIED reference CIFAR-10 chains (through oracle/ref_shim.py): the
train and validation `transforms` lists of recipes/dataset_params/cifar10_dataset_params.yaml, built by the reference's
TransformsFactory and composed as its Cifar10 dataset composes them, on seeded uint8 32 x 32 images given as PIL RGB images (as
torchvision's CIFAR10 returns them).

- train: the images of tests/cifar_augment_cases.images(TRAIN_N, seed=0), in order, under torch.manual_seed(TRAIN_SEED); per sample
  the (top, left) RandomCrop drew and whether RandomHorizontalFlip flipped (logged by wrappers that call the original functions),
  and the float32 [3, 32, 32] output.
- validation: all_values_images() (every channel takes every uint8 value) through the validation chain; it checks that Resize(32)
  returned the image unchanged.
Run once where the reference tree is available:

    python tests/golden/make_cifar_augment_goldens.py
"""
import os
import sys

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cifar_augment_cases import all_values_images, images  # noqa: E402
from oracle import ref_shim  # noqa: E402

TRAIN_N, TRAIN_SEED = 32, 0


def main():
    ref_shim.install()
    import PIL
    import torchvision
    import torchvision.transforms as TT
    import torchvision.transforms.functional as TF
    from PIL import Image
    from super_gradients.common.factories.transforms_factory import TransformsFactory

    params = yaml.safe_load(open(os.path.join(ref_shim.SG_DIR, "recipes", "dataset_params", "cifar10_dataset_params.yaml")))
    train_chain = TT.Compose(TransformsFactory().get(params["train_dataset_params"]["transforms"]))
    val_chain = TT.Compose(TransformsFactory().get(params["val_dataset_params"]["transforms"]))
    print(train_chain, val_chain, sep="\n")

    log = {}
    get_params, hflip, resize = TT.RandomCrop.get_params, TF.hflip, TF.resize

    def rec_get_params(img, output_size):
        out = get_params(img, output_size)
        log["crop"] = (out[0], out[1])
        return out

    def rec_hflip(img):
        log["flip"] = True
        return hflip(img)

    def rec_resize(img, *a, **kw):
        out = resize(img, *a, **kw)
        log["resize_identity"] = out.size == img.size and np.array_equal(np.asarray(out), np.asarray(img))
        return out

    TT.RandomCrop.get_params, TF.hflip, TF.resize = staticmethod(rec_get_params), rec_hflip, rec_resize
    try:
        train_images = images(TRAIN_N, seed=0)
        torch.manual_seed(TRAIN_SEED)
        draws, train_out = [], []
        for im in train_images:
            log.clear()
            log["flip"] = False
            train_out.append(train_chain(Image.fromarray(im)))
            draws.append((*log["crop"], int(log["flip"])))
        val_images = all_values_images()
        val_out = []
        for im in val_images:
            log.clear()
            val_out.append(val_chain(Image.fromarray(im)))
            assert log["resize_identity"], "Resize(32) changed a 32 x 32 image"
    finally:
        TT.RandomCrop.get_params, TF.hflip, TF.resize = staticmethod(get_params), hflip, resize
    out = dict(versions={"pillow": PIL.__version__, "torch": torch.__version__, "torchvision": torchvision.__version__, "numpy": np.__version__},
               train=dict(seed=TRAIN_SEED, images=torch.from_numpy(train_images), draws=torch.tensor(draws, dtype=torch.int32), output=torch.stack(train_out)),
               val=dict(images=torch.from_numpy(val_images), output=torch.stack(val_out)))  # fmt: skip
    assert out["train"]["output"].dtype == torch.float32 and out["val"]["output"].shape == (8, 3, 32, 32)
    torch.save(out, os.path.join(HERE, "cifar_augment.pt"))
    print("draws:", draws)


if __name__ == "__main__":
    main()
