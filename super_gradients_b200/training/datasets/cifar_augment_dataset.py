"""Loading for the GPU CIFAR-10 augmentation (the cifar10_resnet recipe, recipes/dataset_params/cifar10_dataset_params.yaml).

Two ways to feed `Trainer`, both producing `PackedCifarBatch`es whose `to_model_input(device, out=None)` makes the bf16 NHWC model
input [B, 16, 32, 32] with one launch of kernels.cifar_augment (zero-padded RandomCrop(32, padding=4) -> RandomHorizontalFlip ->
ToTensor -> Normalize, bit-exact with torchvision's chain rounded to bf16):

- `Cifar10AugmentDataset` + `Cifar10AugmentCollateFN` in a DataLoader: the workers make the draws torchvision's chain makes, from
  the same torch RNG calls in the same order, and pack the batch's uint8 images, draws and labels into ONE buffer (one copy per
  batch).  `Cifar10ValidationDataset` + `Cifar10ValidationCollateFN` do the same for the validation chain (Resize(32) is the
  identity on 32 x 32 images: top = left = 4, no flip).
- `Cifar10DeviceLoader`: the whole data set (50 000 x 3 KB = 154 MB) resident on the device, no worker processes; per batch only
  the small table of (source index, top, left, flip) and the labels are copied."""
from typing import Optional, Sequence, Tuple

import numpy as np
import torch
from torch.utils.data import BatchSampler, DistributedSampler, RandomSampler, SequentialSampler

from ... import kernels as K
from ...common.registry import register_collate_function

CIFAR10_MEAN = (0.4914, 0.4822, 0.4465)
CIFAR10_STD = (0.2023, 0.1994, 0.2010)
SIZE, PAD = 32, 4
VALIDATION_DRAW = (PAD, PAD, 0)  # the crop of the unpadded image, not flipped


def as_cifar_array(image) -> np.ndarray:
    """A PIL RGB or uint8 32 x 32 x 3 image as a uint8 array; any other size is refused (the GPU path does not resample)."""
    if isinstance(image, np.ndarray):
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f"images must be uint8 H x W x 3 RGB arrays, got {image.dtype} {image.shape}")
        arr = image
    elif getattr(image, "mode", None) == "RGB":
        arr = np.asarray(image)
    else:
        raise ValueError(f"images must be PIL RGB images or uint8 H x W x 3 arrays, got {type(image).__name__} {getattr(image, 'mode', '')}")
    if arr.shape[:2] != (SIZE, SIZE):
        raise ValueError(f"the GPU CIFAR-10 path takes 32 x 32 images only, got {arr.shape[0]} x {arr.shape[1]}")
    return arr


def draw_crop_flip() -> Tuple[int, int, int]:
    """RandomCrop(32, padding=4).get_params on the 40 x 40 padded image, then RandomHorizontalFlip's draw: the same torch calls in
    the same order as torchvision 0.26 (transforms.py RandomCrop.get_params, RandomHorizontalFlip.forward) -> (top, left, flip)."""
    top = torch.randint(0, 2 * PAD + 1, size=(1,)).item()
    left = torch.randint(0, 2 * PAD + 1, size=(1,)).item()
    flip = bool(torch.rand(1) < 0.5)
    return int(top), int(left), int(flip)


class Cifar10AugmentDataset(torch.utils.data.Dataset):
    """The recipe's train chain over any dataset returning (PIL RGB or uint8 32 x 32 x 3 image, label): items are (image, label,
    (top, left, flip)), with the draws torchvision's RandomCrop(32, padding=4) and RandomHorizontalFlip make under the same seed."""

    def __init__(self, dataset, mean=CIFAR10_MEAN, std=CIFAR10_STD):
        self.dataset = dataset
        self.mean, self.std = tuple(float(m) for m in mean), tuple(float(s) for s in std)

    def __len__(self) -> int:
        return len(self.dataset)

    def __getitem__(self, index: int):
        image, label = self.dataset[index]
        image = as_cifar_array(image)
        return image, int(label), draw_crop_flip()


class Cifar10ValidationDataset(Cifar10AugmentDataset):
    """The recipe's validation chain Resize(32) -> ToTensor -> Normalize: Resize(32) leaves a 32 x 32 image as it is, so items
    carry the fixed draw of the unpadded crop; other sizes are refused."""

    def __getitem__(self, index: int):
        image, label = self.dataset[index]
        return as_cifar_array(image), int(label), VALIDATION_DRAW


def pack(table: np.ndarray, labels: np.ndarray, images: Optional[Sequence[np.ndarray]] = None, pin: bool = False) -> torch.Tensor:
    """ONE uint8 buffer: the int32 [B, CF_FIELDS] table, the int64 [B] labels, then (packed mode) the B uint8 images."""
    B = len(table)
    n_img = 0 if images is None else B * K.CF_IMAGE_BYTES
    buf = torch.empty(B * (K.CF_FIELDS * 4 + 8) + n_img, dtype=torch.uint8, pin_memory=pin)
    raw = buf.numpy()
    head = B * K.CF_FIELDS * 4
    raw[:head].view(np.int32)[:] = np.asarray(table, np.int32).reshape(-1)
    raw[head : head + 8 * B].view(np.int64)[:] = labels
    if images is not None:
        raw[head + 8 * B :].reshape(B, SIZE, SIZE, 3)[:] = images
    return buf


class PackedCifarBatch:
    """A batch for the CIFAR-10 kernel: `buffer` (see pack()) and `images`, the device-resident data set the table indexes, or
    None when the images follow in the buffer."""

    def __init__(self, buffer: torch.Tensor, batch: int, mean, std, images: Optional[torch.Tensor] = None):
        self.buffer, self.batch, self.mean, self.std, self.images = buffer, batch, mean, std, images

    def pin_memory(self) -> "PackedCifarBatch":
        """Called by DataLoader(pin_memory=True) in the main process, so the copy to the device is asynchronous."""
        return PackedCifarBatch(self.buffer.pin_memory(), self.batch, self.mean, self.std, self.images)

    @property
    def table(self) -> torch.Tensor:
        """The host int32 [B, CF_FIELDS] table (source index, top, left, flip)."""
        return self.buffer[: self.batch * K.CF_FIELDS * 4].view(torch.int32).view(self.batch, K.CF_FIELDS)

    @property
    def labels(self) -> torch.Tensor:
        head = self.batch * K.CF_FIELDS * 4
        return self.buffer[head : head + 8 * self.batch].view(torch.int64)

    @property
    def input_shape(self) -> Tuple[int, int, int, int]:
        """Shape of the model input to_model_input makes."""
        return (self.batch, 16, SIZE, SIZE)

    def to_model_input(self, device, out=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(images bf16 NHWC [B, 16, 32, 32], int64 labels [B]) on `device`: one copy and one augmentation launch, no host
        synchronisation.  out: a bf16 channels_last tensor of input_shape the images are written into instead of a new one."""
        head = self.batch * K.CF_FIELDS * 4
        dev = self.buffer.to(device, non_blocking=True)
        out = K.empty_nhwc(*self.input_shape, device) if out is None else K.require_nhwc_out(out, self.input_shape)
        src = dev[head + 8 * self.batch :] if self.images is None else self.images
        K.cifar_augment(self.table, dev[:head].view(torch.int32).view(self.batch, K.CF_FIELDS), src, out, self.mean, self.std)
        return out, dev[head : head + 8 * self.batch].view(torch.int64)


@register_collate_function()
class Cifar10AugmentCollateFN:
    """Collates Cifar10AugmentDataset / Cifar10ValidationDataset items into a PackedCifarBatch (labels as default_collate's
    int64); touches no CUDA state, so it runs in DataLoader workers."""

    def __init__(self, mean=CIFAR10_MEAN, std=CIFAR10_STD):
        self.mean, self.std = tuple(float(m) for m in mean), tuple(float(s) for s in std)

    @classmethod
    def for_dataset(cls, dataset: Cifar10AugmentDataset) -> "Cifar10AugmentCollateFN":
        return cls(dataset.mean, dataset.std)

    def __call__(self, data) -> PackedCifarBatch:
        B = len(data)
        table = np.array([(b, *d[2]) for b, d in enumerate(data)], np.int32).reshape(B, K.CF_FIELDS)
        labels = np.array([d[1] for d in data], np.int64)
        return PackedCifarBatch(pack(table, labels, [as_cifar_array(d[0]) for d in data]), B, self.mean, self.std)


@register_collate_function()
class Cifar10ValidationCollateFN(Cifar10AugmentCollateFN):
    """Collates Cifar10ValidationDataset items (the validation chain) into a PackedCifarBatch."""


class Cifar10DeviceLoader:
    """The CIFAR-10 train (or validation) loader with the data set resident on the device: no worker processes and no pixel copies
    per step.  images: uint8 [N, 32, 32, 3] (array or tensor), labels: [N].  Yields PackedCifarBatch objects, so Trainer (and its
    CUDA-graph input path) consumes them as it consumes the packed DataLoader's.

    Sample order: each __iter__ takes the next epoch of the sampler the reference's DataLoader would use -- RandomSampler over a
    torch.Generator seeded with `seed` for one process (SequentialSampler without shuffle), DistributedSampler(seed=seed, rank,
    world_size) under DDP, whose set_epoch(epoch) Trainer calls through `loader.sampler` -- batched as DataLoader batches them
    (BatchSampler with drop_last).

    Draws: the crop corner and flip of every sample come from ONE host stream per rank (a torch.Generator seeded from (seed, rank)),
    drawn in the main process, not from the per-worker torch streams a DataLoader's workers use.  They are distributed as the
    reference's (top, left uniform in [0, 8], flip with probability 1/2) but are not the reference's numbers.  augment=False gives
    the validation chain (top = left = 4, no flip)."""

    def __init__(self, images, labels, batch_size: int, shuffle: bool = True, drop_last: bool = False, seed: int = 0, rank: int = 0, world_size: int = 1,
                 augment: bool = True, mean=CIFAR10_MEAN, std=CIFAR10_STD, device="cuda"):  # fmt: skip
        images = torch.as_tensor(images)
        if images.dtype != torch.uint8 or images.dim() != 4 or tuple(images.shape[1:]) != (SIZE, SIZE, 3):
            raise ValueError(f"images must be uint8 [N, 32, 32, 3], got {images.dtype} {tuple(images.shape)}")
        self.labels = torch.as_tensor(labels).to(torch.int64).cpu()
        if self.labels.shape != (images.shape[0],):
            raise ValueError("labels must be one per image")
        self.device = torch.device(device)
        self.images = images.to(self.device).contiguous()
        n = images.shape[0]
        if world_size > 1:
            self.sampler = DistributedSampler(range(n), num_replicas=world_size, rank=rank, shuffle=shuffle, seed=seed)
        elif shuffle:
            self.sampler = RandomSampler(range(n), generator=torch.Generator().manual_seed(seed))
        else:
            self.sampler = SequentialSampler(range(n))
        self.batch_size, self.drop_last, self.augment = int(batch_size), bool(drop_last), bool(augment)
        self.batch_sampler = BatchSampler(self.sampler, self.batch_size, self.drop_last)
        self.draws = torch.Generator().manual_seed(int(np.random.SeedSequence([seed, rank]).generate_state(1)[0]))
        self.mean, self.std = tuple(float(m) for m in mean), tuple(float(s) for s in std)

    def __len__(self) -> int:
        return len(self.batch_sampler)

    def __iter__(self):
        pin = self.device.type == "cuda"
        for idx in self.batch_sampler:
            idx = torch.as_tensor(idx, dtype=torch.int64)
            B = len(idx)
            table = torch.empty(B, K.CF_FIELDS, dtype=torch.int32)
            table[:, 0] = idx
            if self.augment:
                table[:, 1:3] = torch.randint(0, 2 * PAD + 1, (B, 2), generator=self.draws, dtype=torch.int32)
                table[:, 3] = torch.rand(B, generator=self.draws) < 0.5
            else:
                table[:, 1:] = torch.tensor(VALIDATION_DRAW, dtype=torch.int32)
            yield PackedCifarBatch(pack(table.numpy(), self.labels[idx].numpy(), pin=pin), B, self.mean, self.std, images=self.images)
