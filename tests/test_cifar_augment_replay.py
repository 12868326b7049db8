"""CPU replay of the CIFAR-10 loaders: Cifar10AugmentDataset draws, under the same seeds and in DataLoaders with 0 and 2 workers,
exactly what the reference's torchvision chain draws (and the host build of the kernel then reproduces its output bit for bit);
Cifar10DeviceLoader's per-epoch sample order is the RandomSampler's / DistributedSampler's a DataLoader would use; the packed
buffer round-trips."""
import numpy as np
import pytest
import torch
import torchvision.transforms as TT
from torch.utils.data import DataLoader, DistributedSampler, RandomSampler

from cifar_augment_cases import MEAN, STD, golden, host_augment, images
from super_gradients_b200.common.registry import COLLATE_FUNCTIONS
from super_gradients_b200.training.datasets.cifar_augment_dataset import (Cifar10AugmentCollateFN, Cifar10AugmentDataset, Cifar10DeviceLoader,
                                                                          Cifar10ValidationCollateFN, Cifar10ValidationDataset, PackedCifarBatch)  # fmt: skip

IMAGES = images(40, seed=5)


class _Plain(torch.utils.data.Dataset):
    def __init__(self, ims, transform=None):
        self.ims, self.transform = ims, transform

    def __len__(self):
        return len(self.ims)

    def __getitem__(self, i):
        from PIL import Image

        img = Image.fromarray(self.ims[i])
        return (self.transform(img) if self.transform else img), i % 10


def test_golden_draws_replay():
    g = golden()["train"]
    ds = Cifar10AugmentDataset(_Plain(g["images"].numpy()))
    torch.manual_seed(g["seed"])
    assert [ds[i][2] for i in range(len(ds))] == [tuple(d) for d in g["draws"].tolist()]


@pytest.mark.parametrize("workers", [0, 2])
def test_dataloader_draws_are_the_reference_chains(workers):
    """The same DataLoader (seeded generator, shuffled, workers) over the reference chain and over Cifar10AugmentDataset: every
    sample's output made from our draws is the reference's, bit for bit, so the draws are the same."""
    ref_chain = TT.Compose([TT.RandomCrop(32, padding=4), TT.RandomHorizontalFlip(), TT.ToTensor(), TT.Normalize(MEAN, STD)])
    kw = dict(batch_size=8, shuffle=True, num_workers=workers)
    torch.manual_seed(0)  # the draws of the main process (workers=0)
    ref = list(DataLoader(_Plain(IMAGES, ref_chain), generator=torch.Generator().manual_seed(11), **kw))
    ds = Cifar10AugmentDataset(_Plain(IMAGES))
    torch.manual_seed(0)
    ours = list(DataLoader(ds, generator=torch.Generator().manual_seed(11), collate_fn=Cifar10AugmentCollateFN.for_dataset(ds), **kw))
    assert len(ref) == len(ours) == 5
    for (x, y), b in zip(ref, ours):
        assert isinstance(b, PackedCifarBatch) and torch.equal(b.labels, y)
        f32, _ = host_augment(b.table.numpy(), b.buffer[b.batch * 24 :].numpy().reshape(b.batch, 32, 32, 3))
        assert np.array_equal(f32.view(np.int32), x.numpy().view(np.int32))


def test_collate_layout_round_trips():
    ds = Cifar10AugmentDataset(_Plain(IMAGES))
    items = [ds[i] for i in (3, 1, 4, 1, 5)]
    b = Cifar10AugmentCollateFN.for_dataset(ds)(items)
    assert b.input_shape == (5, 16, 32, 32) and b.buffer.dtype == torch.uint8 and b.buffer.numel() == 5 * (16 + 8 + 3072)
    assert b.table.tolist() == [[k, *it[2]] for k, it in enumerate(items)]
    assert b.labels.tolist() == [it[1] for it in items]
    assert np.array_equal(b.buffer[5 * 24 :].numpy().reshape(5, 32, 32, 3), np.stack([it[0] for it in items]))
    assert (b.mean, b.std) == (tuple(MEAN), tuple(STD))


def test_validation_items_and_refusals():
    ds = Cifar10ValidationDataset(_Plain(IMAGES))
    b = Cifar10ValidationCollateFN.for_dataset(ds)([ds[0], ds[7]])
    assert b.table.tolist() == [[0, 4, 4, 0], [1, 4, 4, 0]]
    assert {"Cifar10AugmentCollateFN", "Cifar10ValidationCollateFN"} <= set(COLLATE_FUNCTIONS)
    for bad in (np.zeros((36, 36, 3), np.uint8), np.zeros((32, 32), np.uint8), np.zeros((32, 32, 3), np.float32)):
        for cls in (Cifar10AugmentDataset, Cifar10ValidationDataset):
            with pytest.raises(ValueError):
                cls([(bad, 0)])[0]
    with pytest.raises(ValueError):
        Cifar10DeviceLoader(np.zeros((4, 28, 28, 3), np.uint8), np.zeros(4), 2, device="cpu")


def _reference_batches(n, batch_size, drop_last, seed, rank, world, epochs=3):
    if world == 1:
        sampler = RandomSampler(range(n), generator=torch.Generator().manual_seed(seed))
    else:
        sampler = DistributedSampler(range(n), num_replicas=world, rank=rank, shuffle=True, seed=seed)
    dl = DataLoader(range(n), batch_size=batch_size, sampler=sampler, drop_last=drop_last)
    out = []
    for e in range(epochs):
        if world > 1:
            sampler.set_epoch(e)
        out.append([b.tolist() for b in dl])
    return out


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("drop_last", [False, True])
def test_device_loader_order_is_the_samplers(world, drop_last):
    n, bs, seed = 203, 16, 7
    ims, labels = images(n, seed=9), (np.arange(n) * 7) % 10
    for rank in range(world):
        dl = Cifar10DeviceLoader(ims, labels, bs, shuffle=True, drop_last=drop_last, seed=seed, rank=rank, world_size=world, device="cpu")
        got = []
        for e in range(3):
            if hasattr(dl.sampler, "set_epoch"):  # as Trainer.train does
                dl.sampler.set_epoch(e)
            got.append([b.table[:, 0].tolist() for b in dl])
            assert len(got[-1]) == len(dl)
        assert got == _reference_batches(n, bs, drop_last, seed, rank, world)
        assert len({tuple(map(tuple, ep)) for ep in got}) == 3  # a new order every epoch
        b = next(iter(dl))
        assert b.images.data_ptr() == dl.images.data_ptr() and b.labels.tolist() == [int(labels[i]) for i in b.table[:, 0]]


def test_device_loader_draws():
    n = 4096
    dl = Cifar10DeviceLoader(np.zeros((n, 32, 32, 3), np.uint8), np.zeros(n), 512, seed=3, device="cpu")
    t = torch.cat([b.table for b in dl])
    assert sorted(t[:, 0].tolist()) == list(range(n))
    assert set(t[:, 1].tolist()) == set(t[:, 2].tolist()) == set(range(9)) and set(t[:, 3].tolist()) == {0, 1}
    assert abs(float(t[:, 3].float().mean()) - 0.5) < 0.05
    other_rank = Cifar10DeviceLoader(np.zeros((n, 32, 32, 3), np.uint8), np.zeros(n), 512, seed=3, rank=1, world_size=2, device="cpu")
    assert not torch.equal(next(iter(other_rank)).table[:, 1:], t[:256, 1:])
    val = Cifar10DeviceLoader(np.zeros((10, 32, 32, 3), np.uint8), np.zeros(10), 4, shuffle=False, augment=False, device="cpu")
    assert [b.table.tolist() for b in val][0] == [[k, 4, 4, 0] for k in range(4)]
