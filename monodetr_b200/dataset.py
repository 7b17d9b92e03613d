"""Drop-in for the reference's lib/helpers/dataloader_helper.py `build_dataloader` and the parts of
lib/datasets/kitti/kitti_dataset.py `KITTI_Dataset` a caller sees, over device-resident image and label banks.

  ImageBank(root_dir, split, device)     every PNG of a split decoded ONCE on a host thread pool (the bytes of
                                         np.array(Image.open(f))) and packed into one device uint8 buffer; views(indices) gives
                                         (H, W, 3) CUDA views that ImageBatchPreprocessor / KittiBatchBuilder read in place
  KITTI_Dataset(split, cfg)              host-only and picklable: __getitem__(item) -> (bank index, AugRecord), the draws of
                                         kitti_dataset.py:130-154 on the global numpy.random (none on val / test)
  build_dataloader(cfg, workers=4)       (train_loader, test_loader): a real torch DataLoader over each light dataset with the
                                         reference's arguments, wrapped so that each batch comes out as the reference's
                                         (inputs, calibs, targets, info), built on the device in the main process

Because the loaders are torch DataLoaders with the reference's batch size, shuffle, worker-init rule and drop_last, they consume
the global torch RNG as the reference's do and hand batch i to worker i mod workers: with the same seeds the same images arrive in
the same batches with the same draws, for any number of workers.  Loader workers only make numpy draws; they never touch CUDA.
"""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset

from .labels import CLASS_NAMES, CLS_MEAN_SIZE, AugmentationSampler, KittiBatchBuilder, LabelBank, parse_calib_file
from .preprocess import ImageBatchPreprocessor

RESOLUTION = (1280, 384)          # kitti_dataset.py:32, W * H
DOWNSAMPLE = 32                   # kitti_dataset.py:82
SPLITS = ("train", "val", "trainval", "test")
UNSUPPORTED = ("aug_calib", "class_merging", "use_dontcare")


def _split_paths(root_dir, split):
    """kitti_dataset.py:48-56: (ids as the file's strings, data dir)."""
    if split not in SPLITS:
        raise ValueError(f"KITTI split must be one of {SPLITS}, got {split!r}")
    with open(os.path.join(root_dir, "ImageSets", split + ".txt")) as f:
        idx_list = [x.strip() for x in f.readlines()]
    return idx_list, os.path.join(root_dir, "testing" if split == "test" else "training")


def _image_path(data_dir, img_id):
    return os.path.join(data_dir, "image_2", "%06d.png" % int(img_id))


def read_image_sizes(paths):
    """(n, 2) int64 [W, H] of the PNGs from their headers; ValueError naming the first file that is not 8-bit RGB."""
    from PIL import Image
    sizes = np.zeros((len(paths), 2), np.int64)
    for i, p in enumerate(paths):
        with Image.open(p) as im:
            if im.mode != "RGB":
                raise ValueError(f"{p}: mode {im.mode!r}; only 8-bit RGB images are supported")
            sizes[i] = im.size
    return sizes


def _decode(path):
    from PIL import Image
    with Image.open(path) as im:
        return np.array(im)


class ImageBank:
    """Every image of ImageSets/<split>.txt in one device uint8 buffer, rows packed (pitch 3 * W).  Host tables: `sizes` (n, 2)
    [W, H], `offsets` (n + 1) byte offsets, `img_ids`.  The headers are read and checked before the device buffer is allocated,
    so an image that is not 8-bit RGB raises ValueError without touching the device."""

    def __init__(self, root_dir, split, device="cuda", threads=8):
        idx_list, data_dir = _split_paths(root_dir, split)
        paths = [_image_path(data_dir, i) for i in idx_list]
        self.split = split
        self.img_ids = [int(i) for i in idx_list]
        self.sizes = read_image_sizes(paths)
        nbytes = self.sizes[:, 0] * self.sizes[:, 1] * 3
        self.offsets = np.concatenate([[0], np.cumsum(nbytes)]).astype(np.int64)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("ImageBank: a CUDA device is required")
        self.data = torch.empty(max(int(self.offsets[-1]), 1), dtype=torch.uint8, device=self.device)
        with ThreadPoolExecutor(max(1, int(threads))) as pool:      # PIL releases the GIL while it inflates
            for k, arr in enumerate(pool.map(_decode, paths)):
                W, H = (int(v) for v in self.sizes[k])
                if arr.shape != (H, W, 3) or arr.dtype != np.uint8:
                    raise ValueError(f"{paths[k]}: decoded to {arr.shape} {arr.dtype}, header said ({H}, {W}, 3) uint8")
                self.data[self.offsets[k]:self.offsets[k + 1]].copy_(torch.from_numpy(arr.reshape(-1)))
        torch.cuda.current_stream(self.device).synchronize()

    def __len__(self):
        return len(self.img_ids)

    def view(self, k):
        W, H = (int(v) for v in self.sizes[k])
        return self.data[self.offsets[k]:self.offsets[k + 1]].view(H, W, 3)

    def views(self, indices):
        """(H, W, 3) uint8 CUDA views of images `indices`, in that order (no copy)."""
        return [self.view(int(k)) for k in indices]


class KITTI_Dataset(Dataset):
    """kitti_dataset.py's attributes and `__len__`; `__getitem__(item)` returns (item, AugRecord) -- the image and label banks
    are indexed by the item's position in the split, and the record's size is the image's (`img_sizes`, [W, H] per item; read
    from the PNG headers when not given).  Holds no CUDA tensor."""

    def __init__(self, split, cfg, img_sizes=None):
        self.root_dir = cfg.get("root_dir")
        self.split = split
        self.num_classes = 3
        self.max_objs = 50
        self.class_name = list(CLASS_NAMES)
        self.cls2id = {c: i for i, c in enumerate(CLASS_NAMES)}
        self.resolution = np.array(RESOLUTION)
        self.writelist = cfg.get("writelist", ["Car"])
        self.meanshape = cfg.get("meanshape", False)
        self.idx_list, self.data_dir = _split_paths(self.root_dir, split)
        self.image_dir = os.path.join(self.data_dir, "image_2")
        self.calib_dir = os.path.join(self.data_dir, "calib")
        self.label_dir = os.path.join(self.data_dir, "label_2")
        self.data_augmentation = split in ("train", "trainval")
        self.cls_mean_size = CLS_MEAN_SIZE.copy() if self.meanshape else np.zeros_like(CLS_MEAN_SIZE, dtype=np.float32)
        self.downsample = DOWNSAMPLE
        if img_sizes is None:
            img_sizes = read_image_sizes([_image_path(self.data_dir, i) for i in self.idx_list])
        self.img_sizes = np.asarray(img_sizes, np.int64).reshape(len(self.idx_list), 2)
        self.cfg = dict(cfg)
        self._augmentation = None

    @property
    def augmentation(self):
        if self._augmentation is None:                  # built lazily: it holds the numpy.random module, which does not pickle
            self._augmentation = AugmentationSampler.from_config(self.cfg, self.split, RESOLUTION)
        return self._augmentation

    def __getstate__(self):
        return dict(self.__dict__, _augmentation=None)

    def __len__(self):
        return len(self.idx_list)

    def __getitem__(self, item):
        return item, self.augmentation.sample(self.img_sizes[item])


def my_worker_init_fn(worker_id):
    """dataloader_helper.py:8-9"""
    np.random.seed(np.random.get_state()[1][0] + worker_id)


def _keep_lists(batch):
    return batch


def kitti_loader(dataset, batch_size, shuffle, workers):
    """The reference's DataLoader (dataloader_helper.py:21-33) over the light dataset; batches stay lists of (item, AugRecord)."""
    return DataLoader(dataset=dataset, batch_size=batch_size, num_workers=workers, worker_init_fn=my_worker_init_fn,
                      shuffle=shuffle, pin_memory=False, drop_last=False, collate_fn=_keep_lists)


class _TestBatchBuilder:
    """The test split's batch (kitti_dataset.py:169-171): the pre-processed images, P2 from the calib files, the images again
    as `targets`, and `info`."""

    def __init__(self, dataset, device="cuda"):
        self.resolution = RESOLUTION
        self.device = torch.device(device)
        self.img_ids = [int(i) for i in dataset.idx_list]
        self.P2 = np.stack([parse_calib_file(os.path.join(dataset.calib_dir, "%06d.txt" % i)) for i in self.img_ids])
        self.preprocessor = ImageBatchPreprocessor(self.resolution, device=device)

    def __call__(self, images, bank_indices, records):
        idx = np.asarray(bank_indices, np.int64)
        inputs = self.preprocessor(images, np.stack([r.trans_inv for r in records]))
        P2 = torch.from_numpy(self.P2[idx]).to(self.device)
        sizes = np.array([r.img_size for r in records], np.int64)
        feat = np.array(self.resolution, np.int64) // DOWNSAMPLE
        info = {"img_id": torch.tensor([self.img_ids[k] for k in idx], dtype=torch.int64), "img_size": torch.from_numpy(sizes),
                "bbox_downsample_ratio": torch.from_numpy(sizes / feat)}
        return inputs, P2, inputs, info


class DeviceLoader:
    """A DataLoader over a KITTI_Dataset whose collated (item, AugRecord) lists become the reference's batches: `inputs`,
    `calibs` and `targets` on the device (built on the current stream), `info` on the host.  len() and every DataLoader
    attribute (`dataset`, `batch_size`, ...) are the wrapped loader's."""

    def __init__(self, loader, bank, builder):
        self.loader, self.bank, self.builder = loader, bank, builder

    def __len__(self):
        return len(self.loader)

    def __getattr__(self, name):
        if name == "loader":
            raise AttributeError(name)
        return getattr(self.loader, name)

    def __iter__(self):
        return self.shard(0, 1)

    def shard(self, rank, world):
        """Batches b with b % world == rank, in order.  Every batch of the wrapped DataLoader is still drawn, so that the
        loader's composition and order are those of the whole pass, but only this rank's batches are built on the device."""
        for b, batch in enumerate(self.loader):
            if b % world != rank:
                continue
            idx = [int(k) for k, _ in batch]
            yield self.builder(self.bank.views(idx), idx, [r for _, r in batch])


def shard_batches(loader, rank, world):
    """Batches b with b % world == rank of `loader`, in its order: a DeviceLoader builds only those; any other iterable is run
    whole and the other ranks' batches are dropped."""
    if isinstance(loader, DeviceLoader):
        return loader.shard(rank, world)
    return (batch for b, batch in enumerate(loader) if b % world == rank)


def check_config(cfg):
    """The errors build_dataloader raises before it reads any image."""
    if cfg["type"] != "KITTI":
        raise NotImplementedError("%s dataset is not supported" % cfg["type"])
    for opt in UNSUPPORTED:
        if cfg.get(opt, False):
            raise NotImplementedError(f"build_dataloader: {opt} is not implemented on the device path")
    for key in ("train_split", "test_split"):
        if cfg[key] not in SPLITS:
            raise ValueError(f"build_dataloader: {key} must be one of {SPLITS}, got {cfg[key]!r}")


def _device_loader(cfg, split, shuffle, workers, device, threads):
    bank = ImageBank(cfg["root_dir"], split, device, threads)
    dataset = KITTI_Dataset(split, cfg, img_sizes=bank.sizes)
    if split == "test":
        builder = _TestBatchBuilder(dataset, device)
    else:
        builder = KittiBatchBuilder(cfg, split, LabelBank.from_kitti(cfg["root_dir"], split, device), RESOLUTION, device)
    return DeviceLoader(kitti_loader(dataset, cfg["batch_size"], shuffle, workers), bank, builder)


def build_dataloader(cfg, workers=4, device="cuda", threads=8):
    """dataloader_helper.py:12-35: (train_loader, test_loader) over cfg['train_split'] / cfg['test_split'].  Each split's
    images are decoded once here (`threads` host threads) into a device ImageBank; its labels and calibs go into a LabelBank."""
    check_config(cfg)
    train_loader = _device_loader(cfg, cfg["train_split"], True, workers, device, threads)
    test_loader = _device_loader(cfg, cfg["test_split"], False, workers, device, threads)
    return train_loader, test_loader
