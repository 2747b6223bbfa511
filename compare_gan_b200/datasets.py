"""Dataset surface (reference datasets.py:66-329, 374-648).  BASELINE measures on synthetic data (`sample_images`:
uniform [0,1) images, seed 547, datasets.py:136-145).  The input pipeline of `train_input_fn` / `eval_input_fn`
(datasets.py:261-329: repeat -> transform -> shuffle -> batch(drop_remainder) -> prefetch) runs in the native loader
(`csrc/loader.cu`, `cgan_loader_*`) over the reference's fake data set or over decoded uint8 sources on disk; TFDS
itself (download + decode) is not available offline.

Sources under `data_dir`, looked up in this order:

* `<name>_<split>_images.npy`, uint8 [N, H, W, C] at the data set's own image shape (`<name>` is the data set's name):
  loaded as is, converted to float32 / 255 on the host (`BatchIterator`).  No transform, for every data set.
* For the data sets with a transform (ImageNet, CelebA, LSUN; `_transform`), a source at any size under the data set's
  source prefix (`imagenet2012` for the whole ImageNet family, else the data set's name), in one of two forms:
  - `<prefix>_<split>_images.npy`: uint8 [N, H, W, C], any H and W;
  - `<prefix>_<split>_pixels.npy` uint8 1-D (the images concatenated, each HWC) with `<prefix>_<split>_index.npy`
    int64 [N, 3] rows of (byte offset, h, w), for images that differ in size.
  Both become one table of (offset, h, w) rows over a byte blob.  The host picks each element's crop window and packs
  its rows (`cgan_loader_create_transformed`); the device crops or pads, resizes and converts them
  (`cgan_crop_resize_u8`).  `TransformedBatchIterator` hands out float32 device batches.  ImageNet's eval split is
  `validation`, as in the reference.
* `_labels.npy` int32 [N], optional in every form (labels default to 0)."""
import ctypes
import os

import numpy as np

from . import _lib
from . import gin_lite as gin

# name -> (resolution, colors, num_classes, eval_test_samples)   (datasets.py:370-512, 620-640)
DATASETS = {
    "cifar10": (32, 3, 10, 10000),
    "celeb_a": (64, 3, None, 10000),
    "celeb_a_hq_128": (128, 3, None, 10000),      # named by sndcgan_celebahq128.gin:4 (SURVEY App. C note)
    "lsun-bedroom": (128, 3, None, 30000),
    "imagenet_64": (64, 3, 1000, 50000),           # datasets.py:500-532, 624-637
    "imagenet_128": (128, 3, 1000, 50000),
    "imagenet_256": (256, 3, 1000, 50000),
    "imagenet_512": (512, 3, 1000, 50000),
    "imagenet_512_hq400": (512, 3, 1000, 50000),
    "single_class_imagenet_128": (128, 3, 1, 50000),
    "random_class_imagenet_128": (128, 3, 1000, 50000),
    "labeled_only_imagenet_128": (128, 3, 1000, 50000),
    "mnist": (28, 1, 10, 10000),                   # datasets.py:332-343
    "fashion-mnist": (28, 1, 10, 10000),           # datasets.py:346-357
}
# keys whose data set goes by another name (ImageDatasetV2.name, which also names the shard files)
DATASET_NAMES = {"fashion-mnist": "fashion_mnist", "labeled_only_imagenet_128": "imagenet_128"}

# cgan_crop_desc / cgan_image_source / cgan_image_transform (include/cgan_b200.h)
CROP_DESC = np.dtype([("offset", "<i8"), ("position", "<i8"), ("element", "<i4"), ("h", "<i4"), ("w", "<i4"),
                      ("canvas_h", "<i4"), ("canvas_w", "<i4"), ("top", "<i4"), ("left", "<i4"), ("crop_y", "<i4"),
                      ("crop_x", "<i4"), ("reserved", "<i4")])
CROP_METHODS = {"none": 0, "middle": 1, "random": 2, "distorted": 3}
CROP_OR_PAD = 4
LABEL_SOURCE, LABEL_ZERO, LABEL_RANDOM = 0, 1, 2


class ImageSource(ctypes.Structure):
  _fields_ = [("pixels", ctypes.c_void_p), ("pixel_bytes", ctypes.c_int64), ("index", ctypes.c_void_p),
              ("labels", ctypes.c_void_p), ("n", ctypes.c_int64), ("c", ctypes.c_int32), ("reserved", ctypes.c_int32)]


class ImageTransform(ctypes.Structure):
  _fields_ = [(f, ctypes.c_int32) for f in ("crop", "canvas_h", "canvas_w", "min_side", "labeled_only", "label",
                                            "random_classes", "reserved")]


def crop_method_code(crop_method):
  if crop_method not in CROP_METHODS:
    raise ValueError("Unsupported crop method: {}".format(crop_method))
  return CROP_METHODS[crop_method]


@gin.configurable("train_imagenet_transform", whitelist=["crop_method"])
def train_imagenet_transform(crop_method="distorted"):
  """The crop of ImageNet training images (datasets.py:494-500): distorted, random, middle or none."""
  return crop_method_code(crop_method)


@gin.configurable("eval_imagenet_transform", whitelist=["crop_method"])
def eval_imagenet_transform(crop_method="middle"):
  """The crop of ImageNet evaluation images (datasets.py:503-509)."""
  return crop_method_code(crop_method)


class ImageDatasetV2(object):
  """Synthetic stand-in exposing name / image_shape / num_classes / eval_test_samples."""

  # where the source of a transformed split lives: (prefix, {split: source split}); None without a transform
  _source = None

  def __init__(self, name, resolution, colors, num_classes, eval_test_samples, seed=547, fake_dataset=True,
               data_dir=None, shuffle_buffer_size=10000, train_split="train", eval_split="test"):
    self._name, self._resolution, self._colors = name, resolution, colors
    self._num_classes, self._eval_test_samples, self._seed = num_classes, eval_test_samples, seed
    self._rng = np.random.RandomState(seed)
    # FLAGS.data_fake_dataset / tfds_data_dir / data_shuffle_buffer_size of the reference (datasets.py:44-64)
    self._fake_dataset, self._data_dir = fake_dataset, data_dir or os.environ.get("CGAN_DATA_DIR")
    self._shuffle_buffer_size, self._train_split, self._eval_split = shuffle_buffer_size, train_split, eval_split

  @property
  def name(self):
    return self._name

  @property
  def num_classes(self):
    return self._num_classes

  @property
  def eval_test_samples(self):
    return self._eval_test_samples

  @property
  def image_shape(self):
    return (self._resolution, self._resolution, self._colors)

  def sample_images(self, n):
    """float32 U[0,1) NHWC (datasets.py:136-145)."""
    return self._rng.rand(n, self._resolution, self._resolution, self._colors).astype(np.float32)

  def sample_labels(self, n):
    if not self._num_classes:
      return None
    return self._rng.randint(0, self._num_classes, size=n).astype(np.int32)

  # ---- input pipeline (datasets.py:136-145, 229-329) ----------------------------------------------------------
  def _make_fake_dataset(self, split):
    """100 uniform [0,1) float32 images with all-ones labels (datasets.py:136-145)."""
    rng = np.random.RandomState(self._seed)
    images = rng.uniform(size=[100] + list(self.image_shape)).astype(np.float32)
    return images, np.ones((100,), np.int32)

  def _load_dataset(self, split):
    """(images, labels) of a split: the fake data set, or memory-mapped uint8 NHWC shards from `data_dir`."""
    if self._fake_dataset:
      return self._make_fake_dataset(split)
    base = self._shard_base(self._name, split)
    images = np.load(base + "_images.npy", mmap_mode="r")
    if images.dtype != np.uint8 or images.shape[1:] != self.image_shape:
      raise ValueError("%s_images.npy must be uint8 [N,%d,%d,%d], got %s %s" % ((base,) + self.image_shape + (images.dtype, images.shape)))
    labels = np.load(base + "_labels.npy", mmap_mode="r").astype(np.int32) if os.path.exists(base + "_labels.npy") else None
    return images, labels

  def _shard_base(self, prefix, split):
    if not self._data_dir:
      raise ValueError("Dataset %s: no data_dir (dataset.data_dir or $CGAN_DATA_DIR) and fake_dataset is off; TFDS "
                       "downloads are not available here." % self._name)
    return os.path.join(self._data_dir, "%s_%s" % (prefix, split))

  def _transform(self, train):
    """The split's cgan_image_transform fields and divide_after, or None when the data set has no transform."""
    return None

  def _uses_transform(self, split):
    """True when `split` reads a source through the transform: the data set has one and no shard at its own image shape
    exists under its own name (that shard keeps the untransformed path)."""
    if self._fake_dataset or self._source is None:
      return False
    own = self._shard_base(self._name, split) + "_images.npy"
    if os.path.exists(own):
      shape = np.load(own, mmap_mode="r").shape
      if shape[1:] == self.image_shape:
        return False
    return True

  def _load_source(self, split):
    """(pixels uint8 1-D, index int64 [N, 3] of (offset, h, w), labels int32 [N] or None) of the split's source."""
    prefix, splits = self._source
    base = self._shard_base(prefix, splits.get(split, split))
    c = self._colors
    if os.path.exists(base + "_pixels.npy"):
      fp, fi = base + "_pixels.npy", base + "_index.npy"
      pixels = np.load(fp, mmap_mode="r")
      if pixels.dtype != np.uint8 or pixels.ndim != 1:
        raise ValueError("%s must be uint8 1-D, got %s %s" % (fp, pixels.dtype, pixels.shape))
      if not os.path.exists(fi):
        raise ValueError("%s has no index file %s" % (fp, fi))
      index = np.load(fi)
      if index.dtype != np.int64 or index.ndim != 2 or index.shape[1] != 3 or len(index) < 1:
        raise ValueError("%s must be int64 [N>=1, 3] rows of (offset, h, w), got %s %s" % (fi, index.dtype, index.shape))
      off, h, w = index[:, 0], index[:, 1], index[:, 2]
      bad = (off < 0) | (h < 1) | (w < 1) | (h > 1 << 30) | (w > 1 << 30)
      bad |= ~bad & (off + h * w * c > pixels.shape[0])
      if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise ValueError("%s: row %d (offset %d, h %d, w %d) is not a %d-channel image inside the %d bytes of %s" % (
            fi, i, off[i], h[i], w[i], c, pixels.shape[0], fp))
      n = len(index)
    elif os.path.exists(base + "_images.npy"):
      fp = base + "_images.npy"
      images = np.load(fp, mmap_mode="r")
      if images.dtype != np.uint8 or images.ndim != 4 or images.shape[3] != c or min(images.shape) < 1:
        raise ValueError("%s must be uint8 [N,H,W,%d], got %s %s" % (fp, c, images.dtype, images.shape))
      n, h, w, _ = images.shape
      pixels = images.reshape(-1)
      index = np.stack([np.arange(n, dtype=np.int64) * (h * w * c), np.full(n, h, np.int64), np.full(n, w, np.int64)], 1)
    else:
      raise ValueError("Dataset %s: no source for split %s: neither %s_images.npy at %s nor %s_{images,pixels}.npy" % (
          self._name, split, self._shard_base(self._name, split), self.image_shape, base))
    labels = None
    if os.path.exists(base + "_labels.npy"):
      labels = np.ascontiguousarray(np.load(base + "_labels.npy"), dtype=np.int32)
      if labels.shape != (n,):
        raise ValueError("%s_labels.npy must be [%d], got %s" % (base, n, labels.shape))
    return pixels, np.ascontiguousarray(index), labels

  def _transformed_iterator(self, split, train, batch_size, shuffle_buffer, seed, ring, limit_samples=None):
    pixels, index, labels = self._load_source(split)
    transform, divide_after = self._transform(train)
    return TransformedBatchIterator(pixels, index, labels, self._colors, transform, self._resolution, divide_after,
                                    batch_size, shuffle_buffer, seed, ring, limit_samples=limit_samples)

  def _get_per_host_random_seed(self, rank=0):
    """The data seed (datasets.py:147-170); one stream per data-parallel rank, as per TPU host in the reference."""
    return self._seed + rank

  def train_input_fn(self, params=None, preprocess_fn=None, rank=0, ring=8):
    """Infinite iterator of (images float32 [B,H,W,C] in [0,1], labels int32 [B]) batches: repeat -> shuffle(
    shuffle_buffer_size, seed) -> batch(drop_remainder) -> prefetch (datasets.py:261-291).  `preprocess_fn(images,
    labels)`, if given, is applied per batch on the host."""
    params = params or {}
    if "batch_size" not in params:
      raise ValueError("train_input_fn needs params['batch_size'].")
    if self._uses_transform(self._train_split):
      if preprocess_fn is not None:
        raise ValueError("preprocess_fn is not supported on transformed sources (their batches live on the device)")
      return self._transformed_iterator(self._train_split, True, params["batch_size"], self._shuffle_buffer_size,
                                        self._get_per_host_random_seed(rank), ring)
    images, labels = self._load_dataset(self._train_split)
    return BatchIterator(images, labels, params["batch_size"], self._shuffle_buffer_size,
                         self._get_per_host_random_seed(rank), ring, preprocess_fn=preprocess_fn)

  def eval_input_fn(self, params=None, split=None, ring=4):
    """Finite, unshuffled iterator over the first eval_test_samples of the eval split (datasets.py:293-318)."""
    params = params or {}
    if "batch_size" not in params:
      raise ValueError("eval_input_fn needs params['batch_size'].")
    if self._uses_transform(split or self._eval_split):
      return self._transformed_iterator(split or self._eval_split, False, params["batch_size"], 0, self._seed, ring,
                                        limit_samples=self._eval_test_samples)
    images, labels = self._load_dataset(split or self._eval_split)
    n = min(self._eval_test_samples, len(images)) if not self._fake_dataset else self._eval_test_samples
    return BatchIterator(images, labels, params["batch_size"], 0, self._seed, ring, limit=n // params["batch_size"])


class BatchIterator(object):
  """Python face of the native loader (`cgan_loader_*`, include/cgan_b200.h).  Each `next()` returns numpy views of one
  page-locked ring slot; call `release(count)` once the host->device copies of the `count` oldest batches are done."""

  def __init__(self, images, labels, batch, shuffle_buffer, seed, ring, limit=None, preprocess_fn=None):
    _, _, self._fn = _lib.load_functions()
    self._images = images if images.flags["C_CONTIGUOUS"] else np.ascontiguousarray(images)      # keeps the source alive
    self._labels = None if labels is None else np.ascontiguousarray(labels, dtype=np.int32)
    if self._images.dtype not in (np.uint8, np.float32):
      raise ValueError("loader sources are uint8 or float32, got %s" % self._images.dtype)
    n, h, w, c = self._images.shape
    self._shape, self._batch, self._limit, self._count = (batch, h, w, c), batch, limit, 0
    self._preprocess = preprocess_fn
    self._h = ctypes.c_void_p()
    rc = self._fn["cgan_loader_create"](
        ctypes.byref(self._h), self._images.ctypes.data_as(ctypes.c_void_p), 0 if self._images.dtype == np.uint8 else 1,
        None if self._labels is None else self._labels.ctypes.data_as(ctypes.c_void_p), n, h, w, c, batch,
        int(shuffle_buffer), int(seed), int(ring))
    if rc != 0:
      raise _lib.CganError("cgan_loader_create failed (%d)" % rc)

  def __iter__(self):
    return self

  def __next__(self):
    if self._limit is not None and self._count >= self._limit:
      raise StopIteration
    pi, pl = ctypes.c_void_p(), ctypes.c_void_p()
    rc = self._fn["cgan_loader_next"](self._h, ctypes.byref(pi), ctypes.byref(pl))
    if rc != 0:
      raise _lib.CganError("cgan_loader_next failed (%d): %s" % (rc, self._fn["cgan_loader_last_error"](self._h).decode()))
    self._count += 1
    b = self._batch
    nelem = int(np.prod(self._shape))
    images = np.ctypeslib.as_array(ctypes.cast(pi, ctypes.POINTER(ctypes.c_float)), shape=(nelem,)).reshape(self._shape)
    labels = np.ctypeslib.as_array(ctypes.cast(pl, ctypes.POINTER(ctypes.c_int32)), shape=(b,))
    if self._preprocess is not None:
      images, labels = self._preprocess(images, labels)
    return images, labels

  next = __next__

  def release(self, count=1):
    rc = self._fn["cgan_loader_release"](self._h, int(count))
    if rc != 0:
      raise _lib.CganError("cgan_loader_release failed (%d): %s" % (rc, self._fn["cgan_loader_last_error"](self._h).decode()))

  def close(self):
    if self._h:
      self._fn["cgan_loader_destroy"](self._h)
      self._h = ctypes.c_void_p()

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass


class TransformedBatchIterator(object):
  """Python face of a transformed loader (`cgan_loader_create_transformed`, `cgan_crop_resize_u8`).  `next_host()` returns
  numpy views of one page-locked ring slot: the slot's bytes (descriptors, then the packed uint8 windows), the
  descriptors (a CROP_DESC view) and the labels.  `next()` also copies the slot to the slot's device buffer and runs the
  resize there, both on the library's stream, and returns (images float32 [B, R, R, C] on the device, labels).  The
  device batch stays valid until the slot is released: call `release(count)` once the work that reads the `count`
  oldest batches has been issued and completed, as for `BatchIterator`."""

  def __init__(self, pixels, index, labels, colors, transform, resolution, divide_after, batch, shuffle_buffer, seed, ring,
               limit_samples=None):
    _, _, self._fn = _lib.load_functions()
    self._pixels, self._index, self._labels = pixels, index, labels         # keep the source alive
    keep = np.ones(len(index), bool)
    if transform.min_side > 0:
      keep &= np.minimum(index[:, 1], index[:, 2]) >= transform.min_side
    if transform.labeled_only:
      keep &= (labels >= 0) if labels is not None else False
    n = int(keep.sum())
    if n == 0:
      raise ValueError("no element of the source passes the data set's filters")
    self._batch, self._colors, self._resolution, self._divide_after, self._ring = batch, colors, resolution, divide_after, ring
    self._limit = None if limit_samples is None else min(limit_samples, n) // batch
    self._count = 0
    self._dev, self._out = [None] * ring, [None] * ring
    src = ImageSource(pixels.ctypes.data, pixels.shape[0], index.ctypes.data,
                      None if labels is None else labels.ctypes.data, len(index), colors)
    self._h = ctypes.c_void_p()
    rc = self._fn["cgan_loader_create_transformed"](ctypes.byref(self._h), ctypes.byref(src), ctypes.byref(transform),
                                                    int(batch), int(shuffle_buffer), int(seed), int(ring))
    if rc != 0:
      raise _lib.CganError("cgan_loader_create_transformed failed (%d)" % rc)

  def __iter__(self):
    return self

  def next_host(self):
    if self._limit is not None and self._count >= self._limit:
      raise StopIteration
    data, used, lab = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_void_p()
    rc = self._fn["cgan_loader_next_packed"](self._h, ctypes.byref(data), ctypes.byref(used), ctypes.byref(lab))
    if rc != 0:
      raise _lib.CganError("cgan_loader_next_packed failed (%d): %s" % (rc, self._fn["cgan_loader_last_error"](self._h).decode()))
    self._count += 1
    raw = np.ctypeslib.as_array(ctypes.cast(data, ctypes.POINTER(ctypes.c_uint8)), shape=(used.value,))
    descs = raw[:self._batch * CROP_DESC.itemsize].view(CROP_DESC)
    labels = np.ctypeslib.as_array(ctypes.cast(lab, ctypes.POINTER(ctypes.c_int32)), shape=(self._batch,))
    return raw, descs, labels

  def __next__(self):
    import torch
    from . import kernels as K
    raw, _, labels = self.next_host()
    K.lib()
    device = K._RT["device"]
    slot = (self._count - 1) % self._ring
    if self._dev[slot] is None or self._dev[slot].numel() < raw.size:
      self._dev[slot] = torch.empty(raw.size + raw.size // 4, dtype=torch.uint8, device=device)
    if self._out[slot] is None:
      self._out[slot] = torch.empty(self._batch, self._resolution, self._resolution, self._colors, dtype=torch.float32,
                                    device=device)
    buf, out = self._dev[slot], self._out[slot]
    K.sync_stream()
    buf[:raw.size].copy_(torch.from_numpy(raw), non_blocking=True)
    K._call("crop_resize_u8", out.data_ptr(), buf.data_ptr(), buf.data_ptr(), self._batch, self._colors, self._resolution,
            self._divide_after)
    return out, labels

  next = __next__

  def release(self, count=1):
    rc = self._fn["cgan_loader_release"](self._h, int(count))
    if rc != 0:
      raise _lib.CganError("cgan_loader_release failed (%d): %s" % (rc, self._fn["cgan_loader_last_error"](self._h).decode()))

  def close(self):
    if self._h:
      self._fn["cgan_loader_destroy"](self._h)
      self._h = ctypes.c_void_p()
    self._dev, self._out = [None] * self._ring, [None] * self._ring

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass


class CelebaDataset(ImageDatasetV2):
  """CelebA (datasets.py:374-396): resize_image_with_crop_or_pad to 160x160, a bilinear resize of the uint8 values to
  64x64, then / 255; label 0."""
  _source = ("celeb_a", {})

  def _transform(self, train):
    return ImageTransform(crop=CROP_OR_PAD, canvas_h=160, canvas_w=160, label=LABEL_ZERO), 1


class LsunBedroomDataset(ImageDatasetV2):
  """LSUN bedrooms (datasets.py:399-427): resize_image_with_crop_or_pad to 128x128, then / 255; label 0."""
  _source = ("lsun-bedroom", {})

  def _transform(self, train):
    return ImageTransform(crop=CROP_OR_PAD, canvas_h=128, canvas_w=128, label=LABEL_ZERO), 0


class ImagenetDataset(ImageDatasetV2):
  """ImageNet2012 (datasets.py:500-532, 535-584, 638-639): uint8 / 255, then the train or eval crop
  (`train_imagenet_transform.crop_method`, default distorted; `eval_imagenet_transform.crop_method`, default middle) and a
  bilinear resize to R x R.  The train split can be filtered (min(h, w) >= min_side, labels >= 0); labels can be the
  source's, all 0 (single_class) or uniform in [0, 1000) anew for every stream position (random_class)."""
  _source = ("imagenet2012", {"test": "validation"})

  def __init__(self, resolution, seed=547, name=None, num_classes=1000, min_side=0, filter_unlabeled=False,
               label=LABEL_SOURCE, **kwargs):
    if resolution not in (64, 128, 256, 512):
      raise ValueError("Unsupported resolution: {}".format(resolution))
    super(ImagenetDataset, self).__init__(name or "imagenet_%d" % resolution, resolution, 3, num_classes, 50000, seed=seed,
                                          **kwargs)
    self._min_side, self._filter_unlabeled, self._label = min_side, filter_unlabeled, label

  def _transform(self, train):
    t = ImageTransform(crop=train_imagenet_transform() if train else eval_imagenet_transform(), label=self._label,
                       random_classes=1000 if self._label == LABEL_RANDOM else 0)
    if train:
      t.min_side, t.labeled_only = self._min_side, int(self._filter_unlabeled)
    return t, 0


def _imagenet(resolution, **extra):
  return lambda name, res, colors, classes, n_eval, **kw: ImagenetDataset(resolution, name=name, num_classes=classes,
                                                                          **dict(extra, **kw))


_DATASET_CLASSES = {
    "celeb_a": CelebaDataset,
    "lsun-bedroom": LsunBedroomDataset,
    "imagenet_64": _imagenet(64),
    "imagenet_128": _imagenet(128),
    "imagenet_256": _imagenet(256),
    "imagenet_512": _imagenet(512),
    "imagenet_512_hq400": _imagenet(512, min_side=400),
    "single_class_imagenet_128": _imagenet(128, label=LABEL_ZERO),
    "random_class_imagenet_128": _imagenet(128, label=LABEL_RANDOM),
    "labeled_only_imagenet_128": _imagenet(128, filter_unlabeled=True),
}


@gin.configurable("dataset")
def get_dataset(name, seed=547, fake_dataset=True, data_dir=None, shuffle_buffer_size=10000):
  """Instantiates a data set and sets the random seed (reference datasets.py:643-648)."""
  if name not in DATASETS:
    raise ValueError("Dataset %s is not available." % name)
  res, colors, classes, n_eval = DATASETS[name]
  return _DATASET_CLASSES.get(name, ImageDatasetV2)(
      DATASET_NAMES.get(name, name), res, colors, classes, n_eval, seed=seed, fake_dataset=fake_dataset, data_dir=data_dir,
      shuffle_buffer_size=shuffle_buffer_size)
