"""Dataset surface (reference datasets.py:66-329, 620-648).  BASELINE measures on synthetic data (`sample_images`:
uniform [0,1) images, seed 547, datasets.py:136-145).  The input pipeline of `train_input_fn` / `eval_input_fn`
(datasets.py:261-329: repeat -> shuffle -> batch(drop_remainder) -> prefetch) runs in the native loader
(`csrc/loader.cu`, `cgan_loader_*`) over the reference's fake data set or over uint8 NHWC shards on disk; TFDS itself
(download + decode) is not available offline and is replaced by `<data_dir>/<name>_<split>_images.npy` /
`_labels.npy` files."""
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
    "imagenet_128": (128, 3, 1000, 50000),
    "mnist": (28, 1, 10, 10000),                   # datasets.py:332-343
    "fashion-mnist": (28, 1, 10, 10000),           # datasets.py:346-357
}
# keys whose data set goes by another name (ImageDatasetV2.name, which also names the shard files)
DATASET_NAMES = {"fashion-mnist": "fashion_mnist"}


class ImageDatasetV2(object):
  """Synthetic stand-in exposing name / image_shape / num_classes / eval_test_samples."""

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
    if not self._data_dir:
      raise ValueError("Dataset %s: no data_dir (dataset.data_dir or $CGAN_DATA_DIR) and fake_dataset is off; TFDS "
                       "downloads are not available here." % self._name)
    base = os.path.join(self._data_dir, "%s_%s" % (self._name, split))
    images = np.load(base + "_images.npy", mmap_mode="r")
    if images.dtype != np.uint8 or images.shape[1:] != self.image_shape:
      raise ValueError("%s_images.npy must be uint8 [N,%d,%d,%d], got %s %s" % ((base,) + self.image_shape + (images.dtype, images.shape)))
    labels = np.load(base + "_labels.npy", mmap_mode="r").astype(np.int32) if os.path.exists(base + "_labels.npy") else None
    return images, labels

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
    images, labels = self._load_dataset(self._train_split)
    return BatchIterator(images, labels, params["batch_size"], self._shuffle_buffer_size,
                         self._get_per_host_random_seed(rank), ring, preprocess_fn=preprocess_fn)

  def eval_input_fn(self, params=None, split=None, ring=4):
    """Finite, unshuffled iterator over the first eval_test_samples of the eval split (datasets.py:293-318)."""
    params = params or {}
    if "batch_size" not in params:
      raise ValueError("eval_input_fn needs params['batch_size'].")
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


@gin.configurable("dataset")
def get_dataset(name, seed=547, fake_dataset=True, data_dir=None, shuffle_buffer_size=10000):
  """Instantiates a data set and sets the random seed (reference datasets.py:643-648)."""
  if name not in DATASETS:
    raise ValueError("Dataset %s is not available." % name)
  res, colors, classes, n_eval = DATASETS[name]
  return ImageDatasetV2(DATASET_NAMES.get(name, name), res, colors, classes, n_eval, seed=seed, fake_dataset=fake_dataset, data_dir=data_dir,
                        shuffle_buffer_size=shuffle_buffer_size)
