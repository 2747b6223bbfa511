"""ImageNet / CelebA / LSUN input transforms (reference datasets.py:374-427, 440-584) without a GPU: the numpy oracle
(tests/image_transform_oracle.py) pinned by hand, the transformed loader (csrc/loader.cu) against the oracle's model of
its stream, the device entry above the emulated ABI, and the data set surface."""
import ctypes
import os

import numpy as np
import pytest
import torch

from compare_gan_b200 import datasets as D
from compare_gan_b200 import gin_lite as gin
from tests import image_transform_oracle as O
from tests.abi_emulator import EmulatedLib, emulated_library, f32


def ragged(n=23, seed=0, c=3, lo=1, hi=40, extra=()):
  """A ragged uint8 source: (images, pixels, index)."""
  rng = np.random.RandomState(seed)
  images = [rng.randint(0, 256, size=(rng.randint(lo, hi), rng.randint(lo, hi), c)).astype(np.uint8) for _ in range(n)]
  images += [rng.randint(0, 256, size=s + (c,)).astype(np.uint8) for s in extra]
  pixels, index = pack(images)
  return images, pixels, index


def pack(images):
  off = np.cumsum([0] + [im.size for im in images])[:-1]
  pixels = np.concatenate([im.ravel() for im in images])
  index = np.stack([off, [im.shape[0] for im in images], [im.shape[1] for im in images]], 1).astype(np.int64)
  return pixels, index


def iterator(pixels, index, labels, transform, batch=5, shuffle=7, seed=123, ring=3, c=3, r=16, divide_after=0, limit=None):
  return D.TransformedBatchIterator(pixels, index, labels, c, transform, r, divide_after, batch, shuffle, seed, ring,
                                    limit_samples=limit)


def check_host_batches(it, images, expect):
  for ps, es, wins, _, lab in expect:
    raw, descs, labels = it.next_host()
    assert list(descs["position"]) == ps and list(descs["element"]) == es
    c = images[0].shape[2]
    end = len(descs) * D.CROP_DESC.itemsize
    for d, win, e in zip(descs, wins, es):
      assert {k: int(d[k]) for k in win} == win
      assert d["offset"] == end                                    # windows packed back to back after the table
      window = images[e][win["crop_y"]:win["crop_y"] + win["h"], win["crop_x"]:win["crop_x"] + win["w"]]
      np.testing.assert_array_equal(raw[d["offset"]:d["offset"] + window.size], window.ravel())
      end += win["h"] * win["w"] * c
    assert raw.size == end
    np.testing.assert_array_equal(labels, lab)
    it.release(1)


# ---- the oracle, pinned by hand -------------------------------------------------------------------------------------

def test_oracle_resize_3x5_to_2x2_by_hand():
  img = (10 * np.arange(3)[:, None] + np.arange(5)[None, :]).astype(np.uint8)[:, :, None]
  # scale 1.5 / 2.5: rows 0 and 1.5 (lerp 0.5 between rows 1 and 2), columns 0 and 2.5
  want = np.array([[0.0, 2.5], [15.0, 17.5]], np.float32)[:, :, None]
  np.testing.assert_array_equal(O.resize_bilinear_tf(img.astype(np.float32), 2, 2), want)
  win = O.crop_window("none", 3, 5)
  np.testing.assert_array_equal(O.transform(img, win, 2, True), want / np.float32(255.0))
  f, k = np.float32, np.float32(255.0)
  top = f(12) / k + (f(13) / k - f(12) / k) * f(0.5)                # divide before: taps / 255, then interpolate
  bot = f(22) / k + (f(23) / k - f(22) / k) * f(0.5)
  assert O.transform(img, win, 2, False)[1, 1, 0] == top + (bot - top) * f(0.5)


def test_oracle_celeba_crop_offsets():
  win = O.crop_window("crop_or_pad", 218, 178, canvas=(160, 160))
  assert win == dict(crop_y=29, crop_x=9, h=160, w=160, canvas_h=160, canvas_w=160, top=0, left=0)
  img = np.random.RandomState(1).randint(0, 256, size=(218, 178, 3)).astype(np.uint8)
  got = O.transform(img, win, 64, True)
  want = O.resize_bilinear_tf(img[29:189, 9:169].astype(np.float32), 64, 64) / np.float32(255.0)
  assert got.shape == (64, 64, 3)
  np.testing.assert_array_equal(got, want)
  # the two orders of operations differ in the last bits, and the order matters
  assert (O.transform(img, win, 64, False) != got).any()
  # padding: a short side sits at (target - size) // 2 on a zero canvas
  pad = O.crop_window("crop_or_pad", 100, 200, canvas=(128, 128))
  assert pad == dict(crop_y=0, crop_x=36, h=100, w=128, canvas_h=128, canvas_w=128, top=14, left=0)


def test_oracle_crop_methods():
  assert O.crop_window("middle", 375, 500) == dict(crop_y=0, crop_x=62, h=375, w=375, canvas_h=375, canvas_w=375, top=0, left=0)
  assert O.crop_window("middle", 7, 4)["crop_y"] == 1               # int(float(3) / 2.0) truncates
  for p in range(20):
    win = O.crop_window("random", 30, 50, seed=3, p=p)
    assert win["h"] == win["w"] == 30 and 0 <= win["crop_x"] < 20 and win["crop_y"] == 0
  with pytest.raises(ValueError, match="Unsupported crop method: bogus"):
    O.crop_window("bogus", 3, 3)


@pytest.mark.parametrize("h,w,oh,ow", [(32, 32, 299, 299), (5, 7, 3, 11), (300, 200, 299, 64), (1, 1, 4, 4), (9, 4, 9, 4)])
def test_oracle_agrees_with_inception_resize(h, w, oh, ow):
  from oracle import inception as oinc
  x = np.random.RandomState(h * w).rand(2, h, w, 3).astype(np.float32)
  ref = oinc.resize_bilinear_tf(torch.from_numpy(x), oh, ow).numpy()
  np.testing.assert_array_equal(O.resize_bilinear_tf(x, oh, ow), ref)


# ---- distorted windows ---------------------------------------------------------------------------------------------

def test_distorted_windows_over_a_large_sample():
  h, w = 13, 17
  sides, ys, xs = set(), [], []
  for p in range(4000):
    win = O.crop_window("distorted", h, w, seed=5, p=p)
    s = win["h"]
    assert win["w"] == s and win["canvas_h"] == s and 0.5 * h * w <= s * s <= h * w
    assert 0 <= win["crop_y"] <= max(h - s - 1, 0) and 0 <= win["crop_x"] <= max(w - s - 1, 0)  # never the last offset
    sides.add(s)
    if s < h:
      ys.append(win["crop_y"] == h - s - 1)
  lo, hi = int(np.rint(np.sqrt(np.float32(0.5 * h * w)))), min(h, w)
  assert sides == set(range(lo, hi + 1))                   # the side covers its whole integer range
  assert any(ys)                                            # ... and the largest allowed offset occurs
  whole = O.crop_window("distorted", 10, 31, seed=5, p=0)  # 3:1: every attempt fails, the crop is the whole image
  assert whole == dict(crop_y=0, crop_x=0, h=10, w=31, canvas_h=10, canvas_w=31, top=0, left=0)


def test_loader_distorted_windows_match_the_oracle_on_elongated_images():
  images, pixels, index = ragged(n=6, seed=4, extra=[(10, 31), (31, 10), (20, 40), (1, 1), (2, 1)])
  expect = O.expected_batches(images, "distorted", 8, False, 4, 12, 0, 77)
  it = iterator(pixels, index, None, D.ImageTransform(crop=D.CROP_METHODS["distorted"]), batch=4, shuffle=0, seed=77)
  check_host_batches(it, images, expect)
  it.close()


# ---- the loader against the oracle's stream model ------------------------------------------------------------------

@pytest.mark.parametrize("method", ["distorted", "middle", "random", "none"])
@pytest.mark.parametrize("shuffle", [0, 7, 40])
def test_loader_matches_the_stream_model(method, shuffle):
  images, pixels, index = ragged()
  labels = (np.arange(len(images)) * 7 % 1000).astype(np.int32)
  expect = O.expected_batches(images, method, 16, False, 5, 9, shuffle, 123, labels=labels)
  it = iterator(pixels, index, labels, D.ImageTransform(crop=D.CROP_METHODS[method]), shuffle=shuffle)
  check_host_batches(it, images, expect)
  it.close()


def test_loader_crop_or_pad_and_grayscale():
  images, pixels, index = ragged(n=9, seed=2, c=1, lo=1, hi=30)
  t = D.ImageTransform(crop=D.CROP_OR_PAD, canvas_h=12, canvas_w=20, label=D.LABEL_ZERO)
  expect = O.expected_batches(images, "crop_or_pad", 8, True, 3, 10, 4, 9, canvas=(12, 20), label_mode="zero")
  it = iterator(pixels, index, None, t, batch=3, shuffle=4, seed=9, c=1, r=8, divide_after=1)
  check_host_batches(it, images, expect)
  it.close()


def test_filters_and_the_empty_list():
  images, pixels, index = ragged(n=30, seed=3, lo=5, hi=60)
  labels = np.where(np.arange(30) % 3 == 0, -1, np.arange(30)).astype(np.int32)
  keep = [i for i, im in enumerate(images) if min(im.shape[:2]) >= 30]
  t = D.ImageTransform(crop=D.CROP_METHODS["middle"], min_side=30)
  check_host_batches(iterator(pixels, index, labels, t), images,
                     O.expected_batches(images, "middle", 16, False, 5, 6, 7, 123, keep=keep, labels=labels))
  keep = [i for i in range(30) if labels[i] >= 0]
  t = D.ImageTransform(crop=D.CROP_METHODS["middle"], labeled_only=1)
  expect = O.expected_batches(images, "middle", 16, False, 5, 6, 7, 123, keep=keep, labels=labels)
  check_host_batches(iterator(pixels, index, labels, t), images, expect)
  assert all((e[4] >= 0).all() for e in expect)
  with pytest.raises(ValueError, match="filters"):
    iterator(pixels, index, labels, D.ImageTransform(crop=0, min_side=1000))
  with pytest.raises(ValueError, match="filters"):
    iterator(pixels, index, None, D.ImageTransform(crop=0, labeled_only=1))


def test_single_and_random_class_labels():
  images, pixels, index = ragged(n=10)
  labels = np.arange(10, dtype=np.int32) + 5
  it = iterator(pixels, index, labels, D.ImageTransform(crop=1, label=D.LABEL_ZERO), shuffle=0)
  for _ in range(4):
    assert not it.next_host()[2].any()
    it.release(1)
  it.close()
  t = D.ImageTransform(crop=1, label=D.LABEL_RANDOM, random_classes=1000)
  it = iterator(pixels, index, labels, t, batch=10, shuffle=0)
  epochs = []
  expect = O.expected_batches(images, "middle", 16, False, 10, 3, 0, 123, label_mode="random", classes=1000)
  for k in range(3):
    lab = it.next_host()[2].copy()
    np.testing.assert_array_equal(lab, expect[k][4])
    epochs.append(lab)
    it.release(1)
  it.close()
  assert (epochs[0] != epochs[1]).any() and (epochs[1] != epochs[2]).any()   # a new label for each epoch
  assert all(((e >= 0) & (e < 1000)).all() for e in epochs)


def test_ranks_differ_and_reruns_are_identical(tmp_path):
  images, pixels, index = ragged(n=40, seed=6)
  np.save(str(tmp_path / "imagenet2012_train_pixels.npy"), pixels)
  np.save(str(tmp_path / "imagenet2012_train_index.npy"), index)
  ds = D.get_dataset("imagenet_64", fake_dataset=False, data_dir=str(tmp_path), shuffle_buffer_size=16)
  got = []
  for rank in (0, 1, 0):
    it = ds.train_input_fn({"batch_size": 8}, rank=rank, ring=2)
    raw, descs, _ = it.next_host()
    got.append((raw.copy(), descs.copy()))
    it.close()
  assert not np.array_equal(got[0][1], got[1][1])
  np.testing.assert_array_equal(got[0][0], got[2][0])
  expect = O.expected_batches(images, "distorted", 64, False, 8, 1, 16, 547 + 1)
  assert list(got[1][1]["position"]) == expect[0][0]      # rank r draws on seed + r


# ---- the device entry above the emulated ABI ------------------------------------------------------------------------

def _emulated_crop_resize_u8(self, out, packed, desc, n, c, r, divide_after):
  """cgan_crop_resize_u8 as the header states it, read from raw addresses: each descriptor's window placed on its zero
  canvas, then the legacy bilinear resize, dividing by 255 before or after it."""
  assert c in (1, 3) and divide_after in (0, 1)
  descs = np.ctypeslib.as_array((ctypes.c_uint8 * (n * D.CROP_DESC.itemsize)).from_address(int(desc))).view(D.CROP_DESC)
  y = f32(out, n * r * r * c).reshape(n, r, r, c)
  for b, d in enumerate(descs):
    window = np.ctypeslib.as_array((ctypes.c_uint8 * int(d["h"] * d["w"] * c)).from_address(int(packed) + int(d["offset"])))
    canvas = np.zeros((d["canvas_h"], d["canvas_w"], c), np.float32)
    canvas[d["top"]:d["top"] + d["h"], d["left"]:d["left"] + d["w"]] = window.reshape(d["h"], d["w"], c)
    if divide_after:
      y[b] = O.resize_bilinear_tf(canvas, r, r) / np.float32(255.0)
    else:
      y[b] = O.resize_bilinear_tf(canvas / np.float32(255.0), r, r)


@pytest.fixture
def emulated(monkeypatch):
  monkeypatch.setattr(EmulatedLib, "cgan_crop_resize_u8", _emulated_crop_resize_u8, raising=False)
  with emulated_library() as lib:
    yield lib


@pytest.mark.parametrize("method,divide_after,c", [("distorted", 0, 3), ("middle", 1, 3), ("crop_or_pad", 1, 1),
                                                   ("none", 0, 1), ("random", 0, 3)])
def test_emulated_entry_equals_the_oracle(emulated, method, divide_after, c):
  images, pixels, index = ragged(n=11, seed=8, c=c, extra=[(1, 1), (40, 3)])
  canvas = (20, 14) if method == "crop_or_pad" else None
  crop = D.CROP_OR_PAD if canvas else D.CROP_METHODS[method]
  t = D.ImageTransform(crop=crop, canvas_h=canvas[0] if canvas else 0, canvas_w=canvas[1] if canvas else 0)
  expect = O.expected_batches(images, method, 9, divide_after, 4, 5, 3, 31, canvas=canvas)
  it = iterator(pixels, index, None, t, batch=4, shuffle=3, seed=31, c=c, r=9, divide_after=divide_after)
  for k in range(5):
    x, _ = next(it)
    assert x.dtype == torch.float32 and tuple(x.shape) == (4, 9, 9, c)
    np.testing.assert_array_equal(x.numpy(), expect[k][3])
    it.release(1)
  it.close()
  assert emulated.launches == 5


# ---- sources and the data set surface -------------------------------------------------------------------------------

def test_malformed_sources_raise_value_error(tmp_path):
  images, pixels, index = ragged(n=5)
  ds = D.get_dataset("imagenet_64", fake_dataset=False, data_dir=str(tmp_path))
  fp, fi = str(tmp_path / "imagenet2012_train_pixels.npy"), str(tmp_path / "imagenet2012_train_index.npy")
  np.save(fp, pixels)
  cases = [
      (index.astype(np.int32), "index"),
      (index[:, :2], "index"),
      (index + np.array([[0, 0, 0]] * 4 + [[0, 1, 0]]), "index"),                  # the last image runs past the blob
      (np.where(np.arange(5)[:, None] == 2, [[-1, 3, 3]], index), "index"),
      (np.where(np.arange(5)[:, None] == 0, [[0, 0, 3]], index), "index"),
  ]
  for bad, name in cases:
    np.save(fi, bad)
    with pytest.raises(ValueError, match=name):
      ds.train_input_fn({"batch_size": 2})
  np.save(fi, index)
  np.save(fp, pixels.astype(np.int16))
  with pytest.raises(ValueError, match="pixels"):
    ds.train_input_fn({"batch_size": 2})
  os.remove(fp)
  os.remove(fi)
  np.save(str(tmp_path / "imagenet2012_train_images.npy"), np.zeros((3, 8, 9, 1), np.uint8))    # wrong colours
  with pytest.raises(ValueError, match="imagenet2012_train_images"):
    ds.train_input_fn({"batch_size": 2})
  np.save(str(tmp_path / "imagenet2012_train_images.npy"), np.zeros((3, 8, 9, 3), np.uint8))
  np.save(str(tmp_path / "imagenet2012_train_labels.npy"), np.zeros(4, np.int32))
  with pytest.raises(ValueError, match="labels"):
    ds.train_input_fn({"batch_size": 2})
  with pytest.raises(ValueError, match="no source"):
    ds.eval_input_fn({"batch_size": 2})


def test_fixed_size_sources_use_the_same_table(tmp_path):
  imgs = np.random.RandomState(0).randint(0, 256, size=(7, 218, 178, 3)).astype(np.uint8)
  np.save(str(tmp_path / "celeb_a_train_images.npy"), imgs)
  ds = D.get_dataset("celeb_a", fake_dataset=False, data_dir=str(tmp_path), shuffle_buffer_size=0)
  it = ds.train_input_fn({"batch_size": 3})
  assert isinstance(it, D.TransformedBatchIterator)
  expect = O.expected_batches(list(imgs), "crop_or_pad", 64, True, 3, 4, 0, 547, canvas=(160, 160), label_mode="zero")
  check_host_batches(it, list(imgs), expect)
  it.close()
  # a shard at the data set's own image shape keeps the untransformed host path, bit for bit
  own = np.random.RandomState(1).randint(0, 256, size=(6, 64, 64, 3)).astype(np.uint8)
  np.save(str(tmp_path / "celeb_a_train_images.npy"), own)
  it = ds.train_input_fn({"batch_size": 3})
  assert isinstance(it, D.BatchIterator)
  x, _ = next(it)
  np.testing.assert_array_equal(x, own[:3].astype(np.float32) / np.float32(255.0))
  it.close()


def test_imagenet_eval_reads_the_validation_split(tmp_path):
  images, pixels, index = ragged(n=9, seed=2)
  np.save(str(tmp_path / "imagenet2012_validation_pixels.npy"), pixels)
  np.save(str(tmp_path / "imagenet2012_validation_index.npy"), index)
  np.save(str(tmp_path / "imagenet2012_validation_labels.npy"), np.arange(9, dtype=np.int32))
  ds = D.get_dataset("imagenet_64", fake_dataset=False, data_dir=str(tmp_path))
  it = ds.eval_input_fn({"batch_size": 4})
  expect = O.expected_batches(images, "middle", 64, False, 4, 2, 0, 547, labels=np.arange(9))
  check_host_batches(it, images, expect)
  with pytest.raises(StopIteration):                       # the first min(eval_test_samples, N) // batch batches
    it.next_host()
  it.close()


REFERENCE_PROPERTIES = {   # name -> (image_shape, num_classes, eval_test_samples, data set name)   datasets.py:374-640
    "imagenet_64": ((64, 64, 3), 1000, 50000, "imagenet_64"),
    "imagenet_128": ((128, 128, 3), 1000, 50000, "imagenet_128"),
    "imagenet_256": ((256, 256, 3), 1000, 50000, "imagenet_256"),
    "imagenet_512": ((512, 512, 3), 1000, 50000, "imagenet_512"),
    "imagenet_512_hq400": ((512, 512, 3), 1000, 50000, "imagenet_512_hq400"),
    "single_class_imagenet_128": ((128, 128, 3), 1, 50000, "single_class_imagenet_128"),
    "random_class_imagenet_128": ((128, 128, 3), 1000, 50000, "random_class_imagenet_128"),
    "labeled_only_imagenet_128": ((128, 128, 3), 1000, 50000, "imagenet_128"),
    "celeb_a": ((64, 64, 3), None, 10000, "celeb_a"),
    "lsun-bedroom": ((128, 128, 3), None, 30000, "lsun-bedroom"),
}


@pytest.mark.parametrize("name", sorted(REFERENCE_PROPERTIES))
def test_dataset_names_resolve(name):
  ds = D.get_dataset(name)
  shape, classes, n_eval, ds_name = REFERENCE_PROPERTIES[name]
  assert (ds.image_shape, ds.num_classes, ds.eval_test_samples, ds.name) == (shape, classes, n_eval, ds_name)
  with pytest.raises(ValueError, match="not available"):
    D.get_dataset("soft_labeled_imagenet_128")
  with pytest.raises(ValueError, match="Unsupported resolution: 96"):
    D.ImagenetDataset(96)


def test_crop_method_bindings():
  try:
    assert D.train_imagenet_transform() == D.CROP_METHODS["distorted"]
    assert D.eval_imagenet_transform() == D.CROP_METHODS["middle"]
    gin.parse_config('train_imagenet_transform.crop_method = "random"\neval_imagenet_transform.crop_method = "none"')
    assert D.train_imagenet_transform() == D.CROP_METHODS["random"]
    assert D.eval_imagenet_transform() == D.CROP_METHODS["none"]
    t, divide_after = D.get_dataset("imagenet_128")._transform(True)
    assert t.crop == D.CROP_METHODS["random"] and divide_after == 0
    gin.parse_config('train_imagenet_transform.crop_method = "squash"')
    with pytest.raises(ValueError, match="Unsupported crop method: squash"):
      D.train_imagenet_transform()
  finally:
    gin.clear_config()
