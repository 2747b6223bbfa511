"""The data set transforms on the device: `cgan_crop_resize_u8` (csrc/image_transform.cu) bit for bit against the numpy
float32 oracle (tests/image_transform_oracle.py), and the transformed sources end to end through `run_with_schedule`
and the real side of the evaluation."""
import numpy as np
import pytest

from compare_gan_b200 import datasets as D
from tests import image_transform_oracle as O
from tests.test_image_transforms import pack

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  return kernels


def sized_images(shapes, c, seed):
  rng = np.random.RandomState(seed)
  return [rng.randint(0, 256, size=s + (c,)).astype(np.uint8) for s in shapes]


# (method, canvas, r, divide_after, c, image shapes): up- and down-sampling, odd sizes, windows touching every edge,
# padded canvases, 1x1 windows
CASES = [
    ("none", None, 7, 0, 3, [(1, 1), (3, 5), (13, 9), (40, 41), (7, 7), (2, 30)]),
    ("none", None, 33, 1, 1, [(1, 1), (5, 3), (31, 17), (64, 64), (9, 50), (3, 3)]),
    ("middle", None, 16, 0, 3, [(375, 500), (17, 23), (16, 16), (1, 9), (101, 3), (50, 49)]),
    ("random", None, 12, 1, 3, [(30, 45), (45, 30), (12, 12), (1, 1), (7, 100), (99, 98)]),
    ("distorted", None, 64, 0, 3, [(375, 500), (61, 40), (10, 31), (2, 2), (1, 3), (128, 127)]),
    ("distorted", None, 5, 1, 1, [(375, 500), (61, 40), (10, 31), (2, 2), (1, 1), (128, 127)]),
    ("crop_or_pad", (20, 14), 9, 1, 3, [(218, 178), (5, 30), (30, 5), (1, 1), (20, 14), (19, 13)]),
    ("crop_or_pad", (16, 16), 16, 0, 1, [(10, 40), (40, 10), (1, 1), (16, 16), (3, 17), (33, 2)]),
]


def transform_of(method, canvas):
  if canvas:
    return D.ImageTransform(crop=D.CROP_OR_PAD, canvas_h=canvas[0], canvas_w=canvas[1])
  return D.ImageTransform(crop=D.CROP_METHODS[method])


def run_iterator(images, method, canvas, r, divide_after, c, batch, nb, seed):
  pixels, index = pack(images)
  it = D.TransformedBatchIterator(pixels, index, None, c, transform_of(method, canvas), r, divide_after, batch, 5, seed, 3)
  got = []
  for _ in range(nb):
    x, _ = next(it)
    got.append(x.to("cpu", copy=True).numpy())
    it.release(1)
  it.close()
  return got


@pytest.mark.parametrize("case", range(len(CASES)))
def test_crop_resize_matches_the_oracle_bit_for_bit(K, case):
  method, canvas, r, divide_after, c, shapes = CASES[case]
  images = sized_images(shapes, c, case)
  batch, nb = 4, 6
  expect = O.expected_batches(images, method, r, divide_after, batch, nb, 5, 11, canvas=canvas)
  got = run_iterator(images, method, canvas, r, divide_after, c, batch, nb, 11)
  for k in range(nb):
    np.testing.assert_array_equal(got[k], expect[k][3], err_msg="batch %d" % k)
  again = run_iterator(images, method, canvas, r, divide_after, c, batch, nb, 11)
  for a, b in zip(got, again):
    assert a.tobytes() == b.tobytes()                  # reruns are bit-identical
  assert K.lib().launch_count() > 0


def imagenet_source(tmp_path, seed=0):
  rng = np.random.RandomState(seed)
  train = [rng.randint(0, 256, size=(rng.randint(40, 110), rng.randint(40, 110), 3)).astype(np.uint8) for _ in range(37)]
  val = [rng.randint(0, 256, size=(rng.randint(40, 110), rng.randint(40, 110), 3)).astype(np.uint8) for _ in range(21)]
  for split, images in (("train", train), ("validation", val)):
    pixels, index = pack(images)
    np.save(str(tmp_path / ("imagenet2012_%s_pixels.npy" % split)), pixels)
    np.save(str(tmp_path / ("imagenet2012_%s_index.npy" % split)), index)
    np.save(str(tmp_path / ("imagenet2012_%s_labels.npy" % split)), rng.randint(0, 1000, len(images)).astype(np.int32))
  return train, val


def _train(tmp_path, data_dir, use_graph, cycles=3):
  from compare_gan_b200 import configs, gin_lite as gin, runner_lib
  from compare_gan_b200.gans import modular_gan  # noqa: F401
  gin.clear_config()
  gin.parse_config(configs.DCGAN_CELEBA64)
  gin.parse_config("\n".join(['dataset.name = "imagenet_64"', "dataset.fake_dataset = False",
                              'dataset.data_dir = "%s"' % data_dir, "dataset.shuffle_buffer_size = 16",
                              "options.batch_size = 8"]))
  return runner_lib.run_with_schedule("train", model_dir=str(tmp_path / ("run%d" % use_graph)), num_cycles=cycles,
                                      use_graph=use_graph, input_pipeline=True)


def test_imagenet_pipeline_end_to_end(K, tmp_path):
  """run_with_schedule("train", input_pipeline=True) on a ragged imagenet2012 source at imagenet_64: after the last
  cycle the device inputs are the oracle's batches for exactly the stream positions the model predicts; graph replay
  equals eager; the real images of an evaluation are the oracle's centre crops of the validation split."""
  from compare_gan_b200 import eval_gan_lib, gin_lite as gin
  train, val = imagenet_source(tmp_path)
  labels = np.load(str(tmp_path / "imagenet2012_train_labels.npy"))
  try:
    outs = [_train(tmp_path, str(tmp_path), use_graph) for use_graph in (False, True)]
    for out in outs:
      gan = out["gan"]
      k1 = gan._disc_iters + 1
      expect = O.expected_batches(train, "distorted", 64, False, 8, 3 * k1, 16, 547, labels=labels)
      for i in range(k1):
        np.testing.assert_array_equal(gan.inputs[i]["images"].cpu(), expect[2 * k1 + i][3])
        if gan.conditional:
          np.testing.assert_array_equal(np.asarray(gan.inputs[i]["labels"].cpu()).ravel(), expect[2 * k1 + i][4])
      assert np.isfinite(out["g_loss"])
    assert outs[0]["d_loss"] == outs[1]["d_loss"] and outs[0]["g_loss"] == outs[1]["g_loss"]
    ds = D.get_dataset()
    real = eval_gan_lib._real_images(ds, 16, 16, 0, 1, 8)
    expect = O.expected_batches(val, "middle", 64, False, 8, 2, 0, 547)
    np.testing.assert_array_equal(real, np.concatenate([e[3] for e in expect]))
  finally:
    gin.clear_config()


def test_celeba_and_lsun_sources(K, tmp_path):
  rng = np.random.RandomState(3)
  celeb = rng.randint(0, 256, size=(9, 218, 178, 3)).astype(np.uint8)
  np.save(str(tmp_path / "celeb_a_train_images.npy"), celeb)
  ds = D.get_dataset("celeb_a", fake_dataset=False, data_dir=str(tmp_path), shuffle_buffer_size=4)
  it = ds.train_input_fn({"batch_size": 4})
  expect = O.expected_batches(list(celeb), "crop_or_pad", 64, True, 4, 5, 4, 547, canvas=(160, 160), label_mode="zero")
  for k in range(5):
    x, lab = next(it)
    np.testing.assert_array_equal(x.to("cpu", copy=True).numpy(), expect[k][3])
    assert not lab.any()
    it.release(1)
  it.close()
  lsun = [rng.randint(0, 256, size=s + (3,)).astype(np.uint8) for s in [(128, 171), (256, 192), (100, 140), (128, 128),
                                                                          (90, 60), (300, 129)]]
  pixels, index = pack(lsun)
  np.save(str(tmp_path / "lsun-bedroom_train_pixels.npy"), pixels)
  np.save(str(tmp_path / "lsun-bedroom_train_index.npy"), index)
  ds = D.get_dataset("lsun-bedroom", fake_dataset=False, data_dir=str(tmp_path), shuffle_buffer_size=0)
  it = ds.train_input_fn({"batch_size": 3})
  expect = O.expected_batches(lsun, "crop_or_pad", 128, False, 3, 4, 0, 547, canvas=(128, 128), label_mode="zero")
  for k in range(4):
    x, _ = next(it)
    got = x.to("cpu", copy=True).numpy()
    np.testing.assert_array_equal(got, expect[k][3])
    for b, e in enumerate(expect[k][1]):                # no resize: the crop-or-pad canvas / 255 exactly
      win = O.crop_window("crop_or_pad", *lsun[e].shape[:2], canvas=(128, 128))
      np.testing.assert_array_equal(got[b], O.canvas_of(lsun[e], win).astype(np.float32) / np.float32(255.0))
    it.release(1)
  it.close()
