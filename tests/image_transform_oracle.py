"""A numpy float32 restatement of the reference's ImageNet / CelebA / LSUN input transforms (reference datasets.py:374-427,
440-584) and of the stream the transformed loader (csrc/loader.cu, cgan_loader_create_transformed) draws them on.

* Crops: `middle`, `random`, `none`, `distorted` (tf.image.sample_distorted_bounding_box with aspect ratio [1, 1], area
  [0.5, 1], 100 attempts, as TF 1.x's GenerateRandomCrop in core/kernels/sample_distorted_bounding_box_op.cc reads:
  restated from that source, not run against TF, which is not installed here), and
  tf.image.resize_image_with_crop_or_pad.
* Resize: tf.image.resize_images, TF1's legacy bilinear kernel (align_corners = False, no half-pixel offset), every
  operation a separately rounded float32 operation.  Whether TF's own CPU build contracted these multiply-adds is
  unverified.
* Random draws: SplitMix64 streams keyed by (seed, stream position p, stream id), as the loader documents.
"""
import numpy as np

M64 = (1 << 64) - 1
CROP_STREAM, LABEL_STREAM = 0, 1


def _splitmix_out(state):
  z = state
  z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
  z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
  return z ^ (z >> 31)


class Stream(object):
  """SplitMix64 from a 64-bit state."""

  def __init__(self, state):
    self.state = state & M64

  def next(self):
    self.state = (self.state + 0x9E3779B97F4A7C15) & M64
    return _splitmix_out(self.state)

  def below(self, bound):
    limit = M64 - M64 % bound
    while True:
      r = self.next()
      if r < limit:
        return r % bound

  def unit(self):
    return np.float32(self.next() >> 40) * np.float32(1.0 / 16777216.0)


def mix(x):
  return _splitmix_out((x + 0x9E3779B97F4A7C15) & M64)


def draw_stream(seed, p, stream_id):
  return Stream(mix(mix(mix(seed & M64) ^ p) ^ stream_id))


def shuffled_positions(buffer_size, seed, count):
  """Stream positions p of tf.data's shuffle over the repeated stream 0, 1, 2, ... (the element is list[p % n])."""
  if buffer_size <= 1:
    return list(range(count))
  s = Stream(seed)
  buf = list(range(buffer_size))
  nxt, out = buffer_size, []
  for _ in range(count):
    slot = s.below(buffer_size)
    out.append(buf[slot])
    buf[slot] = nxt
    nxt += 1
  return out


def _lrintf(x):
  return int(np.rint(np.float32(x)))


def distorted_window(h, w, s):
  """(y, x, side) of sample_distorted_bounding_box's crop; (0, 0, 0) when 100 attempts fail (the whole image)."""
  f32 = np.float32
  min_area, max_area = f32(0.5) * f32(w) * f32(h), f32(1.0) * f32(w) * f32(h)
  for _ in range(100):
    side = _lrintf(np.sqrt(min_area))
    max_side = min(_lrintf(np.sqrt(max_area)), w, h)
    side = min(side, max_side)
    if side < max_side:
      side += s.below(max_side - side + 1)
    area = f32(side * side)
    if area < min_area:
      side += 1
      area = f32(side * side)
    if area > max_area:
      side -= 1
      area = f32(side * side)
    if area < min_area or area > max_area or side > w or side > h or side <= 0:
      continue
    y = s.below(h - side) if side < h else 0
    x = s.below(w - side) if side < w else 0
    return y, x, side
  return 0, 0, 0


def crop_window(method, h, w, seed=0, p=0, canvas=None):
  """dict(crop_y, crop_x, h, w, canvas_h, canvas_w, top, left): the window in the source and its place on the canvas."""
  s = draw_stream(seed, p, CROP_STREAM)
  cy = cx = top = left = 0
  wh, ww, ch, cw = h, w, h, w
  if method == "middle":
    side = min(h, w)
    cy, cx = int(np.float32(h - side) / np.float32(2.0)), int(np.float32(w - side) / np.float32(2.0))
    wh = ww = ch = cw = side
  elif method == "random":
    side = min(h, w)
    uy, ux = s.unit(), s.unit()
    cy, cx = int(np.float32(h - side) * uy), int(np.float32(w - side) * ux)
    wh = ww = ch = cw = side
  elif method == "distorted":
    y, x, side = distorted_window(h, w, s)
    if side:
      cy, cx, wh, ww, ch, cw = y, x, side, side, side, side
  elif method == "crop_or_pad":
    ch, cw = canvas
    if h > ch:
      cy, wh = (h - ch) // 2, ch
    else:
      top = (ch - h) // 2
    if w > cw:
      cx, ww = (w - cw) // 2, cw
    else:
      left = (cw - w) // 2
  elif method != "none":
    raise ValueError("Unsupported crop method: {}".format(method))
  return dict(crop_y=cy, crop_x=cx, h=wh, w=ww, canvas_h=ch, canvas_w=cw, top=top, left=left)


def canvas_of(image, win):
  """uint8 [canvas_h, canvas_w, C]: the window placed on a zero canvas (resize_image_with_crop_or_pad)."""
  out = np.zeros((win["canvas_h"], win["canvas_w"], image.shape[2]), np.uint8)
  out[win["top"]:win["top"] + win["h"], win["left"]:win["left"] + win["w"]] = \
      image[win["crop_y"]:win["crop_y"] + win["h"], win["crop_x"]:win["crop_x"] + win["w"]]
  return out


def _taps(n_in, n_out):
  f32 = np.float32
  src = np.arange(n_out, dtype=f32) * (f32(n_in) / f32(n_out))
  lo = np.floor(src).astype(np.int64)
  hi = np.minimum(lo + 1, n_in - 1)
  return lo, hi, (src - lo.astype(f32)).astype(f32)


def resize_bilinear_tf(x, oh, ow):
  """tf.image.resize_images (legacy bilinear, align_corners = False) of float32 [..., H, W, C] without FMA contraction."""
  x = np.asarray(x, np.float32)
  h, w = x.shape[-3], x.shape[-2]
  y0, y1, ly = _taps(h, oh)
  x0, x1, lx = _taps(w, ow)
  lx = lx[:, None]
  ly = ly[:, None, None]
  rows0, rows1 = x[..., y0, :, :], x[..., y1, :, :]
  tl, tr, bl, br = rows0[..., x0, :], rows0[..., x1, :], rows1[..., x0, :], rows1[..., x1, :]
  top = tl + (tr - tl) * lx
  bot = bl + (br - bl) * lx
  return (top + (bot - top) * ly).astype(np.float32)


def transform(image, win, r, divide_after):
  """One element: crop (or pad) `image` uint8 [H, W, C] by `win`, resize to r x r.  divide_after = False divides by 255
  before the resize (ImageNet), True after it (CelebA)."""
  canvas = canvas_of(image, win).astype(np.float32)
  if divide_after:
    return resize_bilinear_tf(canvas, r, r) / np.float32(255.0)
  return resize_bilinear_tf(canvas / np.float32(255.0), r, r)


def random_label(seed, p, classes):
  return draw_stream(seed, p, LABEL_STREAM).below(classes)


def expected_batches(images, method, r, divide_after, batch, nbatches, shuffle_buffer, seed, canvas=None, keep=None,
                     labels=None, label_mode="source", classes=1000):
  """The loader's batches: for each, (positions, elements, windows, float32 [batch, r, r, C], labels).  images: a list
  of uint8 [h, w, C] arrays; keep: the element list after the filters (default: every image)."""
  lst = list(range(len(images))) if keep is None else list(keep)
  pos = shuffled_positions(shuffle_buffer, seed, batch * nbatches)
  out = []
  for k in range(nbatches):
    ps = pos[k * batch:(k + 1) * batch]
    es = [lst[p % len(lst)] for p in ps]
    wins = [crop_window(method, images[e].shape[0], images[e].shape[1], seed, p, canvas) for p, e in zip(ps, es)]
    x = np.stack([transform(images[e], wn, r, divide_after) for e, wn in zip(es, wins)])
    if label_mode == "zero":
      lab = [0] * batch
    elif label_mode == "random":
      lab = [random_label(seed, p, classes) for p in ps]
    else:
      lab = [int(labels[e]) if labels is not None else 0 for e in es]
    out.append((ps, es, wins, x, np.array(lab, np.int32)))
  return out
