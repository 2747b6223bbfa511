"""What the transformed ImageNet input path (csrc/loader.cu's cgan_loader_create_transformed, csrc/image_transform.cu's
cgan_crop_resize_u8) costs at imagenet_128, on a seeded ragged ImageNet-like source written to a temporary directory
(sides drawn around 500 x 375, landscape and portrait):

* producer throughput: batches of 256 taken from the loader's ring on the host (crop windows picked, their rows packed),
  in images/s;
* host->device bytes per batch (descriptors plus packed uint8 windows) against the float32 batch the target-shaped path
  uploads (256 x 128 x 128 x 3 x 4 bytes);
* the time of one batch's host->device copy and of one cgan_crop_resize_u8 launch, from CUDA events over many repeats;
* a biggan_imagenet128-shaped training cycle (CUDA-graph replay, batch 64 per GPU as bench.py's biggan_imagenet128
  workload) fed from the pipeline against the same cycle fed synthetic inputs, in ms per cycle, alternated twice.

Writes OUT_DIR/prof_image_pipeline.json with the card's name and power limit.

  python profiles/prof_image_pipeline.py [--images 2000] [--batch 256] [--cycles 10] [--cycle-batch 64] [--skip-cycle] [--out OUT_DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from compare_gan_b200 import datasets, kernels as K

RES = 128


def write_source(d, n, seed=0):
  """A ragged imagenet2012_train source: n images of about 500 x 375 (either orientation), random labels."""
  rng = np.random.RandomState(seed)
  long_side = rng.randint(400, 600, n)
  short_side = (long_side * rng.uniform(0.6, 0.9, n)).astype(np.int64)
  portrait = rng.rand(n) < 0.25
  h, w = np.where(portrait, long_side, short_side), np.where(portrait, short_side, long_side)
  sizes = h * w * 3
  index = np.stack([np.concatenate([[0], np.cumsum(sizes)[:-1]]), h, w], 1).astype(np.int64)
  pixels = np.lib.format.open_memmap(os.path.join(d, "imagenet2012_train_pixels.npy"), mode="w+", dtype=np.uint8,
                                     shape=(int(sizes.sum()),))
  for i in range(n):                   # random content: the values do not matter to the timings
    pixels[index[i, 0]:index[i, 0] + sizes[i]] = rng.randint(0, 256, sizes[i], dtype=np.uint8)
  pixels.flush()
  del pixels
  np.save(os.path.join(d, "imagenet2012_train_index.npy"), index)
  np.save(os.path.join(d, "imagenet2012_train_labels.npy"), rng.randint(0, 1000, n).astype(np.int32))


def producer_throughput(ds, batch, batches):
  it = ds.train_input_fn({"batch_size": batch}, ring=4)
  nbytes = []
  it.next_host()                       # the first fill includes the ring's allocation
  it.release(1)
  t0 = time.perf_counter()
  for _ in range(batches):
    raw, _, _ = it.next_host()
    nbytes.append(raw.size)
    it.release(1)
  dt = time.perf_counter() - t0
  it.close()
  return batch * batches / dt, float(np.mean(nbytes)), float(np.max(nbytes))


def device_times(ds, batch, repeats=50):
  it = ds.train_input_fn({"batch_size": batch}, ring=2)
  raw, _, _ = it.next_host()
  host = torch.from_numpy(raw)
  buf = torch.empty(raw.size, dtype=torch.uint8, device="cuda")
  out = torch.empty(batch, RES, RES, 3, device="cuda")
  K.sync_stream()

  def timed(fn):
    for _ in range(3):
      fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(repeats):
      fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / repeats

  copy_ms = timed(lambda: buf.copy_(host, non_blocking=True))
  kernel_ms = timed(lambda: K._call("crop_resize_u8", out.data_ptr(), buf.data_ptr(), buf.data_ptr(), batch, 3, RES, 0))
  it.release(1)
  it.close()
  return copy_ms, kernel_ms


def cycle_ms(data_dir, batch, cycles, pipeline):
  """ms per graph-replayed cycle, inputs included: run_with_schedule's loop, timed from after three warm-up cycles to a
  device synchronise."""
  import gc
  from compare_gan_b200 import configs, gin_lite as gin, runner_lib
  from compare_gan_b200.gans import modular_gan  # noqa: F401
  gin.clear_config()
  gin.parse_config(configs.BIGGAN_IMAGENET128)
  gin.parse_config("\n".join(["options.batch_size = %d" % batch, "dataset.fake_dataset = False",
                              'dataset.data_dir = "%s"' % data_dir]))
  dataset = datasets.get_dataset()
  options = runner_lib.get_options_dict()
  with tempfile.TemporaryDirectory() as md:
    gan = options["gan_class"](dataset=dataset, parameters=options, model_dir=md)
    gan.build(batch)
    gan.capture()
    rng = np.random.RandomState(0)
    feeder = runner_lib.PipelineFeeder(gan, dataset, batch) if pipeline else None

    def step():
      if feeder is not None:
        feeder.feed(gan, dataset, batch, rng)
      else:
        gan.set_inputs(*runner_lib.sample_cycle_inputs(gan, dataset, batch, rng))
      gan.run_cycle()
    for _ in range(3):
      step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(cycles):
      step()
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t0) / cycles
    if feeder is not None:
      feeder.close()
  del gan, feeder
  gin.clear_config()
  gc.collect()
  torch.cuda.empty_cache()
  return ms


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--images", type=int, default=2000)
  ap.add_argument("--batch", type=int, default=256)
  ap.add_argument("--batches", type=int, default=20)
  ap.add_argument("--cycles", type=int, default=10)
  ap.add_argument("--cycle-batch", type=int, default=64)
  ap.add_argument("--skip-cycle", action="store_true")
  ap.add_argument("--out", default="prof_image_pipeline_out")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("prof_image_pipeline.py measures on a CUDA device; none is present")
  K.init(0)
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip()
  res = {"card": card, "images": args.images, "batch": args.batch, "resolution": RES}
  with tempfile.TemporaryDirectory() as d:
    write_source(d, args.images)
    ds = datasets.get_dataset("imagenet_128", fake_dataset=False, data_dir=d)
    ips, mean_bytes, max_bytes = producer_throughput(ds, args.batch, args.batches)
    res["producer_images_per_s"] = ips
    res["h2d_bytes_per_batch_mean"] = mean_bytes
    res["h2d_bytes_per_batch_max"] = max_bytes
    res["float_path_bytes_per_batch"] = args.batch * RES * RES * 3 * 4
    res["h2d_copy_ms"], res["crop_resize_kernel_ms"] = device_times(ds, args.batch)
    print(json.dumps(res, indent=1), flush=True)
    if not args.skip_cycle:
      res["cycle_batch"] = args.cycle_batch
      for rep in range(2):               # alternated, to see the spread
        for mode in ("pipeline", "synthetic"):
          res.setdefault("cycle_ms_" + mode, []).append(cycle_ms(d, args.cycle_batch, args.cycles, mode == "pipeline"))
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "prof_image_pipeline.json"), "w") as f:
    json.dump(res, f, indent=1)
  print(json.dumps(res, indent=1))


if __name__ == "__main__":
  main()
