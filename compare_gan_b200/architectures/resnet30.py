"""30-block ResNet pair for 128x128 (reference architectures/resnet30.py:36-143; after the 64x64 ResNet of Gulrajani et
al. 2017) as plans for `resnet_family`.  Both networks are six superblocks of five width-preserving blocks B_<s>_<i>;
the first five superblocks end in a resampling block B_<s>_up (the discriminator's down-sampling ones keep that name).
The generator runs 4x4 x 8ch -> 128x128 x ch/4 with no final norm or ReLU before final_conv; the discriminator maps the
colours to ch/4 with color_conv, doubles the width in every B_<s>_up up to 8ch at 4x4 and feeds the flattened 4x4 x 8ch
map straight to disc_final_fc.  No spectral norm outside the blocks but in disc_final_fc."""
from .. import gin_lite as gin
from . import resnet_family as family

SUPERBLOCKS = 6
BLOCKS = 5


def _superblocks(first_width, factor, scale):
  """(names, per-block output widths, scales) of the six superblocks, starting at `first_width`."""
  names, widths, scales = [], [], []
  width = first_width
  for s in range(SUPERBLOCKS):
    names += ["B_%d_%d" % (s, i) for i in range(BLOCKS)]
    widths += BLOCKS * [width]
    scales += BLOCKS * ["none"]
    if s < SUPERBLOCKS - 1:
      width = int(width * factor)
      names.append("B_%d_up" % s)
      widths.append(width)
      scales.append(scale)
  return names, widths, scales


@gin.configurable
class Generator(family.PlainResNetGenerator):

  def __init__(self, ch=64, **kwargs):
    super(Generator, self).__init__(**kwargs)
    self._ch = ch

  def _plan(self):
    names, widths, scales = _superblocks(8 * self._ch, 0.5, "up")
    return family.GeneratorPlan(widths=[8 * self._ch] + widths, scales=scales, hierarchical_z=False, embed_z=False,
                                embed_y=False, spectral_norm_outside_blocks=False, names=names, final_norm=False)


@gin.configurable
class Discriminator(family.PlainResNetDiscriminator):

  def __init__(self, ch=64, **kwargs):
    super(Discriminator, self).__init__(**kwargs)
    self._ch = ch

  def _plan(self, colors):
    names, widths, scales = _superblocks(self._ch // 4, 2, "down")
    return family.DiscriminatorPlan(first_block=0, widths=widths, scales=scales, project_y=False, names=names,
                                    color_conv=self._ch // 4, flatten=True)
