"""48x48 ResNet pair (reference architectures/resnet_stl.py:33-108; Miyato et al. 2018, table 5) as plans for
`resnet_family`: generator = 6x6 x 8ch seed + three up-sampling blocks 8ch -> 4ch -> 2ch -> ch, BN-ReLU-conv3x3;
discriminator = blocks B0-B3 down-sampling colours -> ch -> 2ch -> 4ch -> 8ch, B4 8ch -> 16ch at 3x3.  Side 48 is not a
power of two, so the discriminator checks only that its input is square.  Neither network applies spectral norm outside
its blocks' own flag but in disc_final_fc."""
from .. import gin_lite as gin
from . import resnet_family as family

SEED = 6


@gin.configurable
class Generator(family.PlainResNetGenerator):

  def __init__(self, ch=64, **kwargs):
    super(Generator, self).__init__(**kwargs)
    self._ch = ch

  def _plan(self):
    return family.GeneratorPlan(widths=[self._ch * m for m in (8, 4, 2, 1)], scales=3 * ["up"], hierarchical_z=False,
                                embed_z=False, embed_y=False, spectral_norm_outside_blocks=False, seed=SEED)


@gin.configurable
class Discriminator(family.PlainResNetDiscriminator):

  def __init__(self, ch=64, **kwargs):
    super(Discriminator, self).__init__(**kwargs)
    self._ch = ch

  def _plan(self, colors):
    return family.DiscriminatorPlan(first_block=0, widths=[self._ch * m for m in (1, 2, 4, 8, 16)],
                                    scales=4 * ["down"] + ["none"], project_y=False, power_of_two=False)
