"""Public names of the weight initialisers and architectures that gin files and `ModularGAN` refer to (the string values
are the reference's, gans/consts.py:28-40, because `options.architecture = "resnet_cifar_arch"` etc. must keep working).
`IMPLEMENTED_ARCHITECTURES` are the ones the H100 engine builds; asking for any other raises NotImplementedError in
`ModularGAN` exactly as an unknown name does in the reference (modular_gan.py:184-187)."""

# weights.initializer values -> NORMAL_INIT, TRUNCATED_INIT, ORTHOGONAL_INIT
INITIALIZERS = []
for _name in ("normal", "truncated", "orthogonal"):
  globals()[_name.upper() + "_INIT"] = _name
  INITIALIZERS.append(_name)

# options.architecture values -> <NAME>_ARCH = "<name>_arch", listed in the reference's order
ARCHITECTURES = []
for _name in ("infogan", "dcgan", "resnet_cifar", "sndcgan", "resnet5", "resnet30", "resnet_stl", "resnet_biggan",
              "resnet_biggan_deep"):
  globals()[_name.upper() + "_ARCH"] = _name + "_arch"
  ARCHITECTURES.append(_name + "_arch")
DUMMY_ARCH = "dummy_arch"          # the reference's test-only architecture name

IMPLEMENTED_ARCHITECTURES = ["infogan_arch", "dcgan_arch", "resnet_cifar_arch", "sndcgan_arch", "resnet5_arch", "resnet30_arch",
                             "resnet_stl_arch", "resnet_biggan_arch", "resnet_biggan_deep_arch"]
del _name
