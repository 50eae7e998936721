from .sphgen import SphGen, TorchDraws  # noqa: F401
