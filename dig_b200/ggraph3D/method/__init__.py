from .G_SphereNet import G_SphereNet  # noqa: F401

__all__ = ["G_SphereNet"]
