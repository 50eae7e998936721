from .ggraph3D_dataset import QM93DGEN, collate_fn

__all__ = [
    "QM93DGEN",
    "collate_fn"
]
