"""Drop-in replacement for the `simple_knn` package of the reference's submodules/simple-knn (absent from the reference
checkout): `_C.distCUDA2`, the 3-nearest-neighbour distances GaussianModel.create_from_pcd turns into the initial
scales (scene/gaussian_model.py:21, 190-194)."""
from . import _C  # noqa: F401
