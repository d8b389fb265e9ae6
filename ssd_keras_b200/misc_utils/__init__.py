"""Weight-file plumbing (SURVEY.md section 8f(1)): a dependency-free reader and writer for Keras HDF5 weight files
(``hdf5_lite``), and the class transfer of ``weight_sampling_tutorial.ipynb`` (``tensor_sampling_utils``)."""
from . import hdf5_lite, tensor_sampling_utils  # noqa: F401
