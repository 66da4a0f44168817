"""Dataset registry (scripts/train.py:125 picks `dataset.<DATASET.DATASET>`): the reference's
`h36m` and `mpii_integral` (reference lib/dataset/__init__.py), plus `synthetic_h36m`, which needs
no image data.  Indexed in a DataLoader worker, h36m / mpii_integral return deferred samples;
`assemble_batch` builds such a collated batch on the device (lib/dataset/deferred.py)."""
from .synthetic import SyntheticH36M as synthetic_h36m
from .h36m import H36M_Integral as h36m
from .mpii_integral import MPIIDataset as mpii_integral
from .deferred import assemble_batch, is_deferred
