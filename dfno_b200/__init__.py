"""dfno_b200 -- a Hopper-native model-parallel Fourier Neural Operator framework.

Public namespace (same names as slimgroup/dfno, reference ``dfno/__init__.py:1-3``):
``DistributedFNO``, ``DistributedFNONd``, ``DistributedFNOBlock``, ``BroadcastedLinear``,
``DistributedRelativeLpLoss``, ``DistributedMSELoss``, ``create_standard_partitions``,
``create_root_partition``, ``compute_distribution_info``, ``get_env``, ``alphabet``,
``unit_guassian_normalize`` / ``unit_gaussian_denormalize`` -- plus the partition /
Repartition / Broadcast / SumReduce layer the reference gets from DistDL.
"""
__version__ = "0.1.0"

from .parallel import *           # noqa: F401,F403
from .utils import *              # noqa: F401,F403
from .models import *             # noqa: F401,F403
from .trainer import InferenceSession, Trainer      # noqa: E402,F401
from .data import *               # noqa: E402,F401,F403
from .models.fused import FusedDistributedFNO, FusedAdam   # noqa: E402,F401
