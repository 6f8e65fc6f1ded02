from .trajectory import TRAJ_WIDTH, TrajectoryExchange, TrajectorySlab, shard_offset  # noqa: F401
from .unroll import (RECORD_SHAPES, RECORD_WIDTH, hier_slab_records, lambda_returns, sepmc_slab_records, slab_records,  # noqa: F401
                     slab_to_unrolls, unflatten_unroll)
from .rollout import RolloutWorker  # noqa: F401
from .hier_rollout import HierRolloutWorker, HierUnroll  # noqa: F401
from .sepmc_rollout import SepmcRolloutWorker, SepmcUnroll  # noqa: F401
