from .trajectory import TRAJ_WIDTH, HandOver, TrajectoryExchange, TrajectorySlab, shard_offset  # noqa: F401
from .unroll import (RECORD_SHAPES, RECORD_WIDTH, hier_slab_records, lambda_returns, sepmc_slab_records, slab_records,  # noqa: F401
                     slab_to_unrolls, unflatten_unroll)
from .rollout import HierRolloutWorker, RolloutWorker, SepmcRolloutWorker, Unroll, UnrollExchange, pack_learner_seat  # noqa: F401
