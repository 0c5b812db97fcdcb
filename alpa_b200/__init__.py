"""alpa_b200: a H100-native auto-parallel training and serving framework with the capabilities of
alpa-projects/alpa (reference public surface: alpa/__init__.py:22-51)."""
from alpa_b200.version import __version__  # noqa: F401
from alpa_b200.global_env import global_config  # noqa: F401
from alpa_b200.api import (init, shutdown, parallelize, grad, value_and_grad, clear_executable_cache,  # noqa: F401
                           ParallelizedFunc, set_seed)
from alpa_b200.sharding import ShardingSpec, LogicalDeviceMesh  # noqa: F401
from alpa_b200.device_mesh import (DeviceCluster, PhysicalDeviceMesh, LocalPhysicalDeviceMesh,  # noqa: F401
                                   DistributedPhysicalDeviceMesh, VirtualPhysicalMesh, PhysicalDeviceMeshGroup,
                                   DistributedArray, ReplicatedDistributedArray, prefetch,
                                   get_global_cluster, get_global_physical_mesh, get_global_virtual_physical_mesh,
                                   set_global_virtual_physical_mesh, get_global_num_devices)
from alpa_b200.parallel.shard.auto_sharding import AutoShardingOption  # noqa: F401
from alpa_b200.parallel_method import (ShardParallel, DataParallel, Zero2Parallel, Zero3Parallel,  # noqa: F401
                                       PipeshardParallel, CreateStateParallel, FollowParallel,
                                       LocalPipelineParallel, get_3d_parallel_method)
from alpa_b200.parallel_plan import plan_to_method  # noqa: F401
from alpa_b200.parallel.pipeline.primitive_def import mark_pipeline_boundary, mark_remat_boundary  # noqa: F401
from alpa_b200.parallel.pipeline.layer_construction import (AutoLayerOption, ManualLayerOption,  # noqa: F401
                                                            FollowLayerOption, manual_remat, automatic_remat,
                                                            automatic_layer_construction)
from alpa_b200.parallel.pipeline.stage_construction import (AutoStageOption, ManualStageOption,  # noqa: F401
                                                            UniformStageOption)
from alpa_b200.parallel.shard.manual_sharding import ManualShardingOption, PartitionSpec  # noqa: F401
from alpa_b200.timer import timers  # noqa: F401
from alpa_b200.data_loader import DataLoader, MeshDriverDataLoader  # noqa: F401
from alpa_b200.serialization import save_checkpoint, restore_checkpoint  # noqa: F401
from alpa_b200 import collective  # noqa: F401  (named-group collective API, reference: alpa.collective)
# ---- module-level names the reference exposes as `alpa.<module>` (alpa/__init__.py)
from alpa_b200.mesh_profiling import ProfilingResultDatabase  # noqa: F401
from alpa_b200 import create_state_parallel, follow_parallel, mesh_profiling, util  # noqa: F401,E402
from alpa_b200 import wrapped_graph as wrapped_hlo  # noqa: F401,E402  (fx graphs play the role of HLO modules here)
from alpa_b200.parallel import pipeline as pipeline_parallel  # noqa: F401,E402
from alpa_b200.parallel import shard as shard_parallel  # noqa: F401,E402
from alpa_b200 import monkey_patch  # noqa: F401,E402
