"""mppi_isaac_b200 -- H100-native MPPI-with-simulated-rollouts hot path (drop-in for tud-airlab/mppi-isaac's
``MPPIisaacPlanner`` rollout path).  The compute backend is the sm_90a CUDA library ``libmppib.so``
(C ABI: ``include/mppib.h``); there is no CPU fallback."""
from .planner.mppi_isaac import MPPIisaacPlanner  # noqa: F401
from .planner.rollout_sim import RolloutSim  # noqa: F401
from .utils.config_store import (ActorWrapper, ExampleConfig, IsaacGymConfig, MPPIConfig, load_config,  # noqa: F401
                                 load_isaacgym_config)

__all__ = ["MPPIisaacPlanner", "RolloutSim", "ExampleConfig", "MPPIConfig", "IsaacGymConfig", "ActorWrapper",
           "load_config", "load_isaacgym_config"]
