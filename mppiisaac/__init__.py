"""Import-path shim: lets code written against the reference (`from mppiisaac.planner.mppi_isaac import
MPPIisaacPlanner`, ...) run on the H100 rollout path unchanged.  Everything resolves to `mppi_isaac_b200`."""
