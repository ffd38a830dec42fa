"""lcp_physics_b200 -- H100-native batched LCP contact solver behind the
`lcp_physics` API (LCPFunction / PdipmEngine). See DESIGN.md."""
from .lcp import LCPFunction, solve_forward, solve_backward, solve_backward_batched, solve_jvp_batched  # noqa: F401

__all__ = ["LCPFunction", "solve_forward", "solve_backward", "solve_backward_batched", "solve_jvp_batched"]
# fused engine path (contact list in, solution out): lcp_physics_b200.engines.engine_solve / B200PdipmEngine
