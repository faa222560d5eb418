"""Reference module path models/PWCNet/core_costvol.py: `cost_volume` (:20-40), implemented in ...functional on cis_warp_costvol;
`cost_volume_r` is the same op for search ranges 1..4."""
from ..functional import cost_volume, cost_volume_r  # noqa: F401
