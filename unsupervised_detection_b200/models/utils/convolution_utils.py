"""Reference module path models/utils/convolution_utils.py: the layer primitives both networks are built from -- `resize` (:4-24),
`gen_conv` (:26-53), `gen_deconv` (:55-75), `conv` (:77-85), `deconv` (:87-90) -- with the resize functions they take as `func`
and the activations they take as `activation` (implemented in ..functional on libcis_b200 kernels)."""
from ..functional import (LAYER_SUPPORTED, conv, deconv, elu, gen_conv, gen_deconv, identity, leaky_relu, resize,  # noqa: F401
                          resize_bilinear, resize_nearest_neighbor)
