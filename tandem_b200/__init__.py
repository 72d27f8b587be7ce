"""tandem_b200: H100-native (sm_90a) implementation of TANDEM's dense per-frame hot path behind the
libdr call surface (DrMvsnet / DrFusion / CudaCoarseTracker).  Python here is only the host-side mirror
of those classes over the C ABI in include/tandem_b200.h; all compute is in libtandem_b200.so."""
from ._lib import TandemError, lib  # noqa: F401
from .mvsnet import DrMvsnet, DrMvsnetOutput, default_weights  # noqa: F401
from .fusion import DrFusion, DrFusionOptions  # noqa: F401
from .immature import ImmaturePoints, TRACE_DEFAULTS  # noqa: F401
from .active import ActivePoints, LINEARIZE_DEFAULTS  # noqa: F401
from .pixel_selector import PixelSelector, SELECT_DEFAULTS  # noqa: F401
from .undistort import Undistorter  # noqa: F401
from .tracker import (CudaCoarseTracker, ImagePyramid, set_coarse_tracking_ref, set_coarse_tracking_ref_nodia,  # noqa: F401
                      track_new_coarse, track_pyramid)
