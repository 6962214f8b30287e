"""onepose_b200 -- H100-native (sm_90a) GATsSPG 2D-3D matcher, drop-in for the reference's
``GATsSuperGlue`` forward, plus the rows either side of it (SuperPoint extractor, per-object feature
construction, RANSAC-PnP, the grey frames of colour camera frames, the pose-guided crop of the next frame, an annotated scan's poses and colour crops, the PNG files of frames and crops, an object's SfM post-processing, detection by 2D-2D matching, the tracker's optical-flow step and its flow-only tracking).  The CUDA library is loaded lazily by the modules; importing this
package on a machine without the built library works, constructing a matcher / extractor does not."""
from .matcher import GATsSuperGlue, LitModelGATsSPG  # noqa: F401
from .extractor import SuperPoint  # noqa: F401
from .frames import grey_frames  # noqa: F401
from . import crop, detect, features3d, flow, frames, png, pnp, scan, sfm, synthetic, track  # noqa: F401

__all__ = ["GATsSuperGlue", "LitModelGATsSPG", "SuperPoint", "grey_frames", "crop", "detect", "features3d", "flow", "frames", "png", "pnp", "scan", "sfm", "synthetic", "track"]
