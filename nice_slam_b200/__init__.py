"""nice_slam_b200 -- H100 (sm_90a) render-and-backprop path for NICE-SLAM (drop-in for src/utils/Renderer.py).

Public surface:
    FusedRenderer   mirror of the reference's Renderer (render_batch_ray / eval_points / render_img)
    NICEDecoders    parameter container with the reference's state_dict keys
    FusedMapper     one Mapper.optimize_map call on the fused path (mapping.py)
    FusedSLAM       a whole RGB-D sequence on the fused path, NICE_SLAM.run under strict sync (slam.py); ate_rmse
    FusedMesher     Mesher.get_mesh of a fused run's grids, decoders and keyframes on the GPU (mesh.py)
    recon           eval_recon.py's 3D reconstruction metric on the GPU: nice_slam_b200.recon.eval_recon, or
                    python -m nice_slam_b200.recon --rec_mesh A --gt_mesh B -3d (not imported here, so that -m runs it cleanly)
    cull            cull_mesh.py's ground-truth culling on the GPU: nice_slam_b200.cull.cull_mesh, or
                    python -m nice_slam_b200.cull --input_mesh A --traj traj.txt --output_mesh B (not imported here either)
    build_scene     NICE_SLAM.__init__'s initial state (bound, grids, pretrained decoders, renderer) from a config (scene.py)
    FrameReader     the reference's dataset readers, frames prepared on the GPU (datasets.py)
    run             run.py's counterpart: python -m nice_slam_b200.run CONFIG (not imported here)
    to_channels_last, lib (ctypes handle of libnsb.so), get_option / set_option (library options, e.g. "deterministic")
"""
from ._lib import lib, LIB_PATH, get_option, set_option   # noqa: F401
from .decoders import NICEDecoders                     # noqa: F401
from .renderer import FusedRenderer, to_channels_last  # noqa: F401
from .mapping import FusedMapper                       # noqa: F401
from .mesh import FusedMesher                          # noqa: F401
from .slam import FusedSLAM, ate_rmse                  # noqa: F401
from .scene import build_scene                         # noqa: F401
from .datasets import FrameReader                      # noqa: F401

__all__ = ["FusedRenderer", "FusedMapper", "FusedSLAM", "FusedMesher", "ate_rmse", "build_scene", "FrameReader", "NICEDecoders", "to_channels_last", "lib", "LIB_PATH", "get_option", "set_option"]
