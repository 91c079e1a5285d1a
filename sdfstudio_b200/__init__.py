"""sdfstudio_b200 -- H100-native drop-in for sdfstudio's per-ray SDF volume-rendering hot path.

Host side mirrors the reference's plug points (SURVEY.md section 8b):
  encoding.Encoding            <- tinycudann.Encoding (HashGrid)        nerfstudio/fields/sdf_field.py:230-241
  sdf_field.SDFField           <- nerfstudio.fields.sdf_field.SDFField
  nerfacto_field.TCNNNerfactoField <- nerfstudio.fields.nerfacto_field.TCNNNerfactoField (background_model="grid")
  nerf_field.NeRFField         <- nerfstudio.fields.vanilla_nerf_field.NeRFField (background_model="mlp")
  ray_samplers.*               <- nerfstudio.model_components.ray_samplers
  packed.*                     <- nerfacc 0.3.5 render_weight_from_alpha / accumulate_along_rays (neus-acc)
  renderers.*                  <- nerfstudio.model_components.renderers
  losses.*                     <- nerfstudio.model_components.losses (the interlevel losses of the proposal networks)
  rays.*                       <- nerfstudio.cameras.rays (containers + alpha/density -> weights)
  tsdf.*                       <- nerfstudio.exporter.tsdf_utils (TSDF fusion and the ns-export tsdf mesh)
  pointcloud.*                 <- nerfstudio.exporter.exporter_utils.generate_point_cloud (the ns-export pointcloud cloud)
  poisson.*                    <- open3d's create_from_point_cloud_poisson as ns-export poisson calls it (the Poisson mesh)
  render_mesh.*                <- scripts/render_mesh.py (ns-render-mesh) and nerfstudio.cameras.camera_paths
All arithmetic runs in libsdfb200.so (CUDA, sm_90a) behind the C ABI of include/sdfb200.h.  No CPU / PyTorch fallback.
"""
from . import _lib  # noqa: F401
from . import cameras, losses, meshing, packed, pointcloud, poisson, render_mesh, tsdf  # noqa: F401
from .pointcloud import PointCloud, estimate_normals, generate_point_cloud, point_cloud, remove_statistical_outlier  # noqa: F401
from .poisson import create_from_point_cloud_poisson, poisson_mesh, remove_vertices_by_mask  # noqa: F401
from .render_mesh import render_frames, render_trajectory_video  # noqa: F401  (render_mesh.render_mesh: the module keeps the name)
from .density_fields import HashMLPDensityField  # noqa: F401
from .encoding import Encoding, HashEncoding  # noqa: F401
from .field_heads import FieldHeadNames  # noqa: F401
from .losses import interlevel_loss, interlevel_loss_zip, ray_samples_to_sdist  # noqa: F401
from .nerfacto_field import TCNNNerfactoField  # noqa: F401
from .nerf_field import NeRFEncoding, NeRFField  # noqa: F401
from .rays import Frustums, RayBundle, RaySamples  # noqa: F401
from .ray_samplers import (  # noqa: F401
    ErrorBoundedSampler, LinearDisparitySampler, LogSampler, NeuSAccSampler, NeuSSampler, PDFSampler, ProposalNetworkSampler, Sampler, SpacedSampler,
    SqrtSampler, UniformLinDispPiecewiseSampler, UniformSampler, UniSurfSampler,
)
from .renderers import AccumulationRenderer, DepthRenderer, RGBRenderer, SemanticRenderer, render_all, render_from_alphas  # noqa: F401
from .scene_colliders import AABBBoxCollider, NearFarCollider, SceneCollider, SphereCollider  # noqa: F401
from .surface_model import SurfaceRenderer  # noqa: F401
from .spatial_distortions import SceneContraction  # noqa: F401
from .sdf_field import LaplaceDensity, SDFField, SDFFieldConfig, SingleVarianceNetwork  # noqa: F401

__version__ = "0.1.0"
