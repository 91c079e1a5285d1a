"""sdfstudio_b200 -- H100-native drop-in for sdfstudio's per-ray SDF volume-rendering hot path.

Host side mirrors the reference's plug points (SURVEY.md section 8b):
  encoding.Encoding            <- tinycudann.Encoding (HashGrid)        nerfstudio/fields/sdf_field.py:230-241
  sdf_field.SDFField           <- nerfstudio.fields.sdf_field.SDFField
  ray_samplers.*               <- nerfstudio.model_components.ray_samplers
  renderers.*                  <- nerfstudio.model_components.renderers
  rays.*                       <- nerfstudio.cameras.rays (containers + alpha/density -> weights)
All arithmetic runs in libsdfb200.so (CUDA, sm_90a) behind the C ABI of include/sdfb200.h.  No CPU / PyTorch fallback.
"""
from . import _lib  # noqa: F401
from . import cameras, meshing  # noqa: F401
from .density_fields import HashMLPDensityField  # noqa: F401
from .encoding import Encoding, HashEncoding  # noqa: F401
from .field_heads import FieldHeadNames  # noqa: F401
from .rays import Frustums, RayBundle, RaySamples  # noqa: F401
from .ray_samplers import (  # noqa: F401
    ErrorBoundedSampler, LinearDisparitySampler, LogSampler, NeuSSampler, PDFSampler, ProposalNetworkSampler, Sampler, SpacedSampler,
    SqrtSampler, UniformLinDispPiecewiseSampler, UniformSampler, UniSurfSampler,
)
from .renderers import AccumulationRenderer, DepthRenderer, RGBRenderer, SemanticRenderer, render_all, render_from_alphas  # noqa: F401
from .scene_colliders import AABBBoxCollider, NearFarCollider, SceneCollider, SphereCollider  # noqa: F401
from .surface_model import SurfaceRenderer  # noqa: F401
from .spatial_distortions import SceneContraction  # noqa: F401
from .sdf_field import LaplaceDensity, SDFField, SDFFieldConfig, SingleVarianceNetwork  # noqa: F401

__version__ = "0.1.0"
