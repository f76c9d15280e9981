"""PyTorch surface of the rasteriser (mirror of ``deodr.pytorch`` for the hot path): the 2D Functions (colour and
textured), and the 3D render, rigidity and hand fitters of the reference's PyTorch front end on the device."""
from .differentiable_renderer_pytorch import (  # noqa: F401
    CudaDifferentiableRender2D,
    CudaDifferentiableRender2DTextured,
    CudaDifferentiableRender2DWithBackground,
    CudaDifferentiableRenderer2DFunc,
    CudaDifferentiableRenderer2DTexturedFunc,
    CudaDifferentiableRenderer2DWithBackgroundFunc,
    CudaRenderCompare2D,
    CudaRenderCompare2DFunc,
    CudaRenderCompare2DTextured,
    CudaRenderCompare2DTexturedFunc,
    TorchDifferentiableRender2D,
    TorchDifferentiableRenderer2DFunc,
)
from .mesh_fitter_pytorch import MeshDepthFitter, MeshRGBFitterWithPose  # noqa: F401
from .scene3d_pytorch import (  # noqa: F401
    CameraPytorch,
    ColoredTriMeshPytorch,
    LaplacianRigidEnergyPytorch,
    LinearBlendSkinningFunc,
    LitVertexColorsFunc,
    LoopSubdivisionFunc,
    PhongShadeFunc,
    PoseFunc,
    ProjectPointsFunc,
    RenderMesh2DFunc,
    RenderMesh2DTexturedFunc,
    RigidEnergyFunc,
    Scene3DPytorch,
    SelfCollisionEnergyFunc,
    SelfCollisionEnergyPytorch,
    VertexNormalsFunc,
)
