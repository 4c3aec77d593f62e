from .mesh import (RenderPass, render_mesh, mesh_rasterize_interpolate_cuda,  # noqa: F401
                   texture_sample_materials, sg_shade)

__all__ = ["RenderPass", "render_mesh", "mesh_rasterize_interpolate_cuda", "texture_sample_materials", "sg_shade"]
