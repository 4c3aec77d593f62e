"""kaolin.render.lighting drop-ins: spherical-Gaussian diffuse and specular, and SH9 diffuse shading on
sm_90a kernels."""
from .sg import (unbatched_reduced_sg_inner_product, sg_irradiance_inner_product,  # noqa: F401
                 sg_diffuse_inner_product, sg_diffuse_fitted, sg_distribution_term, sg_warp_distribution,
                 fresnel, sg_warp_specular_term)
from .sh import project_onto_sh9, sh9_irradiance, sh9_diffuse  # noqa: F401

__all__ = ["unbatched_reduced_sg_inner_product", "sg_irradiance_inner_product", "sg_diffuse_inner_product",
           "sg_diffuse_fitted", "sg_distribution_term", "sg_warp_distribution", "fresnel", "sg_warp_specular_term",
           "project_onto_sh9", "sh9_irradiance", "sh9_diffuse"]
