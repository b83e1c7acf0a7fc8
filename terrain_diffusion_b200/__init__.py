"""terrain_diffusion_b200: H100-native (sm_90a) InfiniteDiffusion sampling hot path behind the reference's
terrain_diffusion.models / .scheduler / .inference surface.  See DESIGN.md."""
__version__ = "0.1.0"
