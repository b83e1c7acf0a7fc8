"""Mirror of terrain_diffusion.models (reference: terrain_diffusion/models/)."""
from .edm_unet import EDMUnet2D  # noqa: F401
from .edm_autoencoder import EDMAutoencoder  # noqa: F401
