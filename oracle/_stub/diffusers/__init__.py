"""Minimal stand-in for the `diffusers` mixins the reference imports (edm_unet.py:4-6, dpmsolver.py:23-25).

Test infrastructure only: lets tests/golden/make_golden.py import the UNMODIFIED reference checkout in this
container to generate golden vectors.  It contains no arithmetic.  Never imported by the product.
"""
from .configuration_utils import ConfigMixin, register_to_config  # noqa: F401
