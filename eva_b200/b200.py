"""Drop-in for the reference's ``eva.seal`` submodule: generate_keys and the
public / secret contexts, executing on the GPU (H100) through the C-ABI."""
from ._eva_b200._b200 import (B200Public, B200Secret, B200Server, B200Valuation, context_from_raw_keys,  # noqa: F401
                              create_coeff_modulus, generate_keys, public_from_raw, secret_from_raw)
