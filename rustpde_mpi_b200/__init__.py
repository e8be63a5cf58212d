"""rustpde_mpi_b200 -- H100-native spectral hot path of rustpde's Navier2D / Navier2DMpi.

Host-side mirror of the reference's Space / Field / Solve / Integrate surface over the C ABI of
``include/b200pde.h`` (``libb200pde.so``: hand-written sm_90a kernels).  No CPU fallback."""
from .api import (  # noqa: F401
    Context, Space2, Field2, DeviceArray, HholtzAdi, Hholtz, Poisson, Navier2D, SwiftHohenberg2D, integrate,
    chebyshev, cheb_dirichlet, cheb_neumann, cheb_dirichlet_neumann, fourier_r2c, fourier_c2c, poisson_eig, hholtz_eig,
    CHEBYSHEV, CHEB_DIRICHLET, CHEB_NEUMANN, CHEB_DIRICHLET_NEUMANN, FOURIER_R2C, FOURIER_C2C,
    PHYSICAL, SPECTRAL, ORTHO,
)
from ._lib import B2Error, LIB_PATH  # noqa: F401
