"""prysm_b200 -- H100-native (Hopper, sm_90a) engine for the prysm propagation hot path.

Mirrors the reference's module layout for the path only:
    prysm_b200.propagation  <-> prysm.propagation   (focus/unfocus/angular_spectrum/executors/Wavefront)
    prysm_b200.fttools      <-> prysm.fttools       (pad2d/crop_center/MDFT/CZT/FFTDFT)
    prysm_b200.otf / .psf   <-> prysm.otf / prysm.psf (transform_psf, mtf/ptf/otf, centroid)
    prysm_b200.polynomials  <-> prysm.polynomials.sum_of_2d_modes, jacobi / zernike and the Forbes names of qpoly
    prysm_b200.qpoly        <-> prysm.polynomials.qpoly (Q-bfs, Q-con, 2D-Q: bases, derivatives and sag / slope sums)
    prysm_b200.conf         <-> prysm.conf          (config.precision)
    prysm_b200.mathops      <-> prysm.mathops       (set_backend_to_b200 / set_backend_to_defaults)
    prysm_b200.coronagraph  <-> prysm.propagation.coronagraph (re-exported by .propagation like the reference)
    prysm_b200.coordinates / .geometry  <-> prysm.coordinates.make_xy_grid / cart_to_polar, prysm.geometry.circle / antialias
    prysm_b200.convolution  <-> prysm.convolution (conv, apply_transfer_functions)
    prysm_b200.detector     <-> prysm.detector (Detector.expose with shot and read noise, apply_lut, pixel, bindown, tile,
                            pixel_ft, olpf_ft)
    prysm_b200.bayer        <-> prysm.bayer (white balance, composite / decomposite, deinterlace and Malvar demosaicing,
                            assemble_superresolved)
    prysm_b200.dm           <-> prysm.x.dm (DM: render / render_adjoint; coordinates.warp is its spline warp)
    prysm_b200.segmented    <-> prysm.segmented (CompositeHexagonalAperture: rasterise, compose_opd and its adjoint)
    prysm_b200.polarization <-> prysm.x.polarization (Jones constructors, products, Mueller / Pauli, jones_adapter)
    prysm_b200.fibers / .sri / .pdi / .psi  <-> prysm.x.fibers / sri / pdi / psi (LP modes and coupling, the SRI and
                            PS/PDI forward models, PSI phase reconstruction)
    prysm_b200.shack_hartmann <-> prysm.x.shack_hartmann (the lenslet screen in one launch; spot centroids and the
                            ShackHartmann sensor with a modal reconstructor are engine extensions)
    prysm_b200.thinfilm / .coatings  <-> prysm.thinfilm.multilayer_stack_rt, prysm.x.coatings (stack_rt, RTA, internal
                            and depth fields, forward_eval with thickness and index gradients)
    prysm_b200.util / .interferogram  <-> prysm.util statistics, prysm.interferogram (NaN-aware statistics, masked least
                            squares, PSD and windows, band-limited RMS, filters, slopes and Interferogram's metrology)
    prysm_b200.graphs       CUDA-graph capture of launch-bound compositions (no reference counterpart)
Every array operation is a call into libprysm_b200.so (hand-written sm_90a CUDA behind the C ABI
of include/prysm_b200.h).  Importing this package without the built library raises ImportError.
"""
from . import _capi  # noqa: F401  (fails loudly if the CUDA library is missing)
from .conf import config  # noqa: F401
from . import fttools, propagation, coronagraph, otf, psf, polynomials, polychromatic, mathops, graphs  # noqa: F401
from . import coordinates, geometry, convolution, detector, dm, segmented, polarization  # noqa: F401
from . import fibers, sri, pdi, psi, bayer, shack_hartmann, qpoly, thinfilm, coatings, util, interferogram  # noqa: F401
from ._capi import B200Error  # noqa: F401
from .propagation import Wavefront  # noqa: F401
from ._ops import asdevice, asnumpy, set_device  # noqa: F401

__version__ = '0.1.0'
