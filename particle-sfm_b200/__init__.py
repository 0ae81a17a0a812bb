"""H100-native ParticleSfM optimisation hot paths (HP1 path-consistency trajectory
optimiser, HP2 global bundle adjustment).  See DESIGN.md.

The CUDA library is loaded lazily (first use); there is no CPU fallback: without the
built extension or without a CUDA device every compute call raises."""
__version__ = "0.1.0"


def device_count():
    from . import _lib
    return int(_lib.lib().psfm_device_count())


def launch_count():
    from . import _lib
    return int(_lib.lib().psfm_launch_count())
