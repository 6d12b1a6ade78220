"""Exception types mirroring the Julia exceptions the reference throws on this path."""


class ArgumentError(ValueError):
    """Julia ArgumentError (e.g. src/dspbase.jl:28-33, src/periodograms.jl:396)."""


class DomainError(ValueError):
    """Julia DomainError (e.g. src/periodograms.jl:44-45, 397, 565)."""


class InexactError(ValueError):
    """Julia InexactError (a value that the destination eltype cannot hold, e.g. a complex sample in a real filter state)."""


class DimensionMismatch(ValueError):
    """Julia DimensionMismatch (e.g. src/periodograms.jl:255, 735-737)."""


class BoundsError(IndexError):
    """Julia BoundsError (e.g. levinson(r, p) with p >= length(r), src/lpc.jl:122-146)."""
