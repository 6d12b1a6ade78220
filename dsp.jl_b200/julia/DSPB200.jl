# DSPB200.jl -- Julia glue over libdspb200.so (include/dspb200.h).
#
# Host code stays in Julia (BASELINE.json north_star): this module re-exposes the reference's call signatures for
# the hot path and `ccall`s the C ABI.  Host-side scalar logic (window values, nextfastfft, default resampling
# taps, result structs, argument validation and exception types) is taken from DSP.jl itself, so behaviour outside
# the kernels is the reference's by construction.  Array eltypes the GPU path does not cover (integers, Float16, IIR,
# arrays of rank > 3) are not given methods here and keep dispatching to DSP.jl.
#
# NOTE: the build container has no Julia toolchain, so this file is exercised only by reading; the Python mirror
# (`dsp.jl_b200/*.py`, same ABI, same call order) is what the test-suite drives.  See INTEGRATION.md.
module DSPB200

import DSP
using DSP: Periodograms, Filters, Util

const libdspb200 = get(ENV, "DSPB200_LIB", joinpath(@__DIR__, "..", "libdspb200.so"))

const GPUReal = Union{Float32,Float64}
const GPUNumber = Union{Float32,Float64,ComplexF32,ComplexF64}

dtype_code(::Type{Float32}) = Cint(0)
dtype_code(::Type{Float64}) = Cint(1)
dtype_code(::Type{ComplexF32}) = Cint(2)
dtype_code(::Type{ComplexF64}) = Cint(3)

struct DSPB200Error <: Exception
    code::Cint
    msg::String
end

function check(rc::Cint)
    rc == 0 && return nothing
    throw(DSPB200Error(rc, unsafe_string(ccall((:dspb200_last_error, libdspb200), Cstring, ()))))
end

# ------------------------------------------------------------------------------------------------ plan handles
mutable struct Plan
    ptr::Ptr{Cvoid}
    destroy::Symbol
    function Plan(ptr::Ptr{Cvoid}, destroy::Symbol)
        p = new(ptr, destroy)
        finalizer(close!, p)
        return p
    end
end

function close!(p::Plan)
    if p.ptr != C_NULL
        if p.destroy === :dspb200_os_plan_destroy
            ccall((:dspb200_os_plan_destroy, libdspb200), Cint, (Ptr{Cvoid},), p.ptr)
        elseif p.destroy === :dspb200_spec_plan_destroy
            ccall((:dspb200_spec_plan_destroy, libdspb200), Cint, (Ptr{Cvoid},), p.ptr)
        elseif p.destroy === :dspb200_fir_plan_destroy
            ccall((:dspb200_fir_plan_destroy, libdspb200), Cint, (Ptr{Cvoid},), p.ptr)
        else
            ccall((:dspb200_resample_plan_destroy, libdspb200), Cint, (Ptr{Cvoid},), p.ptr)
        end
        p.ptr = C_NULL
    end
    return nothing
end

function os_plan(v::Vector{T}, nfft::Integer=0) where {T<:GPUNumber}
    h = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve v check(ccall((:dspb200_os_plan_create, libdspb200), Cint,
        (Ref{Ptr{Cvoid}}, Cint, Ptr{Cvoid}, Int64, Int64), h, dtype_code(T), v, length(v), nfft))
    return Plan(h[], :dspb200_os_plan_destroy)
end

function spec_plan(::Type{T}, n, noverlap, nfft, onesided::Bool, win::Union{Nothing,Vector{Float64}}) where {T<:GPUNumber}
    h = Ref{Ptr{Cvoid}}(C_NULL)
    wptr = win === nothing ? Ptr{Cdouble}(C_NULL) : pointer(win)
    GC.@preserve win check(ccall((:dspb200_spec_plan_create, libdspb200), Cint,
        (Ref{Ptr{Cvoid}}, Cint, Int64, Int64, Int64, Cint, Ptr{Cdouble}), h, dtype_code(T), n, noverlap, nfft, onesided, wptr))
    return Plan(h[], :dspb200_spec_plan_destroy)
end

# ------------------------------------------------------------------------------------------------ filt(b, a, x)
# DSP.filt(b, a, x) / DSP.filt!(out, b, a, x): src/dspbase.jl:14-15, 26-66 (FIR: length(a) == 1)
function filt!(out::Array{T}, b::Union{AbstractVector,Number}, a::Union{AbstractVector,Number}, x::Array{T}) where {T<:GPUNumber}
    isempty(b) && throw(ArgumentError("filter vector b must be non-empty"))
    isempty(a) && throw(ArgumentError("filter vector a must be non-empty"))
    a[1] == 0 && throw(ArgumentError("filter vector a[1] must be nonzero"))
    size(x) != size(out) && throw(ArgumentError("output size $(size(out)) must match input size $(size(x))"))
    length(a) == 1 || return DSP.filt!(out, b, a, x)            # IIR stays on the reference path
    iszero(size(x, 1)) && return out
    bT = convert(Vector{T}, (b isa Number ? [b] : collect(b)) ./ a[1])         # a scalar b is a one-tap filter (:14)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve bT check(ccall((:dspb200_fir_plan_create, libdspb200), Cint,
        (Ref{Ptr{Cvoid}}, Cint, Ptr{Cvoid}, Int64), h, dtype_code(T), bT, length(bT)))
    plan = Plan(h[], :dspb200_fir_plan_destroy)
    nx = size(x, 1)
    GC.@preserve x out check(ccall((:dspb200_fir_exec, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ptr{Cvoid}), plan.ptr, x, nx, length(x) ÷ nx, out))
    close!(plan)
    return out
end
filt(b, a, x::Array{T}) where {T<:GPUNumber} = filt!(similar(x), b, a, x)

# DSP.filt!(out, f::DF2TFilter{<:PolynomialRatio}, x): src/Filters/filt.jl:157-181, FIR coefficient sets whose state and
# signal share a GPU eltype the coefficients promote into (then the reference computes every muladd in that eltype).
# The state is staged through the plan, so it is passed as both si_in and si_out and updated in place as the reference does.
function filt!(out::Array{S,N}, f::Filters.DF2TFilter{<:Filters.PolynomialRatio,Array{S,N}}, x::Array{S,N}) where {S<:GPUNumber,N}
    size(x) != size(out) && throw(ArgumentError("out size must match x"))
    si = f.state
    size(x)[2:end] != size(si)[2:end] && throw(ArgumentError("state size must match x"))
    b = Filters.coefb(f.coef)
    (length(Filters.coefa(f.coef)) == 1 && promote_type(eltype(b), S) == S) || return DSP.filt!(out, f, x)
    iszero(length(x)) && return out
    bT = convert(Vector{S}, b)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve bT check(ccall((:dspb200_fir_plan_create, libdspb200), Cint,
        (Ref{Ptr{Cvoid}}, Cint, Ptr{Cvoid}, Int64), h, dtype_code(S), bT, length(bT)))
    plan = Plan(h[], :dspb200_fir_plan_destroy)
    nx = size(x, 1)
    GC.@preserve x out si check(ccall((:dspb200_fir_exec_state, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), plan.ptr, x, nx, length(x) ÷ nx, si, si, out))
    close!(plan)
    return out
end
filt(f::Filters.DF2TFilter{<:Filters.PolynomialRatio,Array{S,N}}, x::Array{S,N}) where {S<:GPUNumber,N} = filt!(similar(x), f, x)

# ------------------------------------------------------------------------------------------------ fftfilt / filt(h, x)
# DSP.Filters.fftfilt(b, x[, nfft]) / fftfilt!: src/Filters/filt.jl:458-521
function fftfilt!(out::Array{T}, b::Vector{T}, x::Array{T}, nfft::Integer=0) where {T<:GPUReal}
    size(out) == size(x) || throw(ArgumentError("out and x must be the same size"))
    isempty(x) && return out
    plan = os_plan(b, nfft)
    nx = size(x, 1)
    GC.@preserve x out check(ccall((:dspb200_os_exec, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ptr{Cvoid}, Int64), plan.ptr, x, nx, length(x) ÷ nx, out, nx))
    close!(plan)
    return out
end
fftfilt(b::Vector{T}, x::Array{T}, nfft::Integer=0) where {T<:GPUReal} = fftfilt!(similar(x), b, x, nfft)
# fftfilt!(out, f::DF2TFilter{<:PolynomialRatio}, x) (an extension, not in DSP.jl): filt!(out, f, x) computed by overlap-save,
# with the same state (updated in place through the host form's staging), within FFT rounding of filt!.  FIR coefficients
# of the state's GPU eltype, as for filt! above; the block transform is the library's choice.
function fftfilt!(out::Array{S,N}, f::Filters.DF2TFilter{<:Filters.PolynomialRatio,Array{S,N}}, x::Array{S,N}) where {S<:GPUNumber,N}
    size(x) != size(out) && throw(ArgumentError("out size must match x"))
    si = f.state
    size(x)[2:end] != size(si)[2:end] && throw(ArgumentError("state size must match x"))
    b = Filters.coefb(f.coef)
    length(Filters.coefa(f.coef)) == 1 || throw(ArgumentError("fftfilt! takes FIR coefficients (length(coefa) == 1)"))
    promote_type(eltype(b), S) == S || throw(ArgumentError("the coefficients must promote into the state's eltype $S"))
    iszero(length(x)) && return out
    plan = os_plan(convert(Vector{S}, b), 0)
    nx = size(x, 1)
    GC.@preserve x out si check(ccall((:dspb200_os_exec_state, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), plan.ptr, x, nx, length(x) ÷ nx, si, si, out))
    close!(plan)
    return out
end
fftfilt(f::Filters.DF2TFilter{<:Filters.PolynomialRatio,Array{S,N}}, x::Array{S,N}) where {S<:GPUNumber,N} =
    fftfilt!(similar(x), f, x)
tdfilt(h::Vector{T}, x::Array{T}) where {T<:GPUNumber} = filt(h, one(T), x)            # src/Filters/filt.jl:431-433
# filt(h, x): src/Filters/filt.jl:525-555 (Real x Real with more than 66 taps -> overlap-save)
filt(h::Vector{T}, x::Array{T}) where {T<:GPUReal} =
    length(h) > DSP.SMALL_FILT_CUTOFF ? fftfilt(h, x) : tdfilt(h, x)
filt(h::Vector{T}, x::Array{T}) where {T<:Complex{<:GPUReal}} = tdfilt(h, x)

# ------------------------------------------------------------------------------------------------ conv
# DSP.conv(u, v; algorithm) / conv!: src/dspbase.jl:709-792 (1-D, FFTTypes)
function conv!(out::Vector{T}, u::Vector{T}, v::Vector{T}; algorithm=:auto) where {T<:GPUNumber}
    nres = length(u) + length(v) - 1
    length(out) >= max(nres, 0) || throw(ArgumentError("out is too small"))
    algorithm === :auto && (algorithm = :fast)
    algorithm === :fast && (algorithm = length(u) * length(v) < 2^16 ? :direct : :fft)
    if isempty(u) || isempty(v)
        fill!(out, zero(T)); return out
    end
    small, large = length(u) >= length(v) ? (v, u) : (u, v)
    if algorithm === :fft
        algorithm = DSP.optimalfftfiltlength(length(small), length(large)) < nres ? :fft_overlapsave : :fft_simple
    end
    if algorithm === :direct
        GC.@preserve u v out check(ccall((:dspb200_conv_direct_exec, libdspb200), Cint,
            (Cint, Ptr{Cvoid}, Int64, Ptr{Cvoid}, Int64, Ptr{Cvoid}), dtype_code(T), u, length(u), v, length(v), out))
    elseif algorithm === :fft_simple
        GC.@preserve u v out check(ccall((:dspb200_conv_fft_exec, libdspb200), Cint,
            (Cint, Ptr{Cvoid}, Int64, Ptr{Cvoid}, Int64, Int64, Ptr{Cvoid}),
            dtype_code(T), u, length(u), v, length(v), DSP.nextfastfft(nres), out))
    elseif algorithm === :fft_overlapsave
        plan = os_plan(small)
        GC.@preserve large out check(ccall((:dspb200_os_exec, libdspb200), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ptr{Cvoid}, Int64), plan.ptr, large, length(large), 1, out, nres))
        close!(plan)
    else
        throw(ArgumentError("algorithm must be :auto, :fast, :direct, :fft, :fft_simple, or :fft_overlapsave"))
    end
    out[nres+1:end] .= zero(T)                                  # src/dspbase.jl:733-735
    return out
end
conv(u::Vector{T}, v::Vector{T}; kwargs...) where {T<:GPUNumber} =
    conv!(Vector{T}(undef, max(length(u) + length(v) - 1, 0)), u, v; kwargs...)

# ------------------------------------------------------------------------------------------------ Welch / periodogram
abs2type(::Type{T}) where {T} = DSP.Util.fftabs2type(T)

# DSP.welch_pgram(s, n, noverlap; kw...): src/periodograms.jl:647-649, 746-759
function welch_pgram(s::Vector{T}, n::Int=length(s) >> 3, noverlap::Int=n >> 1; onesided::Bool=T <: Real,
                     nfft::Int=DSP.nextfastfft(n), fs::Real=1,
                     window::Union{Function,AbstractVector,Nothing}=nothing) where {T<:GPUNumber}
    onesided && T <: Complex && throw(ArgumentError("cannot compute one-sided FFT of a complex signal"))
    nfft >= n || throw(DomainError((; nfft, n), "nfft must be >= n"))
    (0 <= noverlap < n) || throw(DomainError((; noverlap, n), "noverlap must be between zero and n"))
    win, norm2 = Periodograms.compute_window(window, n)
    w64 = win === nothing ? nothing : convert(Vector{Float64}, win)
    plan = spec_plan(T, n, noverlap, nfft, onesided, w64)
    k = length(s) >= n ? div(length(s) - n, n - noverlap) + 1 : 0
    out = zeros(abs2type(T), onesided ? (nfft >> 1) + 1 : nfft)
    if k > 0
        GC.@preserve s out check(ccall((:dspb200_welch_exec, libdspb200), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Cdouble, Ptr{Cvoid}), plan.ptr, s, length(s), k * fs * norm2, out))
    end
    close!(plan)
    return Periodograms.Periodogram(out, onesided ? DSP.rfftfreq(nfft, fs) : DSP.fftfreq(nfft, fs))
end

# DSP.WelchConfig / welch_pgram(s, config) / welch_pgram!(out, s, config): src/periodograms.jl:516-587, 702-705, 734-759.
# The config owns the device plan (segmenter + window + FFT), reused across calls like the reference's plan and buffers.
struct GPUWelchConfig{T<:GPUNumber}
    nsamples::Int
    noverlap::Int
    onesided::Bool
    nfft::Int
    fs::Float64
    r::Float64                     # fs * norm2, :568
    freq::AbstractVector
    plan::Plan
end
function WelchConfig(nsamples::Integer, ::Type{T}; n::Int=nsamples >> 3, noverlap::Int=n >> 1, onesided::Bool=T <: Real,
                     nfft::Int=DSP.nextfastfft(n), fs::Real=1,
                     window::Union{Function,AbstractVector,Nothing}=nothing) where {T<:GPUNumber}
    onesided && T <: Complex && throw(ArgumentError("cannot compute one-sided FFT of a complex signal"))   # :564
    nfft >= n || throw(DomainError((; nfft, n), "nfft must be >= n"))                                      # :565
    (0 <= noverlap < n) || throw(DomainError((; noverlap, n), "noverlap must be between zero and n"))
    win, norm2 = Periodograms.compute_window(window, n)
    w64 = win === nothing ? nothing : convert(Vector{Float64}, win)
    GPUWelchConfig{T}(n, noverlap, onesided, nfft, fs, fs * norm2,
                      onesided ? DSP.rfftfreq(nfft, fs) : DSP.fftfreq(nfft, fs), spec_plan(T, n, noverlap, nfft, onesided, w64))
end
WelchConfig(data::AbstractVector{T}; kwargs...) where {T<:GPUNumber} = WelchConfig(length(data), T; kwargs...)

function welch_pgram!(out::Vector, s::Vector{T}, config::GPUWelchConfig{T}) where {T<:GPUNumber}
    length(out) == length(config.freq) ||
        throw(DimensionMismatch("Expected `output` to be of length `length(config.freq)`; got $(length(out)) and $(length(config.freq))"))
    eltype(out) == abs2type(T) ||
        throw(ArgumentError("Eltype of output ($(eltype(out))) doesn't match the expected type: $(abs2type(T))."))
    k = length(s) >= config.nsamples ? div(length(s) - config.nsamples, config.nsamples - config.noverlap) + 1 : 0
    if k == 0
        fill!(out, 0)
    else
        GC.@preserve s out check(ccall((:dspb200_welch_exec, libdspb200), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Cdouble, Ptr{Cvoid}), config.plan.ptr, s, length(s), k * config.r, out))   # r = k fs norm2, :751
    end
    return Periodograms.Periodogram(out, config.freq)
end
welch_pgram(s::Vector{T}, config::GPUWelchConfig{T}) where {T<:GPUNumber} =
    welch_pgram!(Vector{abs2type(T)}(undef, length(config.freq)), s, config)

# Batched Welch: the columns of `s` are independent channels, each Welch-averaged with the same configuration in one launch
# (dspb200_welch_batch_exec).  The reference has no matrix method, so these are not added to the DSP.* overlay below.
function welch_pgram!(out::Matrix, s::Matrix{T}, config::GPUWelchConfig{T}) where {T<:GPUNumber}
    len, nchan = size(s)
    size(out) == (length(config.freq), nchan) ||
        throw(DimensionMismatch("Expected `output` to be of size (length(config.freq), size(s, 2)) = $((length(config.freq), nchan)); got $(size(out))"))
    eltype(out) == abs2type(T) ||
        throw(ArgumentError("Eltype of output ($(eltype(out))) doesn't match the expected type: $(abs2type(T))."))
    k = len >= config.nsamples ? div(len - config.nsamples, config.nsamples - config.noverlap) + 1 : 0
    if k == 0 || nchan == 0
        fill!(out, 0)
    else
        GC.@preserve s out check(ccall((:dspb200_welch_batch_exec, libdspb200), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Cdouble, Ptr{Cvoid}), config.plan.ptr, s, len, nchan, k * config.r, out))
    end
    return Periodograms.Periodogram(out, config.freq)
end
welch_pgram(s::Matrix{T}, config::GPUWelchConfig{T}) where {T<:GPUNumber} =
    welch_pgram!(Matrix{abs2type(T)}(undef, length(config.freq), size(s, 2)), s, config)
function welch_pgram(s::Matrix{T}, n::Int=size(s, 1) >> 3, noverlap::Int=n >> 1; onesided::Bool=T <: Real,
                     nfft::Int=DSP.nextfastfft(n), fs::Real=1,
                     window::Union{Function,AbstractVector,Nothing}=nothing) where {T<:GPUNumber}
    config = WelchConfig(size(s, 1), T; n, noverlap, onesided, nfft, fs, window)
    p = welch_pgram(s, config)
    close!(config.plan)
    return p
end

# welch_pgram(filt(b, x), config) as one pipelined call (dspb200_filt_welch_exec): x is uploaded in chunks that overlap the
# kernels, the filter output never leaves the GPU.  Same values as `welch_pgram(DSP.filt(b, x), config)`.
function filt_welch(b::Vector{T}, x::Vector{T}, config::GPUWelchConfig{T}) where {T<:GPUNumber}
    out = zeros(abs2type(T), length(config.freq))
    k = length(x) >= config.nsamples ? div(length(x) - config.nsamples, config.nsamples - config.noverlap) + 1 : 0
    if k > 0
        osp = os_plan(b)
        GC.@preserve x out check(ccall((:dspb200_filt_welch_exec, libdspb200), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Cdouble, Ptr{Cvoid}), osp.ptr, config.plan.ptr, x, length(x), k * config.r, out))
        close!(osp)
    end
    return Periodograms.Periodogram(out, config.freq)
end

# DSP.periodogram(s; kw...): src/periodograms.jl:393-417 -- the single-segment case
periodogram(s::Vector{T}; onesided::Bool=T <: Real, nfft::Int=DSP.nextfastfft(length(s)), fs::Real=1,
            window::Union{Function,AbstractVector,Nothing}=nothing) where {T<:GPUNumber} =
    welch_pgram(s, length(s), 0; onesided, nfft, fs, window)

# DSP.stft / DSP.spectrogram: src/periodograms.jl:828-897
function stft(s::Vector{T}, n::Int=length(s) >> 3, noverlap::Int=n >> 1, psdonly::Union{Nothing,Periodograms.PSDOnly}=nothing;
              onesided::Bool=T <: Real, nfft::Int=DSP.nextfastfft(n), fs::Real=1,
              window::Union{Function,AbstractVector,Nothing}=nothing) where {T<:GPUNumber}
    onesided && T <: Complex && throw(ArgumentError("cannot compute one-sided FFT of a complex signal"))
    win, norm2 = Periodograms.compute_window(window, n)
    w64 = win === nothing ? nothing : convert(Vector{Float64}, win)
    nfft >= n || throw(DomainError((; nfft, n), "nfft must be >= n"))
    (0 <= noverlap < n) || throw(DomainError((; noverlap, n), "noverlap must be between zero and n"))
    k = length(s) >= n ? div(length(s) - n, n - noverlap) + 1 : 0
    nout = onesided ? (nfft >> 1) + 1 : nfft
    out = zeros(Periodograms.stfttype(T, psdonly), nout, k)
    if k > 0
        plan = spec_plan(T, n, noverlap, nfft, onesided, w64)
        GC.@preserve s out check(ccall((:dspb200_stft_exec, libdspb200), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Cdouble, Cint, Ptr{Cvoid}),
            plan.ptr, s, length(s), 1, fs * norm2, psdonly !== nothing, out))
        close!(plan)
    end
    return out
end

function spectrogram(s::Vector{T}, n::Int=length(s) >> 3, noverlap::Int=n >> 1; onesided::Bool=T <: Real,
                     nfft::Int=DSP.nextfastfft(n), fs::Real=1,
                     window::Union{Function,AbstractVector,Nothing}=nothing) where {T<:GPUNumber}
    out = stft(s, n, noverlap, Periodograms.PSDOnly(); onesided, nfft, fs, window)
    return Periodograms.Spectrogram(out, onesided ? DSP.rfftfreq(nfft, fs) : DSP.fftfreq(nfft, fs),
                                    (n / 2 : n - noverlap : (size(out, 2) - 1) * (n - noverlap) + n / 2) / fs)
end

# Batched spectrogram: the columns of `s` are independent channels (BASELINE config 4: 64 channels in one launch).  Returns the
# nout x k x nchan power array plus the frequency / time axes of the per-vector method.
function spectrogram(s::Matrix{T}, n::Int=size(s, 1) >> 3, noverlap::Int=n >> 1; onesided::Bool=T <: Real,
                     nfft::Int=DSP.nextfastfft(n), fs::Real=1,
                     window::Union{Function,AbstractVector,Nothing}=nothing) where {T<:GPUNumber}
    onesided && T <: Complex && throw(ArgumentError("cannot compute one-sided FFT of a complex signal"))
    win, norm2 = Periodograms.compute_window(window, n)
    w64 = win === nothing ? nothing : convert(Vector{Float64}, win)
    nfft >= n || throw(DomainError((; nfft, n), "nfft must be >= n"))
    (0 <= noverlap < n) || throw(DomainError((; noverlap, n), "noverlap must be between zero and n"))
    len, nchan = size(s)
    k = len >= n ? div(len - n, n - noverlap) + 1 : 0
    nout = onesided ? (nfft >> 1) + 1 : nfft
    out = zeros(abs2type(T), nout, k, nchan)
    if k > 0 && nchan > 0
        plan = spec_plan(T, n, noverlap, nfft, onesided, w64)
        GC.@preserve s out check(ccall((:dspb200_stft_exec, libdspb200), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Cdouble, Cint, Ptr{Cvoid}), plan.ptr, s, len, nchan, fs * norm2, 1, out))
        close!(plan)
    end
    return out, (onesided ? DSP.rfftfreq(nfft, fs) : DSP.fftfreq(nfft, fs)), (n / 2 : n - noverlap : (k - 1) * (n - noverlap) + n / 2) / fs
end

# A multitaper plan of DSP.jl's own MTConfig: the tapers pre-scaled by 1/sqrt(r_t), as ntapers x n rows
function mt_plan(cfg, ::Type{T}, n, noverlap, nfft, onesided) where {T}
    tapers = permutedims(cfg.window ./ sqrt.(reshape(cfg.r, 1, :)))
    h = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve tapers check(ccall((:dspb200_mt_plan_create, libdspb200), Cint,
        (Ref{Ptr{Cvoid}}, Cint, Int64, Int64, Int64, Cint, Ptr{Cdouble}, Int64),
        h, dtype_code(T), n, noverlap, nfft, onesided, tapers, size(tapers, 1)))
    return Plan(h[], :dspb200_spec_plan_destroy)
end

# DSP.mt_pgram(s; fs, nfft, nw, ntapers, window): src/multitaper.jl:259-304 -- tapers / weights / validation from DSP.jl's own
# MTConfig.  A matrix is the extension: every column a channel, power length(freq) x size(s, 2).
function mt_pgram(s::VecOrMat{T}; onesided::Bool=T <: Real, nfft::Int=nextpow(2, size(s, 1)), fs::Real=1, nw::Real=4,
                  ntapers::Int=ceil(Int, 2nw) - 1, window::Union{AbstractMatrix,Nothing}=nothing) where {T<:GPUNumber}
    len, nchan = size(s, 1), size(s, 2)
    cfg = Periodograms.MTConfig{T}(len; fs, nfft, window, nw, ntapers, onesided)
    plan = mt_plan(cfg, T, len, 0, nfft, onesided)
    out = zeros(abs2type(T), length(cfg.freq), nchan)
    GC.@preserve s out check(ccall((:dspb200_mt_pgram_batch_exec, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ptr{Cvoid}), plan.ptr, s, len, nchan, out))
    close!(plan)
    return Periodograms.Periodogram(s isa Vector ? vec(out) : out, cfg.freq)
end

# DSP.mt_spectrogram(s, n, noverlap; fs, onesided, kwargs...) for a matrix (the extension): src/multitaper.jl:262-404 per
# column; power length(freq) x k x size(s, 2), the layout of the batched spectrogram
function mt_spectrogram(s::Matrix{T}, n::Int, noverlap::Int; onesided::Bool=T <: Real, nfft::Int=nextpow(2, n), fs::Real=1,
                        nw::Real=4, ntapers::Int=ceil(Int, 2nw) - 1, window::Union{AbstractMatrix,Nothing}=nothing) where {T<:GPUNumber}
    len, nchan = size(s)
    n > noverlap || throw(ArgumentError("Need `samples_per_window > n_overlap_samples`"))
    cfg = Periodograms.MTConfig{T}(n; fs, nfft, window, nw, ntapers, onesided)
    k = len >= n ? div(len - n, n - noverlap) + 1 : 0
    out = zeros(abs2type(T), length(cfg.freq), k, nchan)
    if k > 0 && nchan > 0
        plan = mt_plan(cfg, T, n, noverlap, nfft, onesided)
        GC.@preserve s out check(ccall((:dspb200_mt_spectrogram_batch_exec, libdspb200), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ptr{Cvoid}), plan.ptr, s, len, nchan, out))
        close!(plan)
    end
    return out, cfg.freq, (n / 2 : n - noverlap : (k - 1) * (n - noverlap) + n / 2) / fs
end

# ------------------------------------------------------------------------------------------------ resample
# DSP.resample(x, rate::Union{Integer,Rational}, h): src/Filters/stream_filt.jl:688-725
function resample(x::Vector{Tx}, rate::Union{Integer,Rational}, h::Vector{Th}=Filters.resample_filter(rate)) where {Tx<:GPUNumber,Th<:GPUReal}
    sf = Filters.FIRFilter(h, rate)
    Filters.setphase!(sf, Filters.timedelay(sf))                 # undelay!, :706-714
    kern = sf.kernel
    n0 = kern.inputDeficit - 1
    phi0 = kern isa Union{Filters.FIRRational,Filters.FIRInterpolator} ? kern.ϕIdx - 1 : 0
    outlen = ceil(Int, length(x) * rate)
    To = promote_type(Th, Tx)
    out = Vector{To}(undef, outlen)
    hnd = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve h check(ccall((:dspb200_resample_plan_create, libdspb200), Cint,
        (Ref{Ptr{Cvoid}}, Cint, Cint, Ptr{Cvoid}, Int64, Int64, Int64),
        hnd, dtype_code(Tx), dtype_code(Th), h, length(h), numerator(rate), denominator(rate)))
    plan = Plan(hnd[], :dspb200_resample_plan_destroy)
    GC.@preserve x out check(ccall((:dspb200_resample_exec, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Int64, Int64, Ptr{Cvoid}, Int64),
        plan.ptr, x, length(x), 1, n0, phi0, out, outlen))
    close!(plan)
    return out
end

# ---- hilbert(x), src/util.jl:31-75 (real Float32 / Float64 arrays; other reals are converted by DSP.jl's own method)
function hilbert(x::Array{T}) where {T<:GPUReal}
    n = size(x, 1)
    out = Array{Complex{T}}(undef, size(x))
    n == 0 && return out
    GC.@preserve x out check(ccall((:dspb200_hilbert_exec, libdspb200), Cint,
        (Cint, Ptr{Cvoid}, Int64, Int64, Ptr{Cvoid}), dtype_code(T), x, n, length(x) ÷ n, out))
    out
end

# ---- the device work of filtfilt / finddelay / shiftsignal / alignsignals on device memory (src/Filters/filt.jl:245-259,
# src/util.jl:360-427).  Raw device pointers and a cudaStream_t (C_NULL: the default stream), as a CuArray binding would
# pass them; each call enqueues one launch and returns.  Not executed: no `julia` in the build image.
# extrapolate_signal! of every column: x is n x ncols, ext is (n + 2pad) x ncols, eltype T
filtfilt_extend!(::Type{T}, ext::Ptr{Cvoid}, x::Ptr{Cvoid}, n::Integer, ncols::Integer, pad::Integer;
                 stream::Ptr{Cvoid}=C_NULL) where {T<:GPUNumber} =
    check(ccall((:dspb200_filtfilt_extend_async, libdspb200), Cint, (Cint, Ptr{Cvoid}, Int64, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}),
                dtype_code(T), x, n, ncols, pad, ext, stream))
# finddelay's peak of every column of the real correlation s (nres x ncols): Int64 delays and Int32 NaN flags per column
xcorr_peak!(::Type{T}, delay::Ptr{Int64}, nanflag::Ptr{Int32}, s::Ptr{Cvoid}, nres::Integer, ncols::Integer, center::Integer;
            reversed::Bool=false, stream::Ptr{Cvoid}=C_NULL) where {T<:GPUReal} =
    check(ccall((:dspb200_xcorr_peak_async, libdspb200), Cint,
                (Cint, Ptr{Cvoid}, Int64, Int64, Int64, Cint, Ptr{Int64}, Ptr{Int32}, Ptr{Cvoid}),
                dtype_code(T), s, nres, ncols, center, reversed, delay, nanflag, stream))
# shiftsignal of every column, zero-filled: by `shift`, or by the device Int64 shifts (negated when `negate`)
shiftsignal!(::Type{T}, out::Ptr{Cvoid}, x::Ptr{Cvoid}, n::Integer, ncols::Integer; shift::Integer=0,
             shifts::Ptr{Int64}=Ptr{Int64}(C_NULL), negate::Bool=false, stream::Ptr{Cvoid}=C_NULL) where {T<:GPUNumber} =
    check(ccall((:dspb200_shift_async, libdspb200), Cint,
                (Cint, Ptr{Cvoid}, Int64, Int64, Int64, Ptr{Int64}, Cint, Ptr{Cvoid}, Int64, Ptr{Cvoid}),
                dtype_code(T), x, n, ncols, shift, shifts, negate, out, n, stream))

# ---- lpc / arburg / levinson, src/lpc.jl.  UNTESTED: no `julia` in the build image, so none of this has been run.
# Device-pointer forms (column-major n x ncols, a CuArray binding would pass raw pointers and its stream): each enqueues its
# launches on `stream` and returns.  a is (p + 1) x ncols for Burg (arburg's, with the leading 1), p x ncols otherwise.
lpc_work_bytes(::Type{T}, n::Integer, ncols::Integer, p::Integer, method::Integer; pin::Integer=0) where {T<:GPUNumber} =
    (b = Ref{Int64}(0); check(ccall((:dspb200_lpc_work_bytes, libdspb200), Cint, (Cint, Int64, Int64, Int64, Cint, Cint, Ref{Int64}),
                                    dtype_code(T), n, ncols, p, method, pin, b)); b[])
arburg!(::Type{T}, a::Ptr{Cvoid}, err::Ptr{Cvoid}, refl::Ptr{Cvoid}, x::Ptr{Cvoid}, n::Integer, ncols::Integer, p::Integer,
        work::Ptr{Cvoid}; pin::Integer=0, stream::Ptr{Cvoid}=C_NULL) where {T<:GPUNumber} =
    check(ccall((:dspb200_lpc_burg_async, libdspb200), Cint,
                (Cint, Ptr{Cvoid}, Int64, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Cvoid}),
                dtype_code(T), x, n, ncols, p, a, err, refl, work, pin, stream))
lpc_levinson!(::Type{T}, a::Ptr{Cvoid}, err::Ptr{Cvoid}, refl::Ptr{Cvoid}, x::Ptr{Cvoid}, n::Integer, ncols::Integer, p::Integer,
              work::Ptr{Cvoid}; stream::Ptr{Cvoid}=C_NULL) where {T<:GPUNumber} =
    check(ccall((:dspb200_lpc_levinson_async, libdspb200), Cint,
                (Cint, Ptr{Cvoid}, Int64, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                dtype_code(T), x, n, ncols, p, a, err, refl, work, stream))
levinson!(::Type{T}, a::Ptr{Cvoid}, err::Ptr{Cvoid}, refl::Ptr{Cvoid}, r::Ptr{Cvoid}, nr::Integer, ncols::Integer, p::Integer;
          stream::Ptr{Cvoid}=C_NULL) where {T<:GPUNumber} =
    check(ccall((:dspb200_levinson_async, libdspb200), Cint,
                (Cint, Ptr{Cvoid}, Int64, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                dtype_code(T), r, nr, ncols, p, a, err, refl, stream))

# Host vectors: staged through device buffers from dspb200_malloc, computed, copied back after one synchronisation.
function _dev(bytes::Integer)
    p = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:dspb200_malloc, libdspb200), Cint, (Ref{Ptr{Cvoid}}, Csize_t), p, max(bytes, 16)))
    p[]
end
_free(p::Ptr{Cvoid}) = ccall((:dspb200_free, libdspb200), Cint, (Ptr{Cvoid},), p)
_h2d(d::Ptr{Cvoid}, h::Array) = GC.@preserve h check(ccall((:dspb200_memcpy_h2d, libdspb200), Cint,
    (Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}), d, h, sizeof(h), C_NULL))
_d2h(h::Array, d::Ptr{Cvoid}) = GC.@preserve h check(ccall((:dspb200_memcpy_d2h, libdspb200), Cint,
    (Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Ptr{Cvoid}), h, d, sizeof(h), C_NULL))
_sync() = check(ccall((:dspb200_stream_sync, libdspb200), Cint, (Ptr{Cvoid},), C_NULL))

function _lpc_host(x::Vector{T}, p::Integer, method::Symbol) where {T<:GPUNumber}
    n = length(x)
    method === :burg ? (0 <= p <= n || throw(ArgumentError("arburg needs 0 <= p <= length(x)"))) :
                       (1 <= p <= n - 1 || throw(BoundsError(x, p + 1)))
    na = method === :burg ? p + 1 : p
    a, err, refl = Vector{T}(undef, na), Vector{real(T)}(undef, 1), Vector{T}(undef, p)
    wb = method === :levinson_r ? 0 : lpc_work_bytes(T, n, 1, p, method === :burg ? 0 : 1)
    dx, da, de, dr, dw = _dev(sizeof(x)), _dev(sizeof(a)), _dev(sizeof(err)), _dev(sizeof(refl)), _dev(wb)
    try
        _h2d(dx, x)
        method === :burg ? arburg!(T, da, de, dr, dx, n, 1, p, dw) :
        method === :levinson ? lpc_levinson!(T, da, de, dr, dx, n, 1, p, dw) : levinson!(T, da, de, dr, dx, n, 1, p)
        _d2h(a, da); _d2h(err, de); _d2h(refl, dr); _sync()
    finally
        foreach(_free, (dx, da, de, dr, dw))
    end
    return a, err[1], refl
end
arburg(x::Vector{T}, p::Integer) where {T<:GPUNumber} = _lpc_host(x, p, :burg)
levinson(r::Vector{T}, p::Integer) where {T<:GPUNumber} = _lpc_host(r, p, :levinson_r)
function lpc(x::Vector{T}, p::Integer, ::DSP.LPC.LPCBurg) where {T<:GPUNumber}
    a, err, _ = _lpc_host(x, p, :burg)
    return a[2:end], err
end
lpc(x::Vector{T}, p::Integer, ::DSP.LPC.LPCLevinson) where {T<:GPUNumber} = _lpc_host(x, p, :levinson)[1:2]

# ---- mt_cross_power_spectra! / mt_coherence!, src/multitaper.jl:553-603, 722-790.  `plan` is a multitaper plan built
# with dspb200_mt_plan_create from config.mt_config (tapers pre-scaled by 1/sqrt(r_t)); validation stays in DSP.jl.
function mt_cross!(output::Array, signal::Matrix{T}, plan::Ptr{Cvoid}, demean::Bool, freq_inds::UnitRange{Int},
                   coherence::Bool) where {T<:GPUReal}
    GC.@preserve signal output check(ccall((:dspb200_mt_cross_spectra_exec, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Cint, Int64, Int64, Cint, Ptr{Cvoid}),
        plan, signal, size(signal, 1), demean, first(freq_inds) - 1, length(freq_inds), coherence, output))
    output
end
# An extension: the epoch mean over an n_channels x n_samples x n_epochs array (signal[:, :, e] is epoch e's matrix),
# summed in epoch order in the output eltype and divided by n_epochs part by part.
function mt_cross!(output::Array, signal::Array{T,3}, plan::Ptr{Cvoid}, demean::Bool, freq_inds::UnitRange{Int},
                   coherence::Bool) where {T<:GPUReal}
    GC.@preserve signal output check(ccall((:dspb200_mt_cross_spectra_epochs_exec, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Cint, Int64, Int64, Cint, Ptr{Cvoid}),
        plan, signal, size(signal, 1), size(signal, 3), demean, first(freq_inds) - 1, length(freq_inds), coherence, output))
    output
end

# ---- filt!(buffer, ::FIRFilter{FIRArbitrary}, x), src/Filters/stream_filt.jl:579-625.  Output j of a call sits at total
# phase acc + j*delta; the number of outputs and the carried state are computed in exact rational arithmetic
# (dsp.jl_b200/filters.py::_arb_advance), the device evaluates the same phases in double-double.
function arb_advance(acc::Float64, deficit::Int, delta::Float64, Nϕ::Int, xlen::Int)
    A, D = Rational{BigInt}(acc), Rational{BigInt}(delta)
    M = xlen - deficit + 1
    nout = Int(ceil((M * Nϕ - A) / D))                           # number of j >= 0 with A + j*D < M*Nϕ
    P = A + nout * D
    q = fld(P, Nϕ)
    newacc = Float64(P - q * Nϕ)
    newacc >= Nϕ && (newacc = prevfloat(Float64(Nϕ)))
    return nout, deficit + Int(q) - xlen, newacc
end

function filt(self::Filters.FIRFilter{Filters.FIRArbitrary{Th}}, x::Vector{Tx}, plan::Plan) where {Th<:GPUReal,Tx<:GPUNumber}
    kernel = self.kernel
    xlen = length(x)
    hist = convert(Vector{Tx}, self.history)                      # history starts as Vector{Float64}; :587 history::Vector{Tx}
    if xlen < kernel.inputDeficit                                # :590-594
        self.history = Util.shiftin!(hist, x)
        kernel.inputDeficit -= xlen
        return Vector{promote_type(Th, Tx)}(undef, 0)
    end
    nout, deficit, acc = arb_advance(kernel.ϕAccumulator, kernel.inputDeficit, kernel.Δ, kernel.Nϕ, xlen)
    xe = vcat(hist, x)
    n0 = self.historyLen + kernel.inputDeficit - 1
    out = Vector{promote_type(Th, Tx)}(undef, nout)
    GC.@preserve xe out check(ccall((:dspb200_resample_arb_exec, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Cdouble, Cdouble, Ptr{Cvoid}, Int64),
        plan.ptr, xe, length(xe), n0, kernel.ϕAccumulator, kernel.Δ, out, nout))
    kernel.inputDeficit, kernel.ϕAccumulator = deficit, acc       # :620
    kernel.α, foffset = modf(acc)
    kernel.ϕIdx = 1 + Int(foffset)
    self.history = Util.shiftin!(hist, x)                         # :621
    return out
end

function arb_plan(::Type{Tx}, h::Vector{Th}, Nϕ::Integer) where {Tx<:GPUNumber,Th<:GPUReal}
    hnd = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve h check(ccall((:dspb200_resample_arb_plan_create, libdspb200), Cint,
        (Ref{Ptr{Cvoid}}, Cint, Cint, Ptr{Cvoid}, Int64, Int64), hnd, dtype_code(Tx), dtype_code(Th), h, length(h), Nϕ))
    Plan(hnd[], :dspb200_resample_plan_destroy)
end

# DSP.resample(x, rate::AbstractFloat, h, Nϕ): src/Filters/stream_filt.jl:692-725
function resample(x::Vector{Tx}, rate::AbstractFloat, h::Vector{Th}=Filters.resample_filter(rate), Nϕ::Integer=32) where {Tx<:GPUNumber,Th<:GPUReal}
    sf = Filters.FIRFilter(h, rate, Nϕ)
    Filters.setphase!(sf, Filters.timedelay(sf))                 # undelay!, :706-714
    outlen = ceil(Int, length(x) * rate)
    # one sample more than inputlength(sf, outLen, RoundUp) (:699): guarantees the exact output count reaches outLen
    xpad = zeros(Tx, max(Filters.inputlength(sf, outlen, RoundUp), 0) + 1)
    copyto!(xpad, 1, x, 1, min(length(x), length(xpad)))
    plan = arb_plan(Tx, h, Nϕ)
    y = filt(sf, xpad, plan)
    close!(plan)
    length(y) >= outlen || throw(AssertionError("Resample output shorter than expected."))   # :722
    return resize!(y, outlen)
end

# DSP.resample(X, rate::AbstractFloat, h, Nϕ; dims) of a matrix, src/Filters/stream_filt.jl:751-775.  Every column gets a
# fresh filter after undelay!, so all columns share (n0, acc0, delta) and run in one launch.  The kernel reads
# min(size(X, dims), npad) samples of each column (npad: the padded length of the vector method), zero elsewhere.
function resample(X::Matrix{Tx}, rate::AbstractFloat, h::Vector{Th}=Filters.resample_filter(rate), Nϕ::Integer=32;
                  dims::Integer) where {Tx<:GPUNumber,Th<:GPUReal}
    Xc = dims == 1 ? X : dims == 2 ? permutedims(X) : throw(ArgumentError("dims must be 1 or 2"))
    nx, ncols = size(Xc)
    sf = Filters.FIRFilter(h, rate, Nϕ)
    Filters.setphase!(sf, Filters.timedelay(sf))                 # undelay!, :706-714
    kern = sf.kernel
    outlen = ceil(Int, nx * rate)
    npad = max(Filters.inputlength(sf, outlen, RoundUp), 0) + 1
    if ncols > 0
        avail = npad < kern.inputDeficit ? 0 : arb_advance(kern.ϕAccumulator, kern.inputDeficit, kern.Δ, kern.Nϕ, npad)[1]
        avail >= outlen || throw(AssertionError("Resample output shorter than expected."))  # :722
    end
    out = Matrix{promote_type(Th, Tx)}(undef, outlen, ncols)
    plan = arb_plan(Tx, h, Nϕ)
    GC.@preserve Xc out check(ccall((:dspb200_resample_arb_batch_exec, libdspb200), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Int64, Int64, Cdouble, Cdouble, Ptr{Cvoid}, Int64),
        plan.ptr, Xc, min(nx, npad), nx, ncols, kern.inputDeficit - 1, kern.ϕAccumulator, kern.Δ, out, outlen))
    close!(plan)
    return dims == 1 ? out : permutedims(out)
end

# ---- conv(u, v) for matrices / rank-3 arrays (src/dspbase.jl:611-660) and periodogram(s::Matrix) (src/periodograms.jl:473-509)
function conv_nd!(out::Array{T,N}, u::Array{T,N}, v::Array{T,N}; algorithm::Symbol=:auto) where {T<:GPUNumber,N}
    # algorithm resolution of conv!, src/dspbase.jl:720-751
    all(size(out) .== size(u) .+ size(v) .- 1) || throw(ArgumentError("out must have size(u) .+ size(v) .- 1"))
    algorithm === :auto && (algorithm = :fast)
    algorithm === :fast && (algorithm = length(u) * length(v) < 2^16 ? :direct : :fft)
    large, small = length(u) >= length(v) ? (u, v) : (v, u)              # v should be the smaller array (:746-751)
    os_nffts = map(DSP.optimalfftfiltlength, size(small), size(large))    # :736
    if algorithm === :fft
        algorithm = any(os_nffts .< size(out)) ? :fft_overlapsave : :fft_simple        # :737-743
    end
    algorithm in (:direct, :fft_simple, :fft_overlapsave) ||
        throw(ArgumentError("algorithm must be :auto, :fast, :direct, :fft, :fft_simple, or :fft_overlapsave"))
    if algorithm === :fft_overlapsave                                     # unsafe_conv_kern_os!, :371-609 (batched blocks)
        us, vs, nf = collect(Int64, size(large)), collect(Int64, size(small)), collect(Int64, os_nffts)
        GC.@preserve us vs nf large small out check(ccall((:dspb200_conv_nd_os_exec, libdspb200), Cint,
            (Cint, Cint, Ptr{Int64}, Ptr{Cvoid}, Ptr{Int64}, Ptr{Cvoid}, Ptr{Int64}, Ptr{Cvoid}),
            dtype_code(T), N, us, large, vs, small, nf, out))
        return out
    end
    us, vs = collect(Int64, size(u)), collect(Int64, size(v))
    nf = collect(Int64, DSP.nextfastfft(size(u) .+ size(v) .- 1))       # rooted below: the library reads it during the call
    GC.@preserve us vs nf u v out check(ccall((:dspb200_conv_nd_exec, libdspb200), Cint,
        (Cint, Cint, Ptr{Int64}, Ptr{Cvoid}, Ptr{Int64}, Ptr{Cvoid}, Ptr{Int64}, Ptr{Cvoid}),
        dtype_code(T), N, us, u, vs, v, algorithm === :direct ? Ptr{Int64}(C_NULL) : pointer(nf), out))
    out
end
conv(u::Array{T,N}, v::Array{T,N}; algorithm::Symbol=:auto) where {T<:GPUNumber,N} =
    conv_nd!(Array{T,N}(undef, size(u) .+ size(v) .- 1), u, v; algorithm)

function periodogram2!(out::Array{T}, s::Matrix{T}, nfft::NTuple{2,Int}, r::Real, ptype::Int) where {T<:GPUReal}
    GC.@preserve s out check(ccall((:dspb200_periodogram2_exec, libdspb200), Cint,
        (Cint, Ptr{Cvoid}, Int64, Int64, Int64, Int64, Cdouble, Cint, Ptr{Cvoid}),
        dtype_code(T), s, size(s, 1), size(s, 2), nfft[1], nfft[2], r, ptype, out))
    out
end

# ------------------------------------------------------------------------------------------------ drop-in overlay
# DSPB200 is a PARALLEL module with the reference's signatures: `DSPB200.conv(u, v)` next to `DSP.conv(u, v)`.
# `DSPB200.install_overlay!()` turns it into a drop-in: it adds methods to DSP.jl's own generic functions for the concrete
# GPU-eligible argument types (Vector / Array of Float32, Float64, ComplexF32, ComplexF64) -- more specific than DSP.jl's
# AbstractArray methods, so dispatch prefers them and user code calling `DSP.conv`, `DSP.filt`, `DSP.welch_pgram`,
# `DSP.spectrogram`, `DSP.resample` ... runs on the GPU unchanged; every other argument type keeps the reference path.
# (Deliberate type piracy, opt-in; never executed in the build container -- no Julia there.)
function install_overlay!()
    for T in (Float32, Float64, ComplexF32, ComplexF64)
        @eval begin
            DSP.conv(u::Vector{$T}, v::Vector{$T}; kw...) = conv(u, v; kw...)
            DSP.conv!(out::Vector{$T}, u::Vector{$T}, v::Vector{$T}; kw...) = conv!(out, u, v; kw...)
            DSP.conv(u::Matrix{$T}, v::Matrix{$T}; kw...) = conv(u, v; kw...)
            DSP.conv(u::Array{$T,3}, v::Array{$T,3}; kw...) = conv(u, v; kw...)
            DSP.filt(b::Vector{$T}, x::Array{$T}) = filt(b, x)
            DSP.welch_pgram(s::Vector{$T}, n::Int=length(s) >> 3, noverlap::Int=n >> 1; kw...) = welch_pgram(s, n, noverlap; kw...)
            DSP.periodogram(s::Vector{$T}; kw...) = periodogram(s; kw...)
            DSP.spectrogram(s::Vector{$T}, n::Int=length(s) >> 3, noverlap::Int=n >> 1; kw...) = spectrogram(s, n, noverlap; kw...)
            DSP.stft(s::Vector{$T}, n::Int=length(s) >> 3, noverlap::Int=n >> 1, psdonly::Union{Nothing,Periodograms.PSDOnly}=nothing; kw...) =
                stft(s, n, noverlap, psdonly; kw...)
            DSP.resample(x::Vector{$T}, rate::Union{Integer,Rational}) = resample(x, rate)
            DSP.mt_pgram(s::Vector{$T}; kw...) = mt_pgram(s; kw...)
            DSP.mt_pgram(s::Matrix{$T}; kw...) = mt_pgram(s; kw...)
            DSP.mt_spectrogram(s::Matrix{$T}, n::Int, noverlap::Int; kw...) = mt_spectrogram(s, n, noverlap; kw...)
            DSP.LPC.arburg(x::Vector{$T}, p::Integer) = arburg(x, p)
            DSP.LPC.levinson(r::Vector{$T}, p::Integer) = levinson(r, p)
            DSP.LPC.lpc(x::Vector{$T}, p::Integer, m::DSP.LPC.LPCBurg) = lpc(x, p, m)
            DSP.LPC.lpc(x::Vector{$T}, p::Integer, m::DSP.LPC.LPCLevinson) = lpc(x, p, m)
        end
    end
    for T in (Float32, Float64)
        @eval begin
            DSP.Filters.fftfilt(b::Vector{$T}, x::Array{$T}) = fftfilt(b, x)
            DSP.hilbert(x::Array{$T}) = hilbert(x)
        end
    end
    return nothing
end

end # module
