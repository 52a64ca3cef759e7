"""Autograd-aware operator surface over the C-ABI library ``libdfold_b200.so`` (include/dfold_b200.h).

Every function here launches hand-written sm_90a kernels through ctypes with raw device pointers and the
current CUDA stream.  There is NO CPU path and no fallback to torch library kernels for the arithmetic: if the
shared library is missing, or a tensor is not on a CUDA device, the ops raise.  (The tests exercise the host-side
module logic on CPU by monkey-patching these names with the oracle — that seam lives in tests/, not here.)
Every entry point that launches kernels is called through ``launch(name, *args)``, which passes tensors as device
pointers, appends the current stream and raises with the library's message on failure.

torch is used for: device memory (``torch.empty``), streams, autograd bookkeeping, and trivial view / elementwise
glue (cat, slicing, SiLU on tiny tensors, masks).
"""
import contextlib
import ctypes
import functools
import os
import weakref
from typing import Optional

import torch
from torch.autograd import Function

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdfold_b200.so")
_LIB = None

# signature mini-language: p pointer, l long, i int, f float, d double
_SIGS = {
    "dfold_abi_version": "",
    "dfold_capture_id": "pp",
    "dfold_debug_gemm_stats": "p",
    "dfold_debug_ipa_stats": "p",
    "dfold_split2d": "plllipl" + "ppll" + "ppll" + "pp",
    "dfold_split2d_residual_gate": "plllippl" + "ppll" + "ppll" + "pp",
    "dfold_conv_weight_prep": "piii" + "ppl" + "ppl" + "p",
    "dfold_taps_to_param": "piiipip",
    "dfold_sgemm": "pllll" * 4 + "p" + "iiiii" + "ff" + "iii" + "p",
    "dfold_global_layernorm_fwd": "pppplfip",
    "dfold_global_layernorm_bwd": "pppppl" + "ip",
    "dfold_row_layernorm_fwd": "ppppplifp",
    "dfold_row_layernorm_bwd": "ppppppplip",
    "dfold_quat_to_rot_fwd": "pplp",
    "dfold_quat_to_rot_bwd": "ppplp",
    "dfold_rigid_apply_fwd": "ppplp" + "lliip",
    "dfold_rigid_apply_bwd": "ppplp" + "ppp" + "lliip",
    "dfold_compose_q_update_fwd": "pppppplp",
    "dfold_compose_q_update_bwd": "pppppppplp",
    "dfold_gemm_bf16x3": "pplli" + "lll" + "ppllii" + "pl" + "p" + "pl" + "ffi" + "p",
    "dfold_gemm_wgrad_bf16x3": "ppll" + "ppll" + "llilii" + "plf" + "p",
    "dfold_ipa_attn_fwd": "plplppplpppp" + "iiiiiiii" + "ff" + "ppp",
    "dfold_ipa_attn_bwd": "plplppplpppp" + "iiiiiiii" + "ff" + "ppp" + "ppppppppp" + "p",
    "dfold_ipa_pre_bwd": "pp" + "iiiiiii" + "pp" + "pppp" + "p",
    "dfold_ipa_fused_fwd": "pppppppp" + "ppl" + "iiiiiiii" + "ff" + "pp",
    "dfold_ipa_ds_bwd": "ppppl" + "iiiii" + "pppp" + "pp" + "p",
    "dfold_gemm_bf16x3_batched": "ppllll" + "liill" + "ppllll" + "llil" + "pllilf" + "p",
    "dfold_gemm_wgrad_bf16x3_batched": "pplllll" + "pplllll" + "lll" + "i" + "iiiil" + "pllf" + "p",
    "dfold_score_fwd": "ppppp" + "pidddd" + "ffpil" + "ppi" + "p",
    "dfold_score_bwd": "ppppp" + "pidddd" + "ffpil" + "ppi" + "pp" + "p",
    "dfold_frames_to_atoms_fwd": "pippp" + "pppppp" + "ppp" + "lp",
    "dfold_reverse_step": "ppppi" + "ppp" + "dddddd" + "iii" + "pp" + "llp",
    "dfold_adam_amsgrad": "pppppl" + "pi" + "fffff" + "p",
    "dfold_adam_amsgrad_clip": "pppppl" + "pi" + "fffff" + "pp",
    "dfold_grad_norm": "plff" + "ppp" + "p",
    "dfold_adam_amsgrad_dlr": "pppppl" + "pi" + "p" + "ffff" + "pp",
    "dfold_lr_schedule": "p" + "dd" + "lll" + "d" + "pp",
    "dfold_featurize_window": "pppppp" + "ii" + "pppp" + "p",
    "dfold_loss_fwd": "pppppppppppp" + "ii" + "dddd" + "ii" + "pppp" + "p",
    "dfold_quat_mul_fwd": "ppplip",
    "dfold_quat_mul_bwd": "ppppplip",
    "dfold_rot_compose_fwd": "pppp" + "pp" + "liip",
    "dfold_rot_compose_bwd": "pppp" + "pp" + "pppp" + "liip",
    "dfold_igso3_tables": "piiipp" + "p",
    "dfold_forward_marginal": "ppppp" + "pppp" + "iiidddd" + "f" + "iii" + "ppppp" + "lp",
    "dfold_rot_trans_error": "pipi" + "iii" + "pp",
    "dfold_atom_errors": "pipipi" + "iiii" + "pp",
    "dfold_superimpose": "pipi" + "ll" + "pill" + "i" + "ii" + "pppp" + "p",
    "dfold_drmsd": "pipi" + "ll" + "pill" + "i" + "ii" + "pp" + "p",
    "dfold_rollout_advance": "pppppp" + "iiii" + "p",
}
_CT = {"p": ctypes.c_void_p, "l": ctypes.c_long, "i": ctypes.c_int, "f": ctypes.c_float, "d": ctypes.c_double}


def lib():
    """Load the C-ABI library (fails loudly when it has not been built)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build the sm_90a extension first (python -m dynamicpdb_b200.build or "
                "__graft_entry__.build()).  dynamicpdb_b200 has no CPU / PyTorch fallback.")
        L = ctypes.CDLL(LIB_PATH)
        for name, sig in _SIGS.items():
            fn = getattr(L, name)
            fn.argtypes = [_CT[c] for c in sig]
            fn.restype = ctypes.c_int
        L.dfold_last_error.restype = ctypes.c_char_p
        L.dfold_last_error.argtypes = []
        _LIB = L
    return _LIB


def exported_symbols():
    return sorted(list(_SIGS) + ["dfold_last_error"])


# kernels launched per C-ABI call (bench.py reports the total as `gpu_launches`)
_LAUNCHES_PER_CALL = {"dfold_global_layernorm_fwd": 3, "dfold_global_layernorm_bwd": 3, "dfold_ipa_attn_bwd": 4,
                      "dfold_grad_norm": 2}
LAUNCH_COUNT = 0
# When True (set by train_step.TrainStep around its step), weight gradients of the convolution are accumulated by the kernel
# straight into the parameter's existing .grad buffer and autograd receives None: the ConvNet is shared by the four blocks
# (ipa_pytorch_dynamic.py:749,863), so the default path costs three 82 MB add passes per weight and step.
GRAD_ACCUMULATE_INPLACE = False
# optional per-launch timing: when PROFILE is a list, timed(...) appends (name, work, start_event, end_event).  Every launch
# then stays on the current stream, so each event pair times one kernel running alone.
PROFILE = None
# The in-place convolution weight gradients run on one side stream per device (created on first use), overlapping the rest
# of the backward: nothing in the backward reads them.  _SIDE_HELD keeps the tensors that work reads alive until
# join_side_stream(); the caching allocator would otherwise hand their memory to the current stream while it is still read.
_SIDE_STREAMS = {}
_SIDE_HELD = {}


_PASS = frozenset((int, float, type(None), ctypes.c_void_p))


def launch(name: str, *args):
    """Call the launching entry point ``name`` with ``args`` and the current stream (its last parameter): a tensor passes
    its data pointer, None NULL, and anything else (``_ptr`` values, ints, floats) goes as is to the ctypes signature."""
    global LAUNCH_COUNT
    # the set lookup settles the common scalar types before the slower isinstance against torch.Tensor's metaclass:
    # eager sampling is bound by the host cost of its launches
    rc = getattr(lib(), name)(*[a if type(a) in _PASS else ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a
                                for a in args], _stream())
    if rc != 0:
        raise RuntimeError(f"{name}: {lib().dfold_last_error().decode()}")
    LAUNCH_COUNT += _LAUNCHES_PER_CALL.get(name, 1)


class _timed:
    """Brackets one kernel launch with CUDA events on the launching stream when profiling is enabled."""

    def __init__(self, name, work, tag=""):
        self.name, self.work, self.tag = name, work, tag

    def __enter__(self):
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if PROFILE is not None and exc[0] is None:
            self.e1.record()
            PROFILE.append((self.name, self.work, self.e0, self.e1, self.tag))
        return False


@contextlib.contextmanager
def _on_side_stream(dev, held):
    """Run the enclosed launches on ``dev``'s side stream, after all work queued so far on the current stream.  ``held``:
    tensors from the current stream's memory that they read, kept alive until join_side_stream()."""
    side = _SIDE_STREAMS.get(dev.index)
    if side is None:
        side = _SIDE_STREAMS[dev.index] = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    _SIDE_HELD.setdefault(dev.index, []).extend(held)
    with torch.cuda.stream(side):
        yield


def join_side_stream():
    """Make the current stream wait for the work queued on the side streams and release the tensors it read.  Call it after
    a backward that accumulated in place (GRAD_ACCUMULATE_INPLACE) and before the gradient buffer is read; under CUDA-graph
    capture it joins the side branch back into the captured stream."""
    for idx, held in list(_SIDE_HELD.items()):
        torch.cuda.current_stream(idx).wait_stream(_SIDE_STREAMS[idx])
        held.clear()
    _SIDE_HELD.clear()


def _ptr(t: Optional[torch.Tensor], offset: int = 0):
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr() + offset * t.element_size())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


_SMS = {}


def _sm_count(dev) -> int:
    """Streaming multiprocessors of `dev` (132 on an H100 SXM)."""
    idx = torch.device(dev).index
    if idx is None:
        idx = torch.cuda.current_device()
    if idx not in _SMS:
        _SMS[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return _SMS[idx]


def _on_device(fn):
    """Run an autograd Function's forward / backward with the CUDA device of its tensors current.  The C-ABI launches,
    cuTensorMapEncode and the stream lookup all act on the CURRENT device, and the reference trainer's single-GPU
    mode places the model on `cuda:{least loaded}` without torch.cuda.set_device (train_DFOLD_dynamics.py:356,603-606)."""
    @functools.wraps(fn)
    def wrapper(*args, **kw):
        dev = None
        for a in args:
            if isinstance(a, torch.Tensor) and a.is_cuda:
                if dev is None:
                    dev = a.device
                elif a.device != dev:
                    raise RuntimeError(f"dynamicpdb_b200: operands on different devices ({dev} and {a.device})")
        if dev is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kw)
        with torch.cuda.device(dev):
            return fn(*args, **kw)
    return wrapper


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("dynamicpdb_b200 ops need CUDA tensors (H100 / sm_90a); there is no CPU fallback")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


# --------------------------------------------------------------------------------------------------
# raw launch helpers
# --------------------------------------------------------------------------------------------------
def _sgemm(A, a_off, a_rs, a_cs, a_bs, a_bs2, B, b_off, b_rs, b_cs, b_bs, b_bs2, C, c_off, c_rs, c_cs, c_bs, c_bs2,
           M, N, K, *, R=None, r_off=0, r_rs=0, r_cs=0, r_bs=0, r_bs2=0, bias=None, batch=1, batch2=1,
           alpha=1.0, beta=1.0, act=0, pre_relu=0):
    launch("dfold_sgemm", _ptr(A, a_off), a_rs, a_cs, a_bs, a_bs2, _ptr(B, b_off), b_rs, b_cs, b_bs, b_bs2,
           _ptr(C, c_off), c_rs, c_cs, c_bs, c_bs2, _ptr(R, r_off), r_rs, r_cs, r_bs, r_bs2,
           bias, batch, batch2, M, N, K, alpha, beta, act, pre_relu, 1)


def _split2d(x2: torch.Tensor, *, pre_relu=False, gate=None, gate_sub=None, want=True, want_t=False, colsum=None,
             t_out=None, t_ld=None, t_off=0, rpad=None):
    """x2 [R, C] fp32 contiguous -> (hi, lo) [R, C8] and / or transposed planes [C, R8] (or into ``t_out``); ``colsum``
    ([C], zeroed) receives the column sums of the gated input.  The gate passes x2 where ``gate > 0``, or with
    ``gate_sub`` (same strides as ``gate``) where ``gate - gate_sub > 0``."""
    R, C = x2.shape
    hi = lo = hit = lot = None
    c8 = _pad8(C)
    if want:
        hi = torch.empty((R, c8), dtype=torch.int16, device=x2.device)
        lo = torch.empty((R, c8), dtype=torch.int16, device=x2.device)
    ldt = 0
    rp = 0
    if want_t:
        if t_out is None:
            r8 = _pad8(R)
            hit = torch.empty((C, r8), dtype=torch.int16, device=x2.device)
            lot = torch.empty((C, r8), dtype=torch.int16, device=x2.device)
            ldt, rp = r8, r8
        else:
            hit, lot = t_out
            ldt, rp = t_ld, rpad
    ldg = gate.stride(0) if gate is not None else 0
    if gate_sub is None:
        launch("dfold_split2d", x2, R, C, x2.stride(0), int(pre_relu), gate, ldg,
               hi, lo, c8, c8, _ptr(hit, t_off), _ptr(lot, t_off), ldt, rp, colsum)
    else:
        launch("dfold_split2d_residual_gate", x2, R, C, x2.stride(0), int(pre_relu), gate, gate_sub, ldg,
               hi, lo, c8, c8, _ptr(hit, t_off), _ptr(lot, t_off), ldt, rp, colsum)
    return (hi, lo), (hit, lot)


_WCACHE = {}
_WCACHE_EPOCH = 0


def invalidate_weight_cache():
    """Forget every cached weight plane.  A CUDA-graph replay updates the weights on the device without bumping the
    Python-side version counters, so ``train_step.TrainStep`` calls this after each replay; the next EAGER call then
    rebuilds its planes from the current weights (replays themselves never consult this cache).
    Call it as well after any in-place update made through ``param.data`` (EMA swaps, ``p.data.copy_``, manual clipping):
    those do not bump ``_version`` either."""
    global _WCACHE_EPOCH
    _WCACHE_EPOCH += 1


def _capture_id() -> int:
    if not torch.cuda.is_current_stream_capturing():
        return 0
    out = ctypes.c_ulonglong(0)
    rc = lib().dfold_capture_id(_stream(), ctypes.byref(out))
    if rc != 0:
        raise RuntimeError(f"dfold_capture_id: {lib().dfold_last_error().decode()}")
    return int(out.value)


def _cache_get(kind, w: torch.Tensor, build):
    """bf16 operand planes of a weight, rebuilt whenever the tensor object or its version counter changes
    (optimizer steps and load_state_dict bump ``_version``) or a graph replay may have changed it."""
    capturing = _capture_id()
    key = (kind, id(w), capturing)
    ent = _WCACHE.get(key)
    stamp = (w._version, w.data_ptr(), _WCACHE_EPOCH)
    if ent is not None and ent[0]() is w and ent[1] == stamp:
        return ent[2]
    # While a CUDA graph is being captured the planes are (re)built INSIDE that capture, from graph-pool memory: a hit on
    # an eager-pool entry would bake a pointer into the graph that a later eager rebuild frees, and a hit on another
    # graph's entry would read planes only that other graph refreshes.  Within one capture the same weight is split
    # once: the entry keyed with this capture's id serves the remaining call sites.
    val = build()
    if len(_WCACHE) > 512:
        for k in [k for k, e in _WCACHE.items() if e[0]() is None]:
            del _WCACHE[k]
    _WCACHE[key] = (weakref.ref(w), stamp, val)
    return val


def _linear_planes(w: torch.Tensor):
    """(hi, lo) [N, K8] and transposed (hi_t, lo_t) [K, N8] bf16 planes of a Linear weight, cached per version."""
    def build():
        with torch.no_grad():
            (hi, lo), (hit, lot) = _split2d(_f32c(w.detach()), want=True, want_t=True)
        return hi, lo, hit, lot
    return _cache_get("lin", w, build)


def _conv_planes(w: torch.Tensor):
    """fwd planes [25][O][I8] and dgrad planes [25][I][O8] (tap-flipped) of a conv weight [O, I, kh, kw]."""
    def build():
        O, I, kh, kw = w.shape
        T = kh * kw
        i8, o8 = _pad8(I), _pad8(O)
        mk = lambda *s: torch.zeros(s, dtype=torch.int16, device=w.device)
        f_hi, f_lo, d_hi, d_lo = mk(T, O, i8), mk(T, O, i8), mk(T, I, o8), mk(T, I, o8)
        wc = _f32c(w.detach())     # keep the converted tensor alive until the launch is enqueued
        launch("dfold_conv_weight_prep", wc, O, I, T, f_hi, f_lo, i8, d_hi, d_lo, o8)
        return f_hi, f_lo, d_hi, d_lo
    return _cache_get("conv", w, build)


def _gemm(a_hi, a_lo, F, Nr, K, lda, b_hi, b_lo, n_out, ldb, taps_f, taps_n, out, ldo, bias, residual, ldr, alpha, beta, act,
          F_out=None, f_start=0):
    F_out = F if F_out is None else F_out
    with _timed("gemm_bf16x3", 2.0 * F_out * Nr * K * n_out * taps_f * taps_n, f"kmajor F{F_out} N{Nr} K{K} out{n_out} taps{taps_f * taps_n}"):
        launch("dfold_gemm_bf16x3", a_hi, a_lo, F, F_out, f_start, Nr, K, lda, b_hi, b_lo, n_out, ldb, taps_f, taps_n,
               out, ldo, bias, residual, ldr, alpha, beta, act)


def _gemm_wgrad(a, M, lda, b, Nn, ldb, F, Nr, taps_f, taps_n, out, ldo, Fb=None, b_f_add=0):
    Fb = F if Fb is None else Fb
    with _timed("gemm_bf16x3", 2.0 * F * Nr * M * Nn * taps_f * taps_n, f"wgrad F{F} N{Nr} M{M} n{Nn} taps{taps_f * taps_n}"):
        launch("dfold_gemm_wgrad_bf16x3", a[0], a[1], M, lda, b[0], b[1], Nn, ldb, F, Fb, b_f_add, Nr, taps_f, taps_n, out, ldo, 1.0)


_ACT = {None: 0, "relu": 1}


def _use_tensor_cores(M: int, N: int, K: int) -> bool:
    # the 128 x BN wgmma tile needs 16-byte aligned K rows; tiny problems stay on the SIMT kernel
    return K % 8 == 0 and K >= 64 and N >= 16 and M >= 32 and (M * N * K) >= (1 << 18)


# --------------------------------------------------------------------------------------------------
# linear
# --------------------------------------------------------------------------------------------------
class _LinearFn(Function):
    @staticmethod
    @_on_device
    def forward(ctx, x, w, b, act, residual, pre_relu):
        _need_cuda(x, w, b, residual)
        K_ = w.shape[1]
        N_ = w.shape[0]
        x2 = _f32c(x.reshape(-1, K_))
        M_ = x2.shape[0]
        wf = _f32c(w)
        bf = _f32c(b) if b is not None else None
        r2 = _f32c(residual.reshape(-1, N_)) if residual is not None else None
        out = torch.empty((M_, N_), dtype=torch.float32, device=x.device)
        tc = _use_tensor_cores(M_, N_, K_)
        a_hi = a_lo = None
        if tc:
            (a_hi, a_lo), _ = _split2d(x2, pre_relu=pre_relu)
            w_hi, w_lo, _, _ = _linear_planes(w)
            _gemm(a_hi, a_lo, 1, M_, K_, a_hi.shape[1], w_hi, w_lo, N_, w_hi.shape[1], 1, 1, out, N_, bf, r2, N_, 1.0, 1.0, _ACT[act])
        else:
            _sgemm(x2, 0, K_, 1, 0, 0, wf, 0, K_, 1, 0, 0, out, 0, N_, 1, 0, 0, M_, N_, K_, R=r2, r_rs=N_, r_cs=1,
                   bias=bf, act=_ACT[act], pre_relu=int(pre_relu))
        # the tensor-core path keeps the bf16 operand planes (same bytes as x) for the weight gradient instead of x
        ctx.save_for_backward(None if tc else x2, w, out if act == "relu" else None, r2 if act == "relu" else None, a_hi, a_lo)
        ctx.mk = (M_, K_)
        ctx.meta = (x.shape, act, pre_relu, tc, b is not None, residual is not None and residual.shape)
        return out.reshape(x.shape[:-1] + (N_,))

    @staticmethod
    @_on_device
    def backward(ctx, dy):
        x2, w, out, r2, a_hi, a_lo = ctx.saved_tensors
        xshape, act, pre_relu, tc, has_b, rshape = ctx.meta
        M_, K_ = ctx.mk
        N_ = w.shape[0]
        g = _f32c(dy.reshape(M_, N_))
        dres = dy.reshape(rshape) if rshape else None
        need_x, need_w, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1], has_b and ctx.needs_input_grad[2]
        dx = dw = db = None
        if tc:
            db_buf = torch.zeros(N_, dtype=torch.float32, device=g.device) if need_b else None
            (g_hi, g_lo), _ = _split2d(g, gate=out, gate_sub=r2, want=need_x or need_w, colsum=db_buf)
            db = db_buf
            if need_x:
                _, _, wt_hi, wt_lo = _linear_planes(w)
                dx = torch.empty((M_, K_), dtype=torch.float32, device=g.device)
                _gemm(g_hi, g_lo, 1, M_, N_, g_hi.shape[1], wt_hi, wt_lo, K_, wt_hi.shape[1], 1, 1, dx, K_, None, None, 0, 1.0, 0.0, 0)
            if need_w:
                dw = torch.empty((N_, K_), dtype=torch.float32, device=g.device)
                _gemm_wgrad((g_hi, g_lo), N_, g_hi.shape[1], (a_hi, a_lo), K_, a_hi.shape[1], 1, M_, 1, 1, dw, K_)
        else:
            if out is not None:
                g = g * ((out if r2 is None else out - r2) > 0)
            wf = _f32c(w)
            if need_x:
                dx = torch.empty((M_, K_), dtype=torch.float32, device=g.device)
                _sgemm(g, 0, N_, 1, 0, 0, wf, 0, 1, K_, 0, 0, dx, 0, K_, 1, 0, 0, M_, K_, N_)
            if need_w:
                xr = torch.relu(x2) if pre_relu else x2
                # tiny [N, K] output reduced over all M rows: split the reduction over CTAs
                tiles = ((N_ + 63) // 64) * ((K_ + 63) // 64)
                ks = max(1, min(M_ // 512, 4 * _sm_count(g.device) // tiles, 256))
                # chunks of `kc` rows as a batch of partial products [ks (+1 for the tail), N, K], added in a fixed order
                # (split-K with atomics would make the last bits vary from run to run)
                kc = M_ // ks
                tail = M_ - ks * kc
                part = torch.empty((ks + (1 if tail else 0), N_, K_), dtype=torch.float32, device=g.device)
                _sgemm(g, 0, 1, N_, kc * N_, 0, xr, 0, 1, K_, kc * K_, 0, part, 0, K_, 1, N_ * K_, 0, N_, K_, kc, batch=ks)
                if tail:
                    _sgemm(g, ks * kc * N_, 1, N_, 0, 0, xr, ks * kc * K_, 1, K_, 0, 0, part, ks * N_ * K_, K_, 1, 0, 0, N_, K_, tail)
                dw = part.sum(0) if part.shape[0] > 1 else part[0]
            if need_b:
                db = g.sum(0)
        if dx is not None:
            if pre_relu:
                # relu(x) > 0  <=>  its bf16 hi plane is a positive number
                dx = dx * ((x2 > 0) if x2 is not None else (a_hi[:, :K_] > 0))
            dx = dx.reshape(xshape)
        return dx, dw, db, None, dres, None


def linear(x, weight, bias=None, act: Optional[str] = None, residual=None, pre_relu: bool = False):
    """``act(relu?(x) @ weight.T + bias) + residual``; act in {None, 'relu', 'silu'}."""
    if act == "silu":
        y = torch.nn.functional.silu(_LinearFn.apply(x, weight, bias, None, None, pre_relu))
        return y if residual is None else y + residual
    return _LinearFn.apply(x, weight, bias, act, residual, pre_relu)


# --------------------------------------------------------------------------------------------------
# 5x5 (frame x residue) convolution, channels-last, implicit GEMM
# --------------------------------------------------------------------------------------------------
class _Conv5x5Fn(Function):
    @staticmethod
    @_on_device
    def forward(ctx, x, w, b, relu, residual, crop):
        _need_cuda(x, w, b, residual)
        F_, N_, Ci = x.shape
        Co, Ci2, kh, kw = w.shape
        if Ci2 != Ci or Ci % 8 or Co % 8:
            raise ValueError(f"conv5x5: channels must match and be multiples of 8 (got {Ci}->{Co})")
        Fo = F_ - crop                                   # only the last Fo frames are produced
        if Fo < 1:
            raise ValueError("conv5x5: crop removes every frame")
        x2 = _f32c(x.reshape(F_ * N_, Ci))
        r2 = _f32c(residual.reshape(Fo * N_, Co)) if residual is not None else None
        out = torch.empty((Fo * N_, Co), dtype=torch.float32, device=x.device)
        (a_hi, a_lo), _ = _split2d(x2)
        f_hi, f_lo, _, _ = _conv_planes(w)
        _gemm(a_hi, a_lo, F_, N_, Ci, Ci, f_hi, f_lo, Co, f_hi.shape[2], kh, kw, out, Co, _f32c(b) if b is not None else None,
              r2, Co, 1.0, 1.0, 1 if relu else 0, F_out=Fo, f_start=crop)
        ctx.save_for_backward(a_hi, a_lo, w, out if relu else None, r2 if relu else None)
        ctx.meta = (x.shape, relu, b is not None, residual is not None, crop)
        ctx.w_param = w if isinstance(w, torch.nn.Parameter) else None
        return out.reshape(Fo, N_, Co)

    @staticmethod
    @_on_device
    def backward(ctx, dy):
        x_hi, x_lo, w, out, r2 = ctx.saved_tensors
        (F_, N_, Ci), relu, has_b, has_r, crop = ctx.meta
        Co, _, kh, kw = w.shape
        Fo = F_ - crop
        g = _f32c(dy.reshape(Fo * N_, Co))
        need_x, need_w, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1], has_b and ctx.needs_input_grad[2]
        dx = dw = db = None
        db_buf = torch.zeros(Co, dtype=torch.float32, device=g.device) if need_b else None
        (g_hi, g_lo), _ = _split2d(g, gate=out, gate_sub=r2, want=need_x or need_w, colsum=db_buf)
        db = db_buf
        acc = None
        if need_w and GRAD_ACCUMULATE_INPLACE and ctx.w_param is not None:
            acc = ctx.w_param.grad
            if not (acc is not None and acc.dtype == torch.float32 and acc.is_contiguous() and acc.shape == w.shape
                    and acc.device == g.device):
                acc = None
        wgrad = lambda out_, add: _conv_wgrad(g_hi, g_lo, x_hi, x_lo, Co, Ci, kh, kw, F_, Fo, N_, crop, out_, add)
        side = acc is not None and PROFILE is None
        if side:
            # the weight gradient only adds into the parameter's .grad: it overlaps the data gradient and the rest of the
            # backward, which never read it
            with _on_side_stream(g.device, (g_hi, g_lo, x_hi, x_lo)):
                wgrad(acc, 1)
        if need_x:
            _, _, d_hi, d_lo = _conv_planes(w)
            dx = torch.empty((F_ * N_, Ci), dtype=torch.float32, device=g.device)
            _gemm(g_hi, g_lo, Fo, N_, Co, Co, d_hi, d_lo, Ci, d_hi.shape[2], kh, kw, dx, Ci, None, None, 0, 1.0, 0.0, 0,
                  F_out=F_, f_start=-crop)
            dx = dx.reshape(F_, N_, Ci)
        if acc is not None and not side:
            wgrad(acc, 1)
        elif need_w and acc is None:
            dw = torch.empty((Co, Ci, kh, kw), dtype=torch.float32, device=g.device)
            wgrad(dw, 0)
        return dx, dw, db, None, (dy if has_r else None), None


def _conv_wgrad(g_hi, g_lo, x_hi, x_lo, Co, Ci, kh, kw, F_, Fo, N_, crop, out, add):
    """Weight gradient of the convolution: the per-tap GEMMs into a [taps, Co, Ci] scratch (allocated on the current
    stream), then added into (add=1) or written to (add=0) ``out`` [Co, Ci, kh, kw]."""
    taps = torch.empty((kh * kw, Co, Ci), dtype=torch.float32, device=out.device)
    _gemm_wgrad((g_hi, g_lo), Co, Co, (x_hi, x_lo), Ci, Ci, Fo, N_, kh, kw, taps, Ci, Fb=F_, b_f_add=crop)
    launch("dfold_taps_to_param", taps, Co, Ci, kh * kw, out, add)


def conv5x5(x, weight, bias=None, relu: bool = True, residual=None, crop: int = 0):
    """Channels-last ``Conv2d(kernel 5, padding 2)`` over the (frame, residue) image: x [F, N, C_in] ->
    ``relu?(conv(x) + bias) + residual`` [F, N, C_out]; weight keeps the reference's [C_out, C_in, 5, 5] layout.
    ``crop > 0`` produces only the last ``F - crop`` output frames (residual must have that many frames)."""
    return _Conv5x5Fn.apply(x, weight, bias, relu, residual, crop)


# --------------------------------------------------------------------------------------------------
# norms
# --------------------------------------------------------------------------------------------------
class _GlobalLNFn(Function):
    @staticmethod
    @_on_device
    def forward(ctx, x, eps, silu):
        _need_cuda(x)
        xc = _f32c(x)
        y = torch.empty_like(xc)
        stats = torch.empty(2, dtype=torch.float32, device=x.device)
        ws = torch.empty(2048 + 2, dtype=torch.float64, device=x.device)
        launch("dfold_global_layernorm_fwd", xc, y, stats, ws, xc.numel(), eps, int(silu))
        ctx.save_for_backward(xc, stats)
        ctx.silu = silu
        return y

    @staticmethod
    @_on_device
    def backward(ctx, dy):
        xc, stats = ctx.saved_tensors
        g = _f32c(dy)
        dx = torch.empty_like(xc)
        ws = torch.empty(2048 + 2, dtype=torch.float64, device=xc.device)
        launch("dfold_global_layernorm_bwd", xc, g, stats, ws, dx, xc.numel(), int(ctx.silu))
        return dx, None, None


def global_layernorm(x, eps: float = 1e-4, silu: bool = False):
    """MyLayerNorm: one mean / unbiased variance over the whole tensor, optional fused SiLU."""
    return _GlobalLNFn.apply(x, eps, silu)


class _RowLNFn(Function):
    @staticmethod
    @_on_device
    def forward(ctx, x, w, b, eps):
        _need_cuda(x, w, b)
        C = x.shape[-1]
        x2 = _f32c(x.reshape(-1, C))
        y = torch.empty_like(x2)
        stats = torch.empty((x2.shape[0], 2), dtype=torch.float32, device=x.device)
        wc, bc = _f32c(w), _f32c(b)
        launch("dfold_row_layernorm_fwd", x2, wc, bc, y, stats, x2.shape[0], C, eps)
        ctx.save_for_backward(x2, w, stats)
        ctx.shape = x.shape
        return y.reshape(x.shape)

    @staticmethod
    @_on_device
    def backward(ctx, dy):
        x2, w, stats = ctx.saved_tensors
        C = x2.shape[1]
        g = _f32c(dy.reshape(-1, C))
        dx = torch.empty_like(x2)
        dw = torch.zeros(C, dtype=torch.float32, device=x2.device)
        db = torch.zeros(C, dtype=torch.float32, device=x2.device)
        wc = _f32c(w)
        launch("dfold_row_layernorm_bwd", x2, wc, g, stats, dx, dw, db, x2.shape[0], C)
        return dx.reshape(ctx.shape), dw, db, None


def layer_norm(x, weight, bias, eps: float = 1e-5):
    return _RowLNFn.apply(x, weight, bias, eps)


# --------------------------------------------------------------------------------------------------
# rigid algebra
# --------------------------------------------------------------------------------------------------
class _QuatToRotFn(Function):
    @staticmethod
    @_on_device
    def forward(ctx, q):
        _need_cuda(q)
        qc = _f32c(q)
        n = qc.numel() // 4
        R = torch.empty(qc.shape[:-1] + (3, 3), dtype=torch.float32, device=q.device)
        launch("dfold_quat_to_rot_fwd", qc, R, n)
        ctx.save_for_backward(qc)
        return R

    @staticmethod
    @_on_device
    def backward(ctx, dR):
        (qc,) = ctx.saved_tensors
        dq = torch.empty_like(qc)
        gR = _f32c(dR)
        launch("dfold_quat_to_rot_bwd", qc, gR, dq, qc.numel() // 4)
        return dq


def quat_to_rot(q):
    if q.numel() == 0:
        return q.new_zeros(q.shape[:-1] + (3, 3))
    return _QuatToRotFn.apply(q)


class _RigidApplyFn(Function):
    """quat [F,N,4], trans [F,N,3], pts [Fp,N,m,3] with Fp in {1, F} -> [F,N,m,3]."""

    @staticmethod
    @_on_device
    def forward(ctx, quat, trans, pts, inverse):
        F_, N_ = quat.shape[0], quat.shape[1]
        m = pts.shape[2]
        out = torch.empty((F_, N_, m, 3), dtype=torch.float32, device=quat.device)
        fs = 0 if pts.shape[0] == 1 else N_ * m * 3
        launch("dfold_rigid_apply_fwd", quat, trans, pts, fs, out, F_, N_, m, int(inverse))
        ctx.save_for_backward(quat, trans, pts)
        ctx.inverse = inverse
        return out

    @staticmethod
    @_on_device
    def backward(ctx, dout):
        quat, trans, pts = ctx.saved_tensors
        F_, N_ = quat.shape[0], quat.shape[1]
        m = pts.shape[2]
        fs = 0 if pts.shape[0] == 1 else N_ * m * 3
        dpts = torch.empty((F_, N_, m, 3), dtype=torch.float32, device=quat.device)
        dq = torch.empty_like(quat)
        dt = torch.empty_like(trans)
        gout = _f32c(dout)
        launch("dfold_rigid_apply_bwd", quat, trans, pts, fs, gout, dpts, dq, dt, F_, N_, m, int(ctx.inverse))
        if pts.shape[0] == 1 and F_ > 1:
            dpts = dpts.sum(0, keepdim=True)
        return dq, dt, dpts, None


def rigid_apply(quat, trans, pts, inverse: bool = False):
    """Apply frames (quaternion form) to points: ``R p + t`` or ``R^T (p - t)``.

    quat [*,4], trans [*,3], pts [*, 3] broadcastable with one extra trailing point axis allowed
    (the ``r[..., None].apply(pts)`` idiom)."""
    _need_cuda(quat, trans, pts)
    bshape = torch.broadcast_shapes(quat.shape[:-1], pts.shape[:-1])
    if any(d == 0 for d in bshape):
        return pts.new_zeros(bshape + (3,))
    fdims = quat.dim() - 1
    # frames = leading dims of quat that are not broadcast singleton; points = the rest
    lead = bshape[:fdims]
    # split lead into (frames with real quats) and trailing singleton dims of quat that the points fan out over
    k = fdims
    while k > 0 and quat.shape[k - 1] == 1 and bshape[k - 1] != 1:
        k -= 1
    fshape = tuple(bshape[:k])
    mshape = tuple(bshape[k:])
    nfr = 1
    for d in fshape:
        nfr *= d
    m = 1
    for d in mshape:
        m *= d
    q2 = _f32c(quat.expand(fshape + (1,) * (fdims - k) + (4,)).reshape(1, max(nfr, 1), 4))
    t2 = _f32c(trans.expand(fshape + (1,) * (fdims - k) + (3,)).reshape(1, max(nfr, 1), 3))
    p2 = _f32c(pts.expand(bshape + (3,)).reshape(1, max(nfr, 1), m, 3))
    out = _RigidApplyFn.apply(q2, t2, p2, inverse)
    return out.reshape(bshape + (3,))


def ipa_points(raw, quat, trans, H: int):
    """raw [Fs,N,3*H*P] (all x, then all y, then all z) -> global-frame points [F,N,H,P,3]."""
    Fs, N_, W = raw.shape
    hp = W // 3
    pts = raw.reshape(Fs, N_, 3, hp).transpose(-1, -2).contiguous()          # [Fs,N,H*P,3]
    out = _RigidApplyFn.apply(_f32c(quat), _f32c(trans), _f32c(pts), False)  # [F,N,H*P,3]
    return out.reshape(out.shape[0], N_, H, hp // H, 3)


class _ComposeFn(Function):
    @staticmethod
    @_on_device
    def forward(ctx, quat, trans, upd, mask):
        _need_cuda(quat, trans, upd, mask)
        qc, tc, uc = _f32c(quat), _f32c(trans), _f32c(upd)
        mc = _f32c(mask.expand(quat.shape[:-1] + (1,))) if mask is not None else None
        n = qc.numel() // 4
        qo, to = torch.empty_like(qc), torch.empty_like(tc)
        launch("dfold_compose_q_update_fwd", qc, tc, uc, mc, qo, to, n)
        ctx.save_for_backward(qc, uc, mc)
        return qo, to

    @staticmethod
    @_on_device
    def backward(ctx, dqo, dto):
        qc, uc, mc = ctx.saved_tensors
        n = qc.numel() // 4
        dq, dt, du = torch.empty_like(qc), torch.empty(qc.shape[:-1] + (3,), dtype=torch.float32, device=qc.device), torch.empty_like(uc)
        gq, gt = _f32c(dqo), _f32c(dto)    # both must stay alive: two temporaries may otherwise share one block
        launch("dfold_compose_q_update_bwd", qc, uc, mc, gq, gt, dq, dt, du, n)
        return dq, dt, du, None


def compose_q_update(quat, trans, upd6, mask=None):
    """Backbone update: q' = normalise(q + m q*(0,u)), t' = t + m R(q) v with upd6 = (u, v); mask [...,1] or None."""
    return _ComposeFn.apply(quat, trans, upd6, mask)


def keep_last_frame(x):
    """x with every leading-axis slice but the last replaced by zeros (reference ``rigid_update[:-1] *= 0``)."""
    return torch.cat([torch.zeros_like(x[:-1]), x[-1:]], dim=0)


# --------------------------------------------------------------------------------------------------
# invariant point attention
# --------------------------------------------------------------------------------------------------
class _QKLogitsFn(Function):
    """logit0[f,h,i,j] = alpha * q[f,i,h,:] . k[f,j,h,:] + beta * b[f,h,i,j]   (k = first C of each kv head)."""

    @staticmethod
    @_on_device
    def forward(ctx, q, kv, b_hm, alpha, beta):
        _need_cuda(q, kv, b_hm)
        Fs, N_, H_, C_ = q.shape
        Fz = b_hm.shape[0]
        Fl = max(Fs, Fz)
        q, kv = _f32c(q), _f32c(kv)
        out = torch.empty((Fl, H_, N_, N_), dtype=torch.float32, device=q.device)
        sb = b_hm.stride()
        for f in range(Fl):
            fq, fz = (f if Fs > 1 else 0), (f if Fz > 1 else 0)
            _sgemm(q, fq * N_ * H_ * C_, H_ * C_, 1, C_, 0, kv, fq * N_ * H_ * 2 * C_, H_ * 2 * C_, 1, 2 * C_, 0,
                   out, f * H_ * N_ * N_, N_, 1, N_ * N_, 0, N_, N_, C_,
                   R=b_hm, r_off=fz * sb[0], r_rs=sb[2], r_cs=sb[3], r_bs=sb[1],
                   batch=H_, alpha=alpha, beta=beta)
        ctx.save_for_backward(q, kv)
        ctx.meta = (alpha, beta, Fz, tuple(b_hm.shape))
        return out

    @staticmethod
    @_on_device
    def backward(ctx, dl):
        q, kv = ctx.saved_tensors
        alpha, beta, Fz, bshape = ctx.meta
        Fs, N_, H_, C_ = q.shape
        dl = _f32c(dl)
        Fl = dl.shape[0]
        dq = torch.zeros_like(q)
        dkv = torch.zeros_like(kv)
        if Fs == 1 and Fl > 1:
            dls = dl.sum(0, keepdim=True)
        else:
            dls = dl
        for f in range(Fs):
            # dq[n,h,c] = alpha sum_j dl[h,n,j] k[j,h,c]
            _sgemm(dls, f * H_ * N_ * N_, N_, 1, N_ * N_, 0, kv, f * N_ * H_ * 2 * C_, 1, H_ * 2 * C_, 2 * C_, 0,
                   dq, f * N_ * H_ * C_, H_ * C_, 1, C_, 0, N_, C_, N_, batch=H_, alpha=alpha)
            # dk[j,h,c] = alpha sum_n dl[h,n,j] q[n,h,c]
            _sgemm(dls, f * H_ * N_ * N_, 1, N_, N_ * N_, 0, q, f * N_ * H_ * C_, 1, H_ * C_, C_, 0,
                   dkv, f * N_ * H_ * 2 * C_, H_ * 2 * C_, 1, 2 * C_, 0, N_, C_, N_, batch=H_, alpha=alpha)
        db = beta * (dl if Fz > 1 or Fl == 1 else dl.sum(0, keepdim=True))
        return dq, dkv, db.reshape(bshape) if db.shape != bshape else db, None, None


def qk_logits(q, kv, b_hm, alpha: float, beta: float):
    """Scalar part of the IPA logits, head-major [F,H,N,N].  q [Fs,N,H,C]; kv [Fs,N,H,2C]; b_hm [Fz,H,N,N] (any strides)."""
    return _QKLogitsFn.apply(q, kv, b_hm, alpha, beta)


class _IpaAttnFn(Function):
    @staticmethod
    @_on_device
    def forward(ctx, logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, Pq, Pv, dfold, inf, eps):
        _need_cuda(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma)
        logit0, kv, q_pts, kv_pts, pair = _f32c(logit0), _f32c(kv), _f32c(q_pts), _f32c(kv_pts), _f32c(pair)
        quat, trans, mask, gamma = _f32c(quat), _f32c(trans), _f32c(mask), _f32c(gamma)
        F_, N_, H_ = q_pts.shape[0], q_pts.shape[1], q_pts.shape[2]
        C_ = kv.shape[-1] // 2
        Cp = pair.shape[-1]
        D = H_ * (C_ + (8 if dfold else 4) * Pv + Cp)
        cat = torch.empty((F_, N_, D), dtype=torch.float32, device=q_pts.device)
        lse = torch.empty((F_, H_, N_), dtype=torch.float32, device=q_pts.device)
        args = _IpaAttnFn._args(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, F_, N_, H_, C_, Pq, Pv, Cp, dfold, inf, eps)
        # algorithmic fp32 bytes of the fused core (SURVEY.md §8d): per-frame q/k/v/points/rigids/mask in, concat out,
        # plus the per-sample pair bias and pair values
        alg_bytes = 4.0 * (F_ * N_ * (H_ * (4 * C_ + 3 * (2 * Pq + Pv) + 8 * Pv + Cp) + 8) + N_ * N_ * (H_ + Cp))
        with _timed("ipa_fwd", alg_bytes):
            launch("dfold_ipa_attn_fwd", *args, cat, lse)
        ctx.save_for_backward(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, cat, lse)
        ctx.meta = (Pq, Pv, dfold, inf, eps)
        return cat

    @staticmethod
    def _args(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, F_, N_, H_, C_, Pq, Pv, Cp, dfold, inf, eps):
        l_fs = 0 if logit0.shape[0] == 1 else H_ * N_ * N_
        kv_fs = 0 if kv.shape[0] == 1 else N_ * H_ * 2 * C_
        p_fs = 0 if pair.shape[0] == 1 else N_ * N_ * Cp
        return (logit0, l_fs, kv, kv_fs, q_pts, kv_pts, pair, p_fs, quat, trans, mask, gamma, F_, N_, H_, C_, Pq, Pv, Cp, int(dfold),
                inf, eps)

    @staticmethod
    @_on_device
    def backward(ctx, dcat):
        logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, cat, lse = ctx.saved_tensors
        Pq, Pv, dfold, inf, eps = ctx.meta
        F_, N_, H_ = q_pts.shape[0], q_pts.shape[1], q_pts.shape[2]
        C_ = kv.shape[-1] // 2
        Cp = pair.shape[-1]
        PQ3, PV3 = 3 * Pq, 3 * Pv
        D = cat.shape[-1]
        dev = cat.device
        dcat = _f32c(dcat)
        new = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        d_og, delta = new(F_, N_, H_, Pv, 3), new(F_, H_, N_)
        Pm, dS = new(H_, F_, N_, N_), new(H_, F_, N_, N_)
        dq_pts, dkv_pts = new(*q_pts.shape), new(*kv_pts.shape)
        dquat, dtrans = new(*quat.shape), new(*trans.shape)
        dgamma_part = torch.zeros(H_, F_ * N_, dtype=torch.float32, device=dev)      # per-CTA partials, summed in order
        args = _IpaAttnFn._args(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, F_, N_, H_, C_, Pq, Pv, Cp, dfold, inf, eps)
        launch("dfold_ipa_attn_bwd", *args, cat, lse, dcat, d_og, delta, Pm, dS, dq_pts, dkv_pts, dquat, dtrans, dgamma_part)
        dgamma = dgamma_part.sum(1)
        NN = N_ * N_
        # ---- value gradient  dv[j,h,c] = sum_{f,i} P[h,f,i,j] dO[f,i,h,c] ----
        Fs = kv.shape[0]
        dkv = torch.zeros_like(kv)
        if Fs == 1:
            _sgemm(Pm, 0, 1, N_, F_ * NN, 0, dcat, 0, 1, D, C_, 0, dkv, C_, H_ * 2 * C_, 1, 2 * C_, 0,
                   N_, C_, F_ * N_, batch=H_)
        else:
            _sgemm(Pm, 0, 1, N_, F_ * NN, NN, dcat, 0, 1, D, C_, N_ * D, dkv, C_, H_ * 2 * C_, 1, 2 * C_, N_ * H_ * 2 * C_,
                   N_, C_, N_, batch=H_, batch2=F_)
        # ---- value-point gradient  dvp[f,j,h,e] = sum_i P[h,f,i,j] d_og[f,i,h,e] ----
        W = PQ3 + PV3
        _sgemm(Pm, 0, 1, N_, F_ * NN, NN, d_og, 0, 1, H_ * PV3, PV3, N_ * H_ * PV3, dkv_pts, PQ3, H_ * W, 1, W, N_ * H_ * W,
               N_, PV3, N_, batch=H_, batch2=F_)
        # ---- pair gradient  dz[i,j,c] = sum_{h,f} P[h,f,i,j] dOpair[f,i,h,c] ----
        offPair = H_ * C_ + 4 * H_ * Pv
        dop = dcat[..., offPair:offPair + H_ * Cp].reshape(F_, N_, H_, Cp)
        Fz = pair.shape[0]
        dpair = torch.empty_like(pair)
        if Fz == 1:
            dop_hf = dop.permute(2, 0, 1, 3).contiguous()                     # [H,F,N,Cp]
            _sgemm(Pm, 0, 1, NN, N_, 0, dop_hf, 0, 1, N_ * Cp, Cp, 0, dpair, 0, Cp, 1, N_ * Cp, 0, N_, Cp, H_ * F_, batch=N_)
        else:
            dop_fh = dop.permute(0, 2, 1, 3).contiguous()                     # [F,H,N,Cp]
            _sgemm(Pm, 0, 1, F_ * NN, NN, N_, dop_fh, 0, 1, N_ * Cp, H_ * N_ * Cp, Cp, dpair, 0, Cp, 1, NN * Cp, N_ * Cp,
                   N_, Cp, H_, batch=F_, batch2=N_)
        # ---- logits ----
        if logit0.shape[0] == 1:
            dlogit0 = dS.sum(1).unsqueeze(0)
        else:
            dlogit0 = dS.permute(1, 0, 2, 3).contiguous()
        return dlogit0, dkv, dq_pts, dkv_pts, dpair, dquat, dtrans, None, dgamma, None, None, None, None, None


def _planes_rows(x2):
    """bf16 hi/lo planes of a contiguous [R, C] fp32 matrix -> ([R, C8], [R, C8])."""
    (hi, lo), _ = _split2d(x2)
    return hi, lo


class _IpaAttnTCFn(Function):
    """Tensor-core decomposition of the IPA core (csrc/ipa_fused.cu + csrc/ipa_v2.cu + csrc/gemm_sm90.cu) for the preset-A
    head geometry with shared (frame-invariant) q/k/v and pair tensors — the DFOLDv2 case.  Probabilities are materialised
    once as bf16 hi/lo planes."""

    @staticmethod
    @_on_device
    def forward(ctx, logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, Pq, Pv, dfold, inf, eps):
        _need_cuda(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma)
        logit0, kv, q_pts, kv_pts, pair = _f32c(logit0), _f32c(kv), _f32c(q_pts), _f32c(kv_pts), _f32c(pair)
        quat, trans, mask, gamma = _f32c(quat), _f32c(trans), _f32c(mask), _f32c(gamma)
        F_, N_, H_ = q_pts.shape[0], q_pts.shape[1], q_pts.shape[2]
        C_ = kv.shape[-1] // 2
        Cp = pair.shape[-1]
        D = H_ * (C_ + (8 if dfold else 4) * Pv + Cp)
        dev = q_pts.device
        n8 = _pad8(N_)
        cat = torch.empty((F_, N_, D), dtype=torch.float32, device=dev)
        # the probability planes feed the P V GEMM and the backward GEMMs
        p_hi = torch.empty((F_, H_, N_, n8), dtype=torch.int16, device=dev)
        p_lo = torch.empty((F_, H_, N_, n8), dtype=torch.int16, device=dev)
        alg_bytes = 4.0 * (F_ * N_ * (H_ * (4 * C_ + 3 * (2 * Pq + Pv) + 8 * Pv + Cp) + 8) + N_ * N_ * (H_ + Cp))
        with _timed("ipa_fwd", alg_bytes):
            # one kernel: distances, exact softmax, pair + value-point aggregation, frame transform, P planes
            launch("dfold_ipa_fused_fwd", logit0, q_pts, kv_pts, pair, quat, trans, mask, gamma, p_hi, p_lo, n8,
                   F_, N_, H_, C_, Pq, Pv, Cp, int(dfold), inf, eps, cat)
            # O = P V  on the tensor cores, written into the o-columns of the concat buffer
            vt = kv[0, :, :, C_:].permute(1, 2, 0).reshape(H_ * C_, N_).contiguous()        # [H*C, N]
            vt_hi, vt_lo = _planes_rows(vt)
            launch("dfold_gemm_bf16x3_batched",
                   p_hi, p_lo, F_ * H_, N_, N_, n8, F_ * H_, H_, 1, 0, N_,
                   vt_hi, vt_lo, H_, C_, N_, vt_hi.shape[1], 0, 0, 1, C_,
                   cat, D, F_ * N_, H_, C_, 1.0)
        ctx.save_for_backward(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, cat, p_hi, p_lo)
        ctx.meta = (Pq, Pv, dfold, inf, eps)
        return cat

    @staticmethod
    @_on_device
    def backward(ctx, dcat):
        logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, cat, p_hi, p_lo = ctx.saved_tensors
        Pq, Pv, dfold, inf, eps = ctx.meta
        F_, N_, H_ = q_pts.shape[0], q_pts.shape[1], q_pts.shape[2]
        C_ = kv.shape[-1] // 2
        Cp = pair.shape[-1]
        PQ3, PV3 = 3 * Pq, 3 * Pv
        W = PQ3 + PV3
        D = cat.shape[-1]
        dev = cat.device
        n8 = p_hi.shape[-1]
        dcat = _f32c(dcat)
        new = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        d_og, delta = new(F_, N_, H_, Pv, 3), new(F_, H_, N_)
        dquat, dtrans = new(*quat.shape), new(*trans.shape)
        launch("dfold_ipa_pre_bwd", quat, trans, F_, N_, H_, C_, Pv, Cp, int(dfold), cat, dcat, d_og, delta, dquat, dtrans)
        # ---- dP = dO V^T  (batched over (f, h); K = the head's C columns of dO) ----
        dc_hi, dc_lo = _planes_rows(dcat.reshape(F_ * N_, D))                       # [F*N, D8]
        kv_hi, kv_lo = _planes_rows(kv.reshape(N_, H_ * 2 * C_))                    # [N, H*2C]
        dP = new(F_, H_, N_, N_)
        launch("dfold_gemm_bf16x3_batched",
               dc_hi, dc_lo, F_, N_, D, dc_hi.shape[1], F_ * H_, H_, H_, C_, C_,
               kv_hi, kv_lo, 1, N_, H_ * 2 * C_, kv_hi.shape[1], C_, 2 * C_, 0, N_,
               dP, N_, F_ * H_ * N_, 1, 0, 1.0)
        # ---- pair term of dP on the tensor cores:  Tz[i][f*H+h][j] = sum_c dOpair[f,i,h,c] z[i,j,c]  (batched over i) ----
        offPair = H_ * C_ + 4 * H_ * Pv
        dop = dcat[..., offPair:offPair + H_ * Cp].reshape(F_, N_, H_, Cp).permute(1, 0, 2, 3).reshape(N_ * F_ * H_, Cp).contiguous()
        do_hi, do_lo = _planes_rows(dop)                                           # [N*F*H, Cp8]  rows (i, f, h)
        z_hi, z_lo = _planes_rows(pair.reshape(N_ * N_, Cp))                       # [N*N, Cp8]    rows (i, j)
        Tz = new(N_, F_ * H_, N_)
        launch("dfold_gemm_bf16x3_batched",
               do_hi, do_lo, N_, F_ * H_, Cp, do_hi.shape[1], N_, N_, 1, 0, Cp,
               z_hi, z_lo, N_, N_, Cp, z_hi.shape[1], 0, 0, 1, N_,
               Tz, N_, N_ * F_ * H_, 1, 0, 1.0)
        # ---- dS, d(gamma), point gradients ----
        dS = new(F_, H_, N_, N_)
        dgamma_part = torch.zeros(H_, F_ * N_, dtype=torch.float32, device=dev)      # per-CTA partials, summed in order
        dq_pts, dkv_pts = new(*q_pts.shape), new(*kv_pts.shape)
        # rows (f, h, i) of the value-point output gradient: operand of dV_pts below and of the value-point term of dP here
        dg = d_og.reshape(F_, N_, H_, PV3).permute(0, 2, 1, 3).reshape(F_ * H_ * N_, PV3).contiguous()
        dg_hi, dg_lo = _planes_rows(dg)
        # d_og . v_pts on the tensor cores: Tog[(f,h,i), j] = sum_e dg[(f,h,i), e] v_pts[(f,h,j), e]
        vp = kv_pts.reshape(F_, N_, H_, W)[..., PQ3:].permute(0, 2, 1, 3).reshape(F_ * H_ * N_, PV3).contiguous()
        vp_hi, vp_lo = _planes_rows(vp)
        Tog = new(F_ * H_ * N_, N_)
        launch("dfold_gemm_bf16x3_batched",
               dg_hi, dg_lo, F_ * H_, N_, PV3, dg_hi.shape[1], F_ * H_, F_ * H_, 1, 0, PV3,
               vp_hi, vp_lo, F_ * H_, N_, PV3, vp_hi.shape[1], 0, 0, 1, N_,
               Tog, N_, F_ * H_ * N_, 1, 0, 1.0)
        launch("dfold_ipa_ds_bwd", q_pts, kv_pts, p_hi, p_lo, n8, F_, N_, H_, Pq, Pv, delta, dP, Tz, Tog, dS, dgamma_part)
        dgamma = dgamma_part.sum(1)
        del Tz
        del dP
        del Tog
        # Point gradients as two small tensor-core contractions over dS:
        #   dq_pts[i] = -gamma (q_i rowsum_i - sum_j dS_ij k_j),   dk_pts[j] = gamma (sum_i dS_ij q_i - colsum_j k_j)
        # with a ones column appended to the point operands (3 Pq = 24 coordinates + 1, padded to 32 columns) so the
        # row / column sums fall out of the same products.
        ds_hi, ds_lo = _planes_rows(dS.reshape(F_ * H_ * N_, N_))                                   # [F*H*N, n8]
        kq = kv_pts.reshape(F_, N_, H_, W)[..., :PQ3]
        kt = torch.zeros((F_, H_, 32, N_), dtype=torch.float32, device=dev)
        kt[:, :, :PQ3] = kq.permute(0, 2, 3, 1)
        kt[:, :, PQ3] = 1.0
        kt_hi, kt_lo = _planes_rows(kt.reshape(F_ * H_ * 32, N_))                                   # [F*H*32, n8]
        g1 = new(F_ * H_ * N_, 32)
        launch("dfold_gemm_bf16x3_batched",
               ds_hi, ds_lo, F_ * H_, N_, N_, ds_hi.shape[1], F_ * H_, F_ * H_, 1, 0, N_,
               kt_hi, kt_lo, F_ * H_, 32, N_, kt_hi.shape[1], 0, 0, 1, 32,
               g1, 32, F_ * H_ * N_, 1, 0, 1.0)
        qn = torch.zeros((F_, H_, N_, 32), dtype=torch.float32, device=dev)
        qh = q_pts.reshape(F_, N_, H_, PQ3).permute(0, 2, 1, 3)                                     # [F,H,N,24]
        qn[..., :PQ3] = qh
        qn[..., PQ3] = 1.0
        qn_hi, qn_lo = _planes_rows(qn.reshape(F_ * H_ * N_, 32))
        g2 = new(F_ * H_, N_, 32)
        launch("dfold_gemm_wgrad_bf16x3_batched",
               ds_hi, ds_lo, N_, N_, F_ * H_, ds_hi.shape[1], N_ * ds_hi.shape[1],
               qn_hi, qn_lo, 32, N_, F_ * H_, qn_hi.shape[1], N_ * qn_hi.shape[1],
               32, 1, N_, F_ * H_, 0, 1, 0, 1, 0,
               g2, 32, N_ * 32, 1.0)
        g1 = g1.reshape(F_, H_, N_, 32)
        gam = gamma.reshape(1, H_, 1, 1)
        dq = -gam * (qh * g1[..., PQ3:PQ3 + 1] - g1[..., :PQ3])
        dq_pts.copy_(dq.permute(0, 2, 1, 3).reshape(q_pts.shape))
        dk = gam * (g2[..., :PQ3].reshape(F_, H_, N_, PQ3) - g2[..., PQ3:PQ3 + 1].reshape(F_, H_, N_, 1) * kq.permute(0, 2, 1, 3))
        dkv_pts.reshape(F_, N_, H_, W)[..., :PQ3] = dk.permute(0, 2, 1, 3)
        # ---- dV[j,h,c] = sum_{f,i} P[f,h,i,j] dO[f,i,h,c]   (MN-major, K over all frames) ----
        dkv = torch.zeros_like(kv)
        launch("dfold_gemm_wgrad_bf16x3_batched",
               p_hi, p_lo, N_, N_, F_ * H_, n8, N_ * n8,
               dc_hi, dc_lo, D, N_, F_, dc_hi.shape[1], N_ * dc_hi.shape[1],
               C_, F_, N_, H_, H_, 1, 1, 0, C_,
               _ptr(dkv, C_), H_ * 2 * C_, 2 * C_, 1.0)
        # ---- dV_pts[f,j,h,e] = sum_i P[f,h,i,j] d_og[f,i,h,e] ----
        tmp = new(F_ * H_, N_, PV3)
        launch("dfold_gemm_wgrad_bf16x3_batched",
               p_hi, p_lo, N_, N_, F_ * H_, n8, N_ * n8,
               dg_hi, dg_lo, PV3, N_, F_ * H_, dg_hi.shape[1], N_ * dg_hi.shape[1],
               PV3, 1, N_, F_ * H_, 0, 1, 0, 1, 0,
               tmp, PV3, N_ * PV3, 1.0)
        dkv_pts.reshape(F_, N_, H_, W)[..., PQ3:] = tmp.reshape(F_, H_, N_, PV3).permute(0, 2, 1, 3)
        # ---- dZ[i,j,c] = sum_{f,h} P[f,h,i,j] dOpair[f,i,h,c] ----
        dpair = new(1, N_, N_, Cp)
        launch("dfold_gemm_wgrad_bf16x3_batched",
               p_hi, p_lo, N_, F_ * H_, N_, N_ * n8, n8,
               do_hi, do_lo, Cp, F_ * H_, N_, do_hi.shape[1], F_ * H_ * do_hi.shape[1],
               Cp, 1, F_ * H_, N_, 0, 1, 0, 1, 0,
               dpair, Cp, N_ * Cp, 1.0)
        dlogit0 = dS.sum(0, keepdim=True) if logit0.shape[0] == 1 else dS
        return dlogit0, dkv, dq_pts, dkv_pts, dpair, dquat, dtrans, None, dgamma, None, None, None, None, None


def _tc_path_ok(logit0, kv, q_pts, pair, Pq, Pv) -> bool:
    """The tensor-core decomposition is built for the DFOLDv2 preset-A head geometry (H 8, Pq 8, Pv 12, Cp 32: the fused
    forward csrc/ipa_fused.cu and the dS kernel csrc/ipa_v2.cu) and needs frame-shared logit0, q/k/v and pair tensors (the
    fused forward reads logit0 as one [H,N,N] with no frame stride), a head width that is a whole number of 64-wide K
    blocks and rows that fit in shared memory."""
    C_ = kv.shape[-1] // 2
    N_, H_ = q_pts.shape[1], q_pts.shape[2]
    return (H_ == 8 and Pq == 8 and Pv == 12 and pair.shape[-1] == 32 and logit0.shape[0] == 1
            and kv.shape[0] == 1 and pair.shape[0] == 1 and C_ % 64 == 0 and N_ <= 1280 and N_ % 8 == 0)


def ipa_attention(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, *, Pq, Pv, dfold, inf, eps):
    """IPA core -> concat buffer [F,N,D] in the reference's feature order.

    The preset-A head geometry with frame-shared logit0, q/k/v and pair, C % 64 == 0 and N <= 1280 (DFOLDv2) runs the tensor-core
    decomposition (csrc/ipa_fused.cu, csrc/ipa_v2.cu); every other shape runs the single fused CUDA-core kernel
    (csrc/ipa_attn.cu).  Both are this library's kernels."""
    if _tc_path_ok(logit0, kv, q_pts, pair, Pq, Pv):
        return _IpaAttnTCFn.apply(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, Pq, Pv, dfold, inf, eps)
    return _IpaAttnFn.apply(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, Pq, Pv, dfold, inf, eps)


# --------------------------------------------------------------------------------------------------
# score epilogue (K9), structure epilogue (K10), remaining rigid algebra — csrc/epilogue.cu
# --------------------------------------------------------------------------------------------------
class _ScoreFn(Function):
    """(q_pred, q_t, x_pred, x_t) -> (rot_score fp64 [...,3], trans_score [...,3]); see include/dfold_b200.h."""

    @staticmethod
    @_on_device
    def forward(ctx, q_pred, q_t, x_pred, x_t, t64, grid, mask, consts, trans_f64):
        _need_cuda(q_pred, q_t, x_pred, x_t, t64, grid, mask)
        q_pred, q_t = _f32c(q_pred), _f32c(q_t)
        x_pred, x_t = (_f32c(x_pred), _f32c(x_t)) if x_pred is not None else (None, None)
        mask = _f32c(mask) if mask is not None else None
        n = q_pred.numel() // 4
        rot = torch.empty(q_pred.shape[:-1] + (3,), dtype=torch.float64, device=q_pred.device)
        trs = None
        if x_pred is not None:
            trs = torch.empty(x_pred.shape[:-1] + (3,), dtype=torch.float64 if trans_f64 else torch.float32, device=q_pred.device)
        max_s, min_s, min_b, max_b, r3, ipa, L = consts
        launch("dfold_score_fwd", q_pred, q_t, x_pred, x_t, t64, grid, grid.numel(),
               max_s, min_s, min_b, max_b, r3, ipa, mask, L, n, rot, trs, int(trans_f64))
        ctx.save_for_backward(q_pred, q_t, x_pred, x_t, t64, grid, mask)
        ctx.meta = (consts, trans_f64)
        return rot, trs

    @staticmethod
    @_on_device
    def backward(ctx, d_rot, d_trs):
        q_pred, q_t, x_pred, x_t, t64, grid, mask = ctx.saved_tensors
        consts, trans_f64 = ctx.meta
        max_s, min_s, min_b, max_b, r3, ipa, L = consts
        n = q_pred.numel() // 4
        d_rot = d_rot.to(torch.float64).contiguous() if d_rot is not None else None
        d_trs = d_trs.to(torch.float64 if trans_f64 else torch.float32).contiguous() if d_trs is not None else None
        dq = torch.empty_like(q_pred)
        dx = torch.empty_like(x_pred) if x_pred is not None else None
        launch("dfold_score_bwd", q_pred, q_t, x_pred, x_t, t64, grid, grid.numel(),
               max_s, min_s, min_b, max_b, r3, ipa, mask, L, n, d_rot, d_trs, int(trans_f64), dq, dx)
        return dq, None, dx, None, None, None, None, None, None


def score_epilogue(q_pred, q_t, x_pred, x_t, t, grid, mask, *, max_sigma, min_sigma, min_b, max_b, r3_scale, ipa_scale, L=1000):
    """IGSO(3) rotation score (fp64) and VP-SDE translation score of the predicted frames against the noised ones at
    diffusion time ``t`` ([1] tensor), both multiplied by ``mask`` [...]; the translation score takes the dtype
    ``promote(float32, t.dtype)`` as the reference arithmetic does.  ``x_pred`` is the translation BEFORE unscaling."""
    t64 = t.reshape(-1)[:1].to(torch.float64)
    trans_f64 = t.dtype == torch.float64
    consts = (float(max_sigma), float(min_sigma), float(min_b), float(max_b), float(r3_scale), float(ipa_scale), int(L))
    return _ScoreFn.apply(q_pred, q_t, x_pred, x_t, t64, grid, mask, consts, trans_f64)


class _FramesToAtomsFn(Function):
    """Forward: ONE kernel.  Backward (atoms are not in the reference's training loss, train_DFOLD_dynamics.py:1367-1373,
    but stay differentiable): recomputation through ``eager`` — the same chain written with the differentiable rigid
    operators of this module — under enable_grad."""

    @staticmethod
    @_on_device
    def forward(ctx, rot, trans, alpha, aatype, tables, eager, want_frames, rot_is_matrix):
        _need_cuda(rot, trans, alpha, aatype)
        rotc, transc, alphac = _f32c(rot), _f32c(trans), _f32c(alpha)
        aac = aatype.to(torch.int64).contiguous()
        lead = aac.shape
        n = aac.numel()
        dev = rotc.device
        a14 = torch.empty(lead + (14, 3), dtype=torch.float32, device=dev)
        a37 = torch.empty(lead + (37, 3), dtype=torch.float32, device=dev)
        fr = torch.empty(lead + (8, 4, 4), dtype=torch.float32, device=dev) if want_frames else None
        launch("dfold_frames_to_atoms_fwd", rotc, int(rot_is_matrix), transc, alphac, aac,
               *[tables[k] for k in ("default_frames", "atom14_group", "atom14_mask", "atom14_pos", "atom37_to_atom14", "atom37_mask")],
               fr, a14, a37, n)
        ctx.save_for_backward(rotc, transc, alphac, aac)
        ctx.eager = eager
        ctx.want_frames = want_frames
        if want_frames:
            return a14, a37, fr
        return a14, a37

    @staticmethod
    @_on_device
    def backward(ctx, *gouts):
        rotc, transc, alphac, aac = ctx.saved_tensors
        with torch.enable_grad():
            ins = [t.detach().requires_grad_(True) for t in (rotc, transc, alphac)]
            outs = ctx.eager(ins[0], ins[1], ins[2], aac, ctx.want_frames)
            pairs = [(o, g) for o, g in zip(outs, gouts) if g is not None]
            grads = torch.autograd.grad([o for o, _ in pairs], ins, [g for _, g in pairs], allow_unused=True)
        return grads[0], grads[1], grads[2], None, None, None, None, None


def frames_to_atoms(rot, trans, alpha, aatype, tables, eager, want_frames=False, rot_is_matrix=False):
    """(backbone rotation [*,N,4] quaternion or [*,N,3,3], translation [*,N,3], torsions [*,N,7,2], aatype [*,N]) ->
    (atom14 [*,N,14,3], atom37 [*,N,37,3][, frames [*,N,8,4,4]])."""
    return _FramesToAtomsFn.apply(rot, trans, alpha, aatype, tables, eager, want_frames, rot_is_matrix)


class _QuatMulFn(Function):
    @staticmethod
    @_on_device
    def forward(ctx, a, b, b_is_vec):
        _need_cuda(a, b)
        shp = torch.broadcast_shapes(a.shape[:-1], b.shape[:-1])
        ac = _f32c(a.expand(shp + (4,)))
        bc = _f32c(b.expand(shp + (b.shape[-1],)))
        out = torch.empty(shp + (4,), dtype=torch.float32, device=a.device)
        n = out.numel() // 4
        if n:
            launch("dfold_quat_mul_fwd", ac, bc, out, n, int(b_is_vec))
        ctx.save_for_backward(ac, bc)
        ctx.meta = (a.shape, b.shape, b_is_vec)
        return out

    @staticmethod
    @_on_device
    def backward(ctx, g):
        ac, bc = ctx.saved_tensors
        ashape, bshape, b_is_vec = ctx.meta
        g = _f32c(g)
        da, db = torch.empty_like(ac), torch.empty_like(bc)
        n = ac.numel() // 4
        if n:
            launch("dfold_quat_mul_bwd", ac, bc, g, da, db, n, int(b_is_vec))
        return da.sum_to_size(ashape) if da.shape != ashape else da, db.sum_to_size(bshape) if db.shape != bshape else db, None


def quat_mul(a, b, b_is_vec: bool = False):
    """Hamilton product a (x) b; ``b_is_vec``: b [...,3] is the pure quaternion (0, b)."""
    return _QuatMulFn.apply(a, b, b_is_vec)


def _trailing_rep(a_lead, b_lead):
    """b_lead = a_lead[:k] + extra with a_lead[k:] all ones (the ``r[..., None].compose(x)`` idiom) -> numel(extra)."""
    if len(a_lead) != len(b_lead):
        return None
    k = len(a_lead)
    while k > 0 and a_lead[k - 1] == 1:
        k -= 1
    if tuple(a_lead[:k]) != tuple(b_lead[:k]):
        return None
    rep = 1
    for d in b_lead[k:]:
        rep *= d
    return rep


class _RotComposeFn(Function):
    """(Ra [A,3,3], ta [A,3]|None) o (Rb [B,3,3]|None, tb [B,3]|None); A broadcasts over trailing dims of B."""

    @staticmethod
    @_on_device
    def forward(ctx, Ra, ta, Rb, tb, inverse):
        _need_cuda(Ra, ta, Rb, tb)
        a_lead = tuple(Ra.shape[:-2])
        b_lead = tuple(Rb.shape[:-2]) if Rb is not None else tuple(tb.shape[:-1])
        if Rb is not None and tb is not None and tuple(tb.shape[:-1]) != b_lead:
            lead = torch.broadcast_shapes(b_lead, tb.shape[:-1])
            Rb, tb, b_lead = Rb.expand(lead + (3, 3)), tb.expand(lead + (3,)), tuple(lead)
        out_lead = tuple(torch.broadcast_shapes(a_lead, b_lead))
        rep = _trailing_rep(a_lead, out_lead) if len(a_lead) == len(out_lead) else None
        if rep is None or b_lead != out_lead:
            # general broadcast: materialise both sides at the output shape
            Ra_e, ta_e = Ra.expand(out_lead + (3, 3)), (ta.expand(out_lead + (3,)) if ta is not None else None)
            Rb = Rb.expand(out_lead + (3, 3)) if Rb is not None else None
            tb = tb.expand(out_lead + (3,)) if tb is not None else None
            rep = 1
        else:
            Ra_e, ta_e = Ra, (ta.expand(a_lead + (3,)) if ta is not None else None)
        Rac, tac = _f32c(Ra_e), (_f32c(ta_e) if ta_e is not None else None)
        Rbc, tbc = (_f32c(Rb) if Rb is not None else None), (_f32c(tb) if tb is not None else None)
        na = Rac.numel() // 9
        dev = Rac.device
        Ro = torch.empty(out_lead + (3, 3), dtype=torch.float32, device=dev) if Rbc is not None else None
        to = torch.empty(out_lead + (3,), dtype=torch.float32, device=dev) if tbc is not None else None
        if na:
            launch("dfold_rot_compose_fwd", Rac, tac, Rbc, tbc, Ro, to, na, rep, int(inverse))
        ctx.save_for_backward(Rac, tac, Rbc, tbc)
        ctx.meta = (tuple(Ra.shape), tuple(ta.shape) if ta is not None else None, tuple(Rb.shape) if Rb is not None else None,
                    tuple(tb.shape) if tb is not None else None, rep, inverse, na)
        return Ro, to

    @staticmethod
    @_on_device
    def backward(ctx, dRo, dto):
        Rac, tac, Rbc, tbc = ctx.saved_tensors
        Ra_s, ta_s, Rb_s, tb_s, rep, inverse, na = ctx.meta
        dev = Rac.device
        dRo = _f32c(dRo) if (dRo is not None and Rbc is not None) else None
        dto = _f32c(dto) if (dto is not None and tbc is not None) else None
        dRa = torch.empty_like(Rac)
        dta = torch.empty_like(tac) if tac is not None else None
        dRb = torch.empty_like(Rbc) if Rbc is not None else None
        dtb = torch.empty_like(tbc) if tbc is not None else None
        if na:
            launch("dfold_rot_compose_bwd", Rac, tac, Rbc, tbc, dRo, dto, dRa, dta, dRb, dtb, na, rep, int(inverse))

        def fit(g, shape):
            if g is None or shape is None:
                return None
            return g.sum_to_size(shape) if tuple(g.shape) != tuple(shape) else g
        return fit(dRa, Ra_s), fit(dta, ta_s), fit(dRb, Rb_s), fit(dtb, tb_s), None


def rot_compose(Ra, ta, Rb, tb, inverse: bool = False):
    """Rotation-matrix frames: returns (Ra Rb | None, Ra tb + ta | None); ``inverse``: Ra^T (tb - ta)."""
    return _RotComposeFn.apply(Ra, ta, Rb, tb, inverse)


def reverse_step(q_t, x_t, rot_score, trans_score, z_rot, z_trans, mask, *, g_rot, g_trans, b_t, dt, noise_scale=1.0,
                 r3_scale=1.0, center=True, diffuse_rot=True, diffuse_trans=True):
    """One reverse-diffusion step of the noised frames on the device (no autograd: sampling runs under no_grad).
    q_t [F,N,4], x_t [F,N,3], rot_score [F,N,3] fp64, trans_score [F,N,3] fp32/fp64, z_* [F,N,3], mask [F,N] or None."""
    _need_cuda(q_t, x_t, rot_score, trans_score, z_rot, z_trans, mask)
    with torch.cuda.device(q_t.device):
        q_t, x_t, z_rot, z_trans = _f32c(q_t.detach()), _f32c(x_t.detach()), _f32c(z_rot), _f32c(z_trans)
        rs = rot_score.detach().to(torch.float64).contiguous()
        ts = trans_score.detach().contiguous()
        if ts.dtype not in (torch.float32, torch.float64):
            ts = ts.float()
        mk = _f32c(mask) if mask is not None else None
        F_, N_ = q_t.shape[0], q_t.shape[1]
        q_out, x_out = torch.empty_like(q_t), torch.empty_like(x_t)
        launch("dfold_reverse_step", q_t, x_t, rs, ts, int(ts.dtype == torch.float64), z_rot, z_trans,
               mk, float(g_rot), float(g_trans), float(b_t), float(dt), float(noise_scale), float(r3_scale),
               int(center), int(diffuse_rot), int(diffuse_trans), q_out, x_out, F_, N_)
    return q_out, x_out


def igso3_tables(sigma_grid, num_omega: int, L: int = 1000):
    """IGSO(3) tables of the reference's SO3Diffuser (so3_diffuser.py:132-180) for the fp64 ``sigma_grid`` [G] on its device:
    (cdf [G, num_omega], score_scaling [G]), both fp64."""
    _need_cuda(sigma_grid)
    with torch.cuda.device(sigma_grid.device):
        g = sigma_grid.to(torch.float64).contiguous()
        G = g.numel()
        cdf = torch.empty(G, num_omega, dtype=torch.float64, device=g.device)
        scaling = torch.empty(G, dtype=torch.float64, device=g.device)
        launch("dfold_igso3_tables", g, G, int(num_omega), int(L), cdf, scaling)
    return cdf, scaling


def forward_marginal(rigids_0, z_axis, u, z_trans, mask, t64, grid, cdf, score_scaling, *, max_sigma, min_sigma, min_b, max_b,
                     r3_scale, L=1000, diffuse_rot=True, diffuse_trans=True, ref_mode=False, n=None):
    """Forward-marginal noising of frames on the device (csrc/diffuse.cu).  rigids_0 [n,7] fp32 (None with ``ref_mode``),
    draws z_axis [n,3], u [n], z_trans [n,3] fp64, mask [n] or None, t64 a [1] fp64 device tensor.  Returns (rigids_t [n,7]
    fp32, rot_score [n,3] fp64, trans_score [n,3] fp64, rot_scaling [] fp64, trans_scaling [] fp64); with ``ref_mode`` only
    rigids_t is written (the others are None)."""
    _need_cuda(rigids_0, z_axis, u, z_trans, mask, t64, grid, cdf, score_scaling)
    dev = t64.device
    with torch.cuda.device(dev):
        r0 = _f32c(rigids_0.detach()) if rigids_0 is not None else None
        n = r0.shape[0] if r0 is not None else int(n)
        f64 = lambda x: x.detach().to(torch.float64).contiguous() if x is not None else None
        za, uu, zt = f64(z_axis), f64(u), f64(z_trans)
        mk = _f32c(mask.detach()) if mask is not None else None
        rig = torch.empty(n, 7, dtype=torch.float32, device=dev)
        rs = ts = rsc = tsc = None
        if not ref_mode:
            rs = torch.empty(n, 3, dtype=torch.float64, device=dev)
            ts = torch.empty(n, 3, dtype=torch.float64, device=dev)
            sc = torch.empty(2, dtype=torch.float64, device=dev)
            rsc, tsc = sc[0], sc[1]
        launch("dfold_forward_marginal", r0, za, uu, zt, mk, t64, grid, cdf, score_scaling, grid.numel(), cdf.shape[1], int(L),
               float(max_sigma), float(min_sigma), float(min_b), float(max_b), float(r3_scale), int(diffuse_rot),
               int(diffuse_trans), int(ref_mode), rig, rs, ts, rsc, tsc, n)
    return rig, rs, ts, rsc, tsc


def rollout_advance(rigid_pred, atom37, rigids_0, rigid_traj, atom_traj, step):
    """One step of the rollout's bookkeeping on the device (csrc/rollout.cu, eval_extension train_DFOLD_dynamics.py:993-996):
    with s = step[0] in [0, L) writes rigid_traj[s] = rigid_pred[-1] and atom_traj[s] = atom37[-1], shifts rigids_0 in place to
    cat(rigid_pred[1:], rigid_pred[-1:]) and advances step; with s outside [0, L) writes nothing.  rigid_pred [nf,N,7] and
    atom37 [nf,N,A,3] fp32 (copied when not contiguous); rigids_0 [nf,N,7], rigid_traj [L,N,7], atom_traj [L,N,A,3] contiguous
    fp32 and step a [1] int64 device tensor, all written in place.  Nothing is read back, so the call can be graph-captured."""
    _need_cuda(rigid_pred, atom37, rigids_0, rigid_traj, atom_traj, step)
    for name, t in (("rigid_pred", rigid_pred), ("atom37", atom37), ("rigids_0", rigids_0), ("rigid_traj", rigid_traj),
                    ("atom_traj", atom_traj)):
        if t.dtype != torch.float32:
            raise ValueError(f"rollout_advance: {name} must be fp32, got {t.dtype}")
    for name, t in (("rigids_0", rigids_0), ("rigid_traj", rigid_traj), ("atom_traj", atom_traj), ("step", step)):
        if not t.is_contiguous():
            raise ValueError(f"rollout_advance: {name} is written in place and must be contiguous")
    if step.dtype != torch.int64 or step.numel() != 1:
        raise ValueError(f"rollout_advance: step must be one int64, got {step.dtype} {tuple(step.shape)}")
    if rigid_pred.dim() != 3 or rigid_pred.shape[-1] != 7 or rigids_0.shape != rigid_pred.shape:
        raise ValueError(f"rollout_advance: need rigid_pred / rigids_0 [nf, N, 7] of one shape, got {tuple(rigid_pred.shape)} and "
                         f"{tuple(rigids_0.shape)}")
    nf, N = rigid_pred.shape[0], rigid_pred.shape[1]
    if atom37.dim() != 4 or atom37.shape[:2] != (nf, N) or atom37.shape[-1] != 3:
        raise ValueError(f"rollout_advance: atom37 {tuple(atom37.shape)} is not [{nf}, {N}, A, 3]")
    A, L = atom37.shape[2], rigid_traj.shape[0]
    if tuple(rigid_traj.shape) != (L, N, 7) or tuple(atom_traj.shape) != (L, N, A, 3):
        raise ValueError(f"rollout_advance: need rigid_traj [L, {N}, 7] and atom_traj [L, {N}, {A}, 3], got "
                         f"{tuple(rigid_traj.shape)} and {tuple(atom_traj.shape)}")
    with torch.cuda.device(rigids_0.device):
        rp, a37 = rigid_pred.detach().contiguous(), atom37.detach().contiguous()
        launch("dfold_rollout_advance", rp, a37, rigids_0, rigid_traj, atom_traj, step, nf, N, A, L)
