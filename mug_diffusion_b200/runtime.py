"""Runtime: ``MugEngine`` (handle + weights on one GPU) and ``Session`` (compiled state for one shape)."""
from __future__ import annotations

import ctypes as C
import threading
from collections import OrderedDict
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch.utils.weak import WeakIdKeyDictionary

from . import lib as L_
from .audio import check_z_length
from .config import EncoderConfig, ModelConfig
from .engine import (Arena, CTX_TOKENS_MAX, DecoderCompiler, EncoderCompiler, MAX_STEPS, OpList, UNetCompiler, View,
                     guided_scales_ops, tc_weight_map, unit_batch_splits)
from .packer import WeightBlob, pack_model


def _ptr(t: torch.Tensor) -> int:
    return t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class Plan:
    def __init__(self, engine: "MugEngine", ops: OpList):
        self.engine = engine
        self.n_ops = len(ops.ops)
        engine.attach_workspace(ops)
        self._arr = ops.array()
        self.handle = C.c_void_p()
        L_.check(engine.lib.mugd_plan_create(engine.handle, self._arr, self.n_ops, C.byref(self.handle)), "plan_create")
        self.captured = False
        self.launches = 0

    def run(self):
        L_.check(self.engine.lib.mugd_plan_run(self.handle, _stream()), "plan_run")
        self.launches = self.engine.lib.mugd_plan_launch_count(self.handle)

    def capture(self):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            L_.check(self.engine.lib.mugd_plan_capture(self.handle, side.cuda_stream), "plan_capture")
        torch.cuda.current_stream().wait_stream(side)
        self.launches = self.engine.lib.mugd_plan_launch_count(self.handle)
        self.captured = True

    def replay(self, times: int = 1):
        L_.check(self.engine.lib.mugd_plan_replay(self.handle, times, _stream()), "plan_replay")

    def ensure_captured(self):
        if not self.captured:
            self.run()
            self.capture()

    def _launch_steps(self, entry: str, desc, first_step: int, steps: int):
        self.ensure_captured()
        L_.check(getattr(self.engine.lib, entry)(self.handle, C.byref(desc), first_step, steps, _stream()), entry)

    def launch_plms(self, plms: L_.Plms, first_step: int, steps: int):
        """steps first_step .. first_step + steps - 1 of a PLMS request from one C call (mugd_sample_plms)"""
        self._launch_steps("mugd_sample_plms", plms, first_step, steps)

    def launch_ddpm(self, ddpm: L_.Ddpm, first_step: int, steps: int):
        """steps first_step .. first_step + steps - 1 of a DDPM request from one C call (mugd_sample_ddpm); row k of the descriptor's
        noise table is the noise of step first_step + k"""
        self._launch_steps("mugd_sample_ddpm", ddpm, first_step, steps)

    def launch_dpm(self, dpm: L_.Dpm, first_step: int, steps: int):
        """steps first_step .. first_step + steps - 1 of a DPM-Solver++ request from one C call (mugd_sample_dpm)"""
        self._launch_steps("mugd_sample_dpm", dpm, first_step, steps)

    def launch_dpm_ex(self, ex: L_.DpmEx, first_step: int, steps: int):
        """steps first_step .. first_step + steps - 1 of a DPM-Solver++ inpainting or per-chart-start request from one C call
        (mugd_sample_dpm_ex)"""
        self._launch_steps("mugd_sample_dpm_ex", ex, first_step, steps)

    def launch_dpm_stop(self, e: L_.DpmStop, first_step: int, steps: int):
        """steps first_step .. first_step + steps - 1 of a DPM-Solver++ inversion with one stop per chart from one C call
        (mugd_sample_dpm_stop)"""
        self._launch_steps("mugd_sample_dpm_stop", e, first_step, steps)

    def launch_unipc(self, u: L_.Unipc, first_step: int, steps: int):
        """steps first_step .. first_step + steps - 1 of a UniPC request from one C call (mugd_sample_unipc)"""
        self._launch_steps("mugd_sample_unipc", u, first_step, steps)

    def launch_unipc_ex(self, ex: L_.UnipcEx, first_step: int, steps: int):
        """steps first_step .. first_step + steps - 1 of a UniPC inpainting or per-chart-start request from one C call
        (mugd_sample_unipc_ex)"""
        self._launch_steps("mugd_sample_unipc_ex", ex, first_step, steps)

    def launch_unipc_stop(self, e: L_.UnipcStop, first_step: int, steps: int):
        """steps first_step .. first_step + steps - 1 of a UniPC inversion with one stop per chart from one C call
        (mugd_sample_unipc_stop)"""
        self._launch_steps("mugd_sample_unipc_stop", e, first_step, steps)

    def launch_join(self, join: L_.Join, tail: OpList, first_step: int, steps: int):
        """steps first_step .. first_step + steps - 1 of a decode request whose charts join at different iterations, from one C call
        (mugd_sample_join: the join kernel, the graph replay and the tail per step)"""
        self.ensure_captured()
        self.engine.attach_workspace(tail)
        L_.check(self.engine.lib.mugd_sample_join(self.handle, C.byref(join), tail.array(), len(tail.ops), first_step, steps, _stream()),
                 "mugd_sample_join")

    def launch(self, steps: int = 1, tail: Optional[OpList] = None, stage: Optional[L_.Stage] = None):
        """``steps`` replays of the plan's CUDA graph; with ``tail``, every replay is followed by the tail ops and all steps run from
        one C call (mugd_sample); with ``stage`` as well, each step starts with the stage kernel (mugd_sample_staged: inpainting blend,
        step noise).  The first call captures the graph, after a warm-up run outside capture (lazy module load, cudaFuncSetAttribute)."""
        self.ensure_captured()
        if tail is None:
            self.replay(steps)
            return
        self.engine.attach_workspace(tail)
        if stage is None:
            L_.check(self.engine.lib.mugd_sample(self.handle, tail.array(), len(tail.ops), steps, _stream()), "mugd_sample")
        else:
            L_.check(self.engine.lib.mugd_sample_staged(self.handle, C.byref(stage), tail.array(), len(tail.ops), steps, _stream()),
                     "mugd_sample_staged")

    def __del__(self):
        try:
            if self.handle:
                self.engine.lib.mugd_plan_destroy(self.handle)
        except Exception:
            pass


def compile_sized(engine: "MugEngine", compile_fn: Callable[[Arena], dict], batch: Optional[Tuple[int, int]] = None):
    """Compile into a zeroed device arena of exactly the size the plan needs: a dry compile measures it, the real one runs at a
    256-byte aligned base.  compile_fn(arena) returns the compiler's result dict.  ``batch`` = (samples of the plan, samples of one
    chart): the plan takes the engine's batch policy (MugEngine.batch_ops).  Returns (arena tensor, result, Plan)."""
    dry = Arena(0)
    compile_fn(dry)
    nbytes = dry.high + 1024
    arena_t = torch.zeros(nbytes // 4 + 64, device=engine.device)
    base = (arena_t.data_ptr() + 255) // 256 * 256
    res = compile_fn(Arena(base, nbytes))
    if batch is not None:
        engine.batch_ops(res["ops"], *batch)
    return arena_t, res, Plan(engine, res["ops"])


# device-resident blob tensor an engine has split in place -> its lo buffer (an entry lives as long as the tensor).  A second engine
# over the same tensor (dist.broadcast_blob leaves the blob on the device, where .to(device) returns it unchanged) must take this lo
# buffer: splitting again would round hi to itself and leave a zero lo.
_SPLIT_LO = WeakIdKeyDictionary()


class MugEngine:
    """One GPU: libmugd handle + packed weights.  Thread-safe through a single lock (the reference is not
    re-entrant either: webui.py:355-356 mutates model.z_length per request)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], cfg: Optional[ModelConfig] = None,
                 device: Optional[torch.device] = None, gemm_impl: str = "auto", blob: Optional[WeightBlob] = None,
                 max_sessions: int = 4, fold_ln: Optional[bool] = None, batch_invariant: bool = False):
        if not torch.cuda.is_available():
            raise L_.MugdError("mug_diffusion_b200 needs an sm_90 (H100) GPU; there is no CPU fallback")
        self.cfg = cfg or ModelConfig()
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        torch.cuda.set_device(self.device)
        self.lib = L_.load()
        self.handle = C.c_void_p()
        L_.check(self.lib.mugd_create(self.device.index or 0, C.byref(self.handle)), "mugd_create")
        sms, cc_major, cc_minor = C.c_int32(), C.c_int32(), C.c_int32()
        L_.check(self.lib.mugd_device_info(self.handle, C.byref(sms), C.byref(cc_major), C.byref(cc_minor)), "device_info")
        self.sm_count = sms.value
        # batch_invariant: every plan sums each GEMM's K range as the plan of one chart does, so a chart's bits do not depend on the
        # batch it is generated in (DESIGN §6b N18).  Off: today's plans, op for op.
        self.batch_invariant = bool(batch_invariant)
        self.blob = blob if blob is not None else pack_model(state_dict, self.cfg.unet, self.cfg.decoder, encoder_cfg=self.cfg.encoder)
        self.weights = self.blob.data.to(self.device)          # every weight once, fp32 (0.56 GB); tensor-core weights become hi in place
        self.wbase = self.weights.data_ptr()
        self.weights_lo: Optional[torch.Tensor] = None         # the lo operands of the tensor-core weights (second buffer)
        self.tc_split_done = False
        self.tc_map: Dict[int, Tuple[int, int]] = {}          # W -> (W_hi, W_lo) addresses; empty while the weights are plain fp32
        self.lock = threading.RLock()
        # split-K scratch of the tensor-core GEMM: all ops run in stream order, so one buffer serves every plan
        # (bound: tiles*splits < 2*SMs tiles of 128x128 fp32)
        self.tc_ws = torch.zeros(8 * 1024 * 1024, device=self.device)          # 32 MB
        self.tc_counters = torch.zeros(4096, dtype=torch.int32, device=self.device)
        # Compiled shapes are cached in small LRUs: webui derives z_length from each audio's duration (any multiple of
        # 32, webui.py:349-356), so an unbounded cache would grow by one ~1.5 GB arena + CUDA graph per new shape.
        self.sessions: "OrderedDict[tuple, Session]" = OrderedDict()
        self.dec_sessions: "OrderedDict[tuple, object]" = OrderedDict()
        self.max_sessions = max_sessions
        self.fold_ln = fold_ln                # LayerNorm folded into the next Linear: None = below 8192 token rows, True / False = forced
        # internal S4 kernel length per layer (SSKernelNPLR's `L` buffer, s4.py:557-584).  It is ENGINE state: lengthening
        # rewrites this engine's device copy of C~, so the length that goes with it must not live in the shared host blob.
        self.s4_L: Dict[str, int] = {k: int(v) for k, v in self.blob.meta.items() if k.endswith("kernel.kernel.L")}
        self.set_gemm_impl(gemm_impl)

    def set_gemm_impl(self, impl: str):
        # "tc_tf32" is an opt-in speed mode: single-pass TF32 tensor-core products (~2^-11 per product) instead of the
        # fp32-accurate 3xTF32 split.  Per-handle state; never used by the parity tests or bench.py.
        code = {"auto": L_.GEMM_TC, "simt": L_.GEMM_SIMT, "tc": L_.GEMM_TC, "tc_tf32": L_.GEMM_TC}[impl]
        L_.check(self.lib.mugd_set_gemm_impl(self.handle, code), "set_gemm_impl")
        if impl == "simt":
            # the exact-fp32 FFMA path needs the plain weights: restore them if this engine had already split them in place
            if self.tc_split_done:
                if self.blob.data.device.type != "cpu":
                    raise L_.MugdError("this engine's weights were split in place and no host copy exists: build a new engine for gemm_impl='simt'")
                self.weights.copy_(self.blob.data)
                self.tc_split_done = False
            self.tc_map = {}
        else:
            self._split_tc_weights()
            self.tc_map = tc_weight_map(self.blob, self.wbase, self.weights_lo.data_ptr())
        L_.check(self.lib.mugd_set_tc_single_pass_tf32(self.handle, 1 if impl == "tc_tf32" else 0), "set_tc_single_pass_tf32")
        self.gemm_impl = impl
        self.sessions.clear()
        self.dec_sessions.clear()

    def _split_tc_weights(self):
        """TF32 hi / lo operands of every tensor-core weight, computed on the device: hi over the plain weight, lo in a second buffer"""
        if self.tc_split_done:
            return
        if self.weights in _SPLIT_LO:
            self.weights_lo, self.tc_split_done = _SPLIT_LO[self.weights], True
            return
        if self.weights_lo is None:
            self.weights_lo = torch.zeros(max(self.blob.tc_lo_numel, 4), device=self.device)
        if self.weights is self.blob.data:
            _SPLIT_LO[self.weights] = self.weights_lo
        ops = OpList()
        for _, off, n, lo in self.blob.tc:
            d = L_.Tf32Split()
            d.w_hi, d.lo, d.n = self.wbase + 4 * off, self.weights_lo.data_ptr() + 4 * lo, n
            ops.add(L_.OP_TF32_SPLIT, d)
        st = _stream()
        for op in ops.ops:
            L_.check(self.lib.mugd_op_run(self.handle, C.byref(op), st), "tf32_split")
        self.tc_split_done = True

    def attach_workspace(self, ops: OpList):
        for op in ops.ops:
            if op.kind in (L_.OP_GEMM, L_.OP_GEMM_SERIAL):
                g = op.u.gemm
                g.workspace, g.workspace_bytes = self.tc_ws.data_ptr(), self.tc_ws.numel() * 4
                g.counters, g.n_counters = self.tc_counters.data_ptr(), self.tc_counters.numel()

    def batch_ops(self, ops: OpList, B: int, unit: int) -> OpList:
        """``ops`` compiled for B samples, of which ``unit`` make one chart, under this engine's batch policy: unchanged by default;
        with batch_invariant, every tensor-core GEMM takes the K split of the one-chart plan (engine.unit_batch_splits)"""
        if not self.batch_invariant or self.gemm_impl == "simt":
            return ops
        return unit_batch_splits(ops, B, unit, self.sm_count)

    def run_ops(self, ops: OpList):
        self.attach_workspace(ops)
        st = _stream()
        for op in ops.ops:
            L_.check(self.lib.mugd_op_run(self.handle, C.byref(op), st), f"op kind {op.kind}")

    def ncl_to_rows(self, x: torch.Tensor, rows: View):
        """contiguous [B, C, L] device tensor (the reference's layout) -> channels-last rows [B*L, C] at ``rows``"""
        B, Cc, Lr = x.shape
        ops = OpList()
        ops.transpose(_ptr(x), rows.ptr, 0, rows.ld, B, Cc, Lr, True)
        self.run_ops(ops)

    def rows_to_ncl(self, rows: View, B: int, Cc: int, Lr: int) -> torch.Tensor:
        """channels-last rows [B*L, C] at ``rows`` -> a new [B, C, L] tensor"""
        out = torch.empty(B, Cc, Lr, device=self.device)
        ops = OpList()
        ops.transpose(rows.ptr, _ptr(out), rows.ld, 0, B, Cc, Lr, False)
        self.run_ops(ops)
        return out

    def _lru_get(self, cache: OrderedDict, key, make):
        s = cache.get(key)
        if s is None:
            while len(cache) >= max(1, self.max_sessions):
                _, old = cache.popitem(last=False)          # least recently used: frees its arena, plan and graph
                if hasattr(old, "release"):
                    old.release()
                del old
            s = make()
            cache[key] = s
        else:
            cache.move_to_end(key)
        return s

    def session(self, Beff: int, Lz: int, per_sample_t: bool = False, ragged: bool = False, unit: int = 1,
                guided: bool = False, sectioned: bool = False) -> "Session":
        """the compiled U-Net of (Beff, Lz).  ``ragged``: the plan for samples padded to Lz whose valid lengths are set per request
        (Session.set_lengths); a separate session, so requests without lengths keep today's plan.  ``unit``: samples per chart (2 under
        classifier-free guidance); with batch_invariant the plan sums as the plan of ``unit`` samples does, else it is ignored.
        ``guided``: Beff = 2B samples of B charts under classifier-free guidance with one scale per chart, set per request
        (Session.set_scales); a separate session, so requests with one scale keep today's plan.
        ``sectioned``: the plan whose samples change prompt along the song (DESIGN §6b N20), its section starts set per request
        (Session.set_sections); a separate session, so requests without sections keep today's plan."""
        check_z_length(Lz)
        unit = unit if self.batch_invariant else 1
        key = ((Beff, Lz, per_sample_t) + (("ragged",) if ragged else ()) + ((("unit", unit),) if self.batch_invariant else ())
               + (("guided",) if guided else ()) + (("sectioned",) if sectioned else ()))
        return self._lru_get(self.sessions, key, lambda: Session(self, Beff, Lz, per_sample_t, ragged=ragged, unit=unit, guided=guided,
                                                                 sectioned=sectioned))

    def wave_session(self, B: int, T: int):
        """Audio encoder plan for B mel-spectrograms of T frames (SURVEY §8f N1); needs wave weights in the blob."""
        if "wave_cfg" not in self.blob.meta:
            raise L_.MugdError("this engine was packed without model.wave_model.* weights")
        from .wave import WaveSession
        return self._lru_get(self.dec_sessions, ("wave", B, T), lambda: WaveSession(self, B, T))

    def decoder_session(self, B: int, Lz: int, ragged: bool = False) -> "DecoderSession":
        check_z_length(Lz)
        if not ragged:
            return self._lru_get(self.dec_sessions, (B, Lz), lambda: DecoderSession(self, B, Lz))
        return self._lru_get(self.dec_sessions, (B, Lz, "ragged"), lambda: DecoderSession(self, B, Lz, ragged=True))

    @property
    def encoder_cfg(self) -> EncoderConfig:
        if "encoder_cfg" not in self.blob.meta:
            raise L_.MugdError("this engine was packed without model.first_stage_model.encoder.* weights")
        return self.blob.meta["encoder_cfg"]

    def encoder_session(self, B: int, Lz: int) -> "EncoderSession":
        """Chart encoder plan for B note arrays of 2^(levels-1) * Lz frames (8 Lz for the shipped model); needs encoder weights."""
        self.encoder_cfg                      # raises when the blob has no encoder
        return self._lru_get(self.dec_sessions, ("enc", B, Lz), lambda: EncoderSession(self, B, Lz))

    def __del__(self):
        try:
            self.sessions.clear()
            self.dec_sessions.clear()
            if self.handle:
                self.lib.mugd_destroy(self.handle)
        except Exception:
            pass


class Session:
    """Compiled U-Net evaluation for Beff samples of length Lz (Beff = 2B under classifier-free guidance)."""

    scales: Optional[torch.Tensor] = None     # a guided session's per-chart scales (None: not a guided session)
    e_guided: Optional[torch.Tensor] = None   # and the guided noise prediction its plan writes
    starts: Optional[torch.Tensor] = None     # a sectioned session's section starts (None: not a sectioned session)
    n_sec = 1                                 # context slots per sample (8 on a sectioned session)

    def __init__(self, engine: MugEngine, Beff: int, Lz: int, per_sample_t: bool, ragged: bool = False, unit: int = 1,
                 guided: bool = False, sectioned: bool = False):
        self.engine, self.Beff, self.Lz, self.per_sample_t = engine, Beff, Lz, per_sample_t
        self.unit = unit                      # samples of one chart: the batch the batch-invariant policy plans for
        cfg = engine.cfg.unet
        dev = engine.device
        # ragged: valid rows of each sample at every level ([levels, Beff] int32, row l = L_b >> l), data of the captured graph
        self.valid = torch.tensor([[Lz >> l] * Beff for l in range(cfg.levels)], dtype=torch.int32, device=dev) if ragged else None
        self.lens: Optional[List[int]] = None
        # guided: one guidance scale per chart of the Beff / 2 charts ([B] float32, data of the captured graph) and the guided noise
        # prediction [B*Lz, C] the plan's last op writes; every update descriptor of the session reads it unguided
        assert not guided or (Beff % 2 == 0 and not per_sample_t), (Beff, per_sample_t)
        self.scales = torch.ones(Beff // 2, device=dev) if guided else None
        self.e_guided = torch.zeros(Beff // 2 * Lz, cfg.out_channels, device=dev) if guided else None
        # sectioned: each sample's section starts in rows of every level ([levels, Beff, 8] int32, data of the captured graph; slot 0
        # at row 0, unused slots at the level's length) and 8 context slots per sample, sample b's slot s at context row (8b + s) * T
        self.starts = (torch.tensor([[[0] + [Lz >> l] * (L_.SECTIONS - 1)] * Beff for l in range(cfg.levels)], dtype=torch.int32,
                                    device=dev) if sectioned else None)
        self.n_sec = L_.SECTIONS if sectioned else 1
        self.comp = UNetCompiler(cfg, engine.blob, engine.wbase, engine.tc_map)
        emb_total = engine.blob.meta["emb_total"]
        attn_blocks = [b for b in self.comp.lay.blocks() if b.kind == "attn"]
        s4b = [b for b in self.comp.lay.blocks() if b.kind == "s4"]

        # ---- side buffers (owned torch tensors) ----------------------------------------------
        emb_rows = Beff if per_sample_t else MAX_STEPS
        self.emb_table = torch.zeros(emb_rows, emb_total, device=dev)
        self.temb = torch.zeros(emb_rows, cfg.model_channels, device=dev)
        self.emb_h1 = torch.zeros(emb_rows, cfg.time_embed_dim, device=dev)
        self.emb_h2 = torch.zeros(emb_rows, cfg.time_embed_dim, device=dev)
        self.step = torch.zeros(1, dtype=torch.int32, device=dev)
        self.coef = torch.zeros(MAX_STEPS, 4, device=dev)
        self.ctx = torch.zeros(Beff * self.n_sec * CTX_TOKENS_MAX, cfg.context_dim, device=dev)
        self.ctx_kv = [torch.zeros(Beff * self.n_sec * CTX_TOKENS_MAX, 2 * b.cin, device=dev) for b in attn_blocks]
        self.ctx_tokens = 21
        self.s4_kt = {b.prefix: torch.zeros(Lz // b.ds, b.cin, device=dev) for b in s4b}
        self._gen_s4_kernels(s4b)
        self._build()

    # S4 convolution kernels for this length: SSKernelNPLR.forward once per (model, L)  (s4.py:706-832)
    def _gen_s4_kernels(self, s4b):
        eng = self.engine
        N = eng.cfg.unet.s4_state // 2
        ws = None
        for b in s4b:
            k = b.prefix + "s4_model.kernel.kernel."
            L_int = int(eng.s4_L[k + "L"])
            L_req = self.Lz // b.ds
            if L_req > L_int:
                # same one-time, persistent mutation the reference performs in SSKernelNPLR._setup_C (s4.py:557-584):
                # lengthen C~ on the host, store it back into the weight blob and remember the new internal length
                from . import s4_setup

                def grab(n):
                    e = eng.blob.entries[k + n]
                    cnt = int(np.prod(e.shape))
                    return eng.weights[e.offset:e.offset + cnt].view(e.shape).detach().cpu()

                params = {n: grab(n) for n in ("C", "log_dt", "P", "inv_w_real", "w_imag")}
                C_new, L_int = s4_setup.lengthen(params, L_int, L_req)
                e = eng.blob.entries[k + "C"]
                eng.weights[e.offset:e.offset + C_new.numel()].copy_(C_new.reshape(-1).to(eng.device))
                eng.s4_L[k + "L"] = L_int
            need = 16 * b.cin * (L_int // 2 + 1)
            if ws is None or ws.numel() * 8 < need:
                ws = torch.empty(need // 8 + 2, dtype=torch.float64, device=eng.device)

            def w(n):
                return eng.wbase + 4 * eng.blob.offset(k + n)

            om = s4_fft_nodes(L_int).to(eng.device)
            L_.check(eng.lib.mugd_s4_kernel_gen(eng.handle, w("log_dt"), w("B"), w("C"), w("P"), w("inv_w_real"), w("w_imag"),
                                                _ptr(om), b.cin, N, L_int, L_req, _ptr(self.s4_kt[b.prefix]), _ptr(ws), ws.numel() * 8,
                                                _stream()), "s4_kernel_gen")
        torch.cuda.current_stream().synchronize()

    def _ext(self, base_ctx_tokens: int) -> dict:
        return dict(
            emb_table=_ptr(self.emb_table), step=_ptr(self.step), ctx_tokens=base_ctx_tokens,
            ctx_kv=[View(_ptr(t), t.shape[1], self.Beff * self.n_sec * base_ctx_tokens, t.shape[1]) for t in self.ctx_kv],
            s4_kt={p: View(_ptr(t), t.shape[1], t.shape[0], t.shape[1]) for p, t in self.s4_kt.items()},
        )

    def _build(self):
        # the LayerNorm fold lives in the tensor-core GEMM epilogues; the exact-fp32 FFMA path keeps the stand-alone LayerNorm
        # kernels and doubles as the referee of the folded plan.  engine.fold_ln: None = by size, True / False = forced (A/B, tests)
        fold = False if self.engine.gemm_impl == "simt" else self.engine.fold_ln
        if fold is None and self.engine.batch_invariant:
            fold = self.unit * self.Lz < 8192      # the compiler's size rule (UNetCompiler.compile), taken at one chart's rows
        valid = None if self.valid is None else [_ptr(self.valid[l]) for l in range(self.valid.shape[0])]

        def compile_fn(arena):
            res = self.comp.compile(arena, self.Beff, self.Lz, self._ext(self.ctx_tokens), self.per_sample_t, fold, valid,
                                    **({} if self.starts is None else dict(sections=_ptr(self.starts))))
            if self.scales is not None:
                res["ops"] = guided_scales_ops(res["ops"], res["xin"], res["eps"], self.Beff // 2, self.Lz, _ptr(self.e_guided),
                                               _ptr(self.scales))
            return res

        self.arena_t, res, self.plan = compile_sized(self.engine, compile_fn, batch=(self.Beff, self.unit))
        self.xin: View = res["xin"]
        self.eps: View = res["eps"]
        self.audio_slots = res["audio_slots"]
        self.ln_folded = res["ln_folded"]

    def set_ctx_tokens(self, T: int):
        """context length of the cross-attention; Lk is baked into the attention ops, so a new length recompiles the plan"""
        if T != self.ctx_tokens:
            self.ctx_tokens = T
            self._build()

    # ---- per-request preparation ---------------------------------------------------------------
    def set_lengths(self, lens: Sequence[int]):
        """a ragged session's valid length of each of its Beff samples (multiples of 32 in [32, Lz]; under classifier-free guidance
        both halves): written into the device arrays the plan reads, so the captured graph serves any mix"""
        assert self.valid is not None, "set_lengths needs a ragged session"
        lens = [int(v) for v in lens]
        assert len(lens) == self.Beff and all(32 <= v <= self.Lz and v % 32 == 0 for v in lens), lens
        t = torch.tensor([[v >> l for v in lens] for l in range(self.valid.shape[0])], dtype=torch.int32)
        self.valid.copy_(t.to(self.engine.device))
        self.lens = lens

    def set_sections(self, starts: Sequence[Sequence[int]]):
        """a sectioned session's section starts: starts[b] lists the latent frames at which sample b changes prompt (multiples of 8,
        strictly increasing in (0, Lz), at most 7; empty = one prompt), written into the device table the plan reads, so the
        captured graph serves any layout"""
        assert self.starts is not None, "set_sections needs a sectioned session"
        assert len(starts) == self.Beff, (len(starts), self.Beff)
        levels = self.starts.shape[0]
        rows = []
        for l in range(levels):
            lev = []
            for st in starts:
                st = [int(v) for v in st]
                assert len(st) < L_.SECTIONS and all(v % 8 == 0 and 0 < v < self.Lz for v in st), st
                assert all(a < b for a, b in zip(st, st[1:])), st
                lev.append([0] + [v >> l for v in st] + [self.Lz >> l] * (L_.SECTIONS - 1 - len(st)))
            rows.append(lev)
        self.starts.copy_(torch.tensor(rows, dtype=torch.int32).to(self.engine.device))

    def set_scales(self, scales: Sequence[float]):
        """a guided session's guidance scale of each of its Beff / 2 charts (finite; 1 = no guidance for that chart): written into
        the device array the plan reads, so the captured graph serves any mix"""
        assert self.scales is not None, "set_scales needs a guided session"
        assert len(scales) == self.scales.numel(), (len(scales), self.scales.numel())
        self.scales.copy_(torch.tensor([float(v) for v in scales], dtype=torch.float32).to(self.engine.device))

    def set_timestep_table(self, timesteps: Sequence[int]):
        """Time-embedding MLP + all ResBlock emb projections for the given timesteps, one row each
        (unet.py:335-339, 166-172; model/util.py:156-176).  The sinusoid is evaluated on the host exactly
        as the reference does; the three GEMMs run on the GPU.  Integer timesteps go through a long tensor as the samplers' t does;
        float times (the DPM-Solver's model times) are taken as float32, the dtype the sinusoid computes in."""
        cfg = self.engine.cfg.unet
        eng = self.engine
        ts = np.asarray(timesteps)
        if ts.dtype.kind == "f":
            t = torch.as_tensor(ts.astype(np.float32))
        else:
            t = torch.as_tensor(ts, dtype=torch.long)
        R = t.shape[0]
        assert R <= self.temb.shape[0]
        half = cfg.model_channels // 2
        import math
        freqs = torch.exp(-math.log(10000.0) * torch.arange(0, half, dtype=torch.float32) / half)
        args = t[:, None].float() * freqs[None]
        emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
        self.temb[:R].copy_(emb.to(eng.device))
        eng.run_ops(self.timestep_ops(R))

    def timestep_ops(self, R: int) -> OpList:
        """the three GEMMs that turn R sinusoid rows (self.temb) into R rows of the fused ResBlock embedding table"""
        cfg = self.engine.cfg.unet
        eng = self.engine
        ops = OpList(eng.tc_map)
        up = self.comp.prefix
        tv = View(_ptr(self.temb), cfg.model_channels, R, cfg.model_channels)
        h1 = View(_ptr(self.emb_h1), cfg.time_embed_dim, R, cfg.time_embed_dim)
        h2 = View(_ptr(self.emb_h2), cfg.time_embed_dim, R, cfg.time_embed_dim)
        et = View(_ptr(self.emb_table), self.emb_table.shape[1], R, self.emb_table.shape[1])
        w = self.comp.w
        ops.gemm(tv, w(up + "time_embed.0.weight"), cfg.time_embed_dim, cfg.model_channels, h1, bias=w(up + "time_embed.0.bias"),
                 act=L_.ACT_SILU)
        # emb is only ever consumed through emb_layers = SiLU -> Linear, so SiLU(emb) is stored
        ops.gemm(h1, w(up + "time_embed.2.weight"), cfg.time_embed_dim, cfg.time_embed_dim, h2, bias=w(up + "time_embed.2.bias"),
                 act=L_.ACT_SILU)
        ops.gemm(h2, w(up + "emb_all.weight"), self.emb_table.shape[1], cfg.time_embed_dim, et, bias=w(up + "emb_all.bias"))
        # per-sample timesteps: one row per sample; otherwise one row per schedule step, the same rows at any batch
        return eng.batch_ops(ops, self.Beff, self.unit) if self.per_sample_t else ops

    def set_context(self, context):
        """context [Beff, ctx_dim, T] (reference layout; or a list of such tensors that follow each other along the batch, e.g.
        [uc, c] under classifier-free guidance, ddim.py:173) -> per-layer cross-attention K|V projections (attention.py:97-98),
        constant over the DDIM steps.  A sectioned session takes Beff * 8 contexts: sample b's section slot s at index 8b + s."""
        eng = self.engine
        cfg = eng.cfg.unet
        parts = list(context) if isinstance(context, (list, tuple)) else [context]
        parts = [c.to(eng.device, torch.float32).contiguous() for c in parts]
        Bc = sum(int(c.shape[0]) for c in parts)
        _, Cd, T = parts[0].shape
        assert Bc == self.Beff * self.n_sec and Cd == cfg.context_dim and T <= CTX_TOKENS_MAX and all(c.shape[1:] == parts[0].shape[1:] for c in parts)
        self.set_ctx_tokens(T)
        eng.run_ops(self.context_ops([(_ptr(c), int(c.shape[0])) for c in parts], T))
        self._keep = parts

    def context_ops(self, parts: Sequence, T: int) -> OpList:
        """parts: (device address of a [b, ctx_dim, T] tensor, b) in batch order -> transposes + the 16 K|V projections"""
        eng = self.engine
        cfg = eng.cfg.unet
        Cd = cfg.context_dim
        Bc = sum(b for _, b in parts)
        ops = OpList(eng.tc_map)
        row = 0
        for addr, bpart in parts:
            ops.transpose(addr, _ptr(self.ctx) + 4 * row * Cd, 0, Cd, bpart, Cd, T, True)
            row += bpart * T
        cv = View(_ptr(self.ctx), Cd, Bc * T, Cd)
        blocks = [b for b in self.comp.lay.blocks() if b.kind == "attn"]
        for b, kv in zip(blocks, self.ctx_kv):
            o = View(_ptr(kv), kv.shape[1], Bc * T, kv.shape[1])
            ops.gemm(cv, self.comp.w(b.prefix + "transformer_blocks.0.attn2.kv.weight"), 2 * b.cin, Cd, o, Lout=T)
        return eng.batch_ops(ops, Bc, self.unit * (Bc // self.Beff))      # a chart's contexts: 8 per sample on a sectioned session

    def set_audio(self, audios: Sequence[torch.Tensor], dup: bool = False):
        """The last ``levels`` entries of the wave-encoder output list (unet.py:527-543), NCL layout, written
        (transposed) into every concat slot that holds them.  ``dup``: the tensors hold Beff/2 samples and both halves of the
        batch get them (the reference concatenates them with themselves under classifier-free guidance, ddim.py:171-174)."""
        cfg = self.engine.cfg.unet
        w4 = [a.to(self.engine.device, torch.float32).contiguous() for a in list(audios)[-cfg.levels:]]
        Bh = self.Beff // 2 if dup else self.Beff
        for lvl in range(cfg.levels):
            assert w4[lvl].shape == (Bh, cfg.audio_channels[lvl], self.Lz >> lvl), (w4[lvl].shape, lvl)
        self.engine.run_ops(self.audio_ops([_ptr(a) for a in w4], dup))
        self._keep_audio = w4

    def audio_ops(self, addrs: Sequence[int], dup: bool) -> OpList:
        """addrs[lvl] = device address of the [Beff (or Beff/2 when dup), C_lvl, L_lvl] audio feature map of level lvl"""
        cfg = self.engine.cfg.unet
        Bh = self.Beff // 2 if dup else self.Beff
        ops = OpList()
        for lvl, view in self.audio_slots:
            Cc, Lr = cfg.audio_channels[lvl], self.Lz >> lvl
            ops.transpose(addrs[lvl], view.ptr, 0, view.ld, Bh, Cc, Lr, True)
            if dup:
                ops.transpose(addrs[lvl], view.r(Bh * Lr, 2 * Bh * Lr).ptr, 0, view.ld, Bh, Cc, Lr, True)
        return ops

    def load_x(self, x: torch.Tensor, dup: bool):
        """x [B,C,L] -> xin rows (both halves when dup)."""
        x = x.to(self.engine.device, torch.float32).contiguous()
        B, Cc, Lr = x.shape
        self.engine.run_ops(self.loadx_ops(_ptr(x), B, dup))
        self._keep_x = x

    def loadx_ops(self, addr: int, B: int, dup: bool) -> OpList:
        Cc, Lr = self.engine.cfg.unet.in_channels, self.Lz
        ops = OpList()
        ops.transpose(addr, self.xin.ptr, 0, self.xin.ld, B, Cc, Lr, True)
        if dup:
            ops.transpose(addr, self.xin.r(B * Lr, 2 * B * Lr).ptr, 0, self.xin.ld, B, Cc, Lr, True)
        return ops

    def read_rows(self, view: View, B: int, Cc: int, Lr: int) -> torch.Tensor:
        return self.engine.rows_to_ncl(view, B, Cc, Lr)

    def eval(self, graph: bool = True):
        if graph:
            self.plan.launch()
        else:
            self.plan.run()

    def set_ddim_schedule(self, alphas, alphas_prev, sigmas, sqrt_one_minus_alphas):
        """coef row i = (alpha, alpha_prev, sigma, sqrt(1 - alpha)) of DDIM step i, rows past the schedule zero"""
        coef = np.stack([np.asarray(a, dtype=np.float32) for a in (alphas, alphas_prev, sigmas, sqrt_one_minus_alphas)], axis=1)
        self.coef.zero_()
        self.coef[:len(coef)].copy_(torch.from_numpy(coef).to(self.engine.device))

    def _x_rows(self, B: int, cfg_on: bool):
        """the device addresses of the x rows a step updates: the first B samples' xin rows, and under classifier-free guidance
        their copy in the second half (else None; also on a guided session, whose plan copies them itself)"""
        return self.xin.ptr, (self.xin.r(B * self.Lz, 2 * B * self.Lz).ptr if cfg_on and self.scales is None else None)

    def _guidance(self, cfg_on: bool, scale) -> Tuple[int, int, float]:
        """(eps rows, cfg, scale) of an update: the plan's eps rows with the request's guidance, or on a guided session the guided
        rows the plan's last op wrote, read unguided"""
        if self.scales is not None:
            return _ptr(self.e_guided), 0, 1.0
        return self.eps.ptr, int(cfg_on), 1.0 if isinstance(scale, list) else float(scale)

    def ddim_update(self, B: int, S: int, cfg_on: bool, scale: float, temperature: float, pred_x0: int, noise: int = 0) -> L_.DdimUpdate:
        """the DDIM update of ddim_tail"""
        n = B * self.Lz * self.engine.cfg.unet.in_channels
        upd = L_.DdimUpdate()
        upd.x, upd.x_dup = self._x_rows(B, cfg_on)
        upd.eps, upd.cfg, upd.scale = self._guidance(cfg_on, scale)
        upd.noise, upd.pred_x0 = noise or None, pred_x0
        upd.coef, upd.step = _ptr(self.coef), _ptr(self.step)
        upd.S, upd.n, upd.temperature = S, n, float(temperature)
        return upd

    def plms(self, B: int, S: int, cfg_on: bool, scale: float, pred_x0: int, work: torch.Tensor) -> L_.Plms:
        """the mugd_sample_plms descriptor of an S-step request for B samples: the combine reads eps (both halves under
        classifier-free guidance), the update (cfg = 0, no noise) runs on e' and writes the xin rows of both halves and pred_x0.
        ``work``: a [5, B*Lz*C] device tensor owned by the caller = e', the ring of the last three e_t, the x stash."""
        n = B * self.Lz * self.engine.cfg.unet.in_channels
        assert work.shape == (5, n) and work.dtype == torch.float32 and work.is_contiguous()
        p = L_.Plms()
        p.update = self.ddim_update(B, S, cfg_on, 1.0, 1.0, pred_x0)
        p.update.cfg, p.update.eps = 0, _ptr(work[0])
        p.eps, p.cfg, p.scale = self._guidance(cfg_on, scale)
        p.e_prime, p.hist, p.x_stash = _ptr(work[0]), _ptr(work[1]), _ptr(work[4])
        return p

    def ddpm(self, B: int, T: int, cfg_on: bool, scale: float, clip: bool, pred_x0: int, noise: int, coef: torch.Tensor) -> L_.Ddpm:
        """the mugd_sample_ddpm descriptor of a T-step request for B samples: the update reads eps (both halves under
        classifier-free guidance), ``coef`` (the model's [T, 5] table, kept alive by the caller) and the noise table at ``noise``
        ([n][B, C, Lz]), and writes the xin rows of both halves and pred_x0"""
        assert coef.shape == (T, 5) and coef.dtype == torch.float32 and coef.is_contiguous()
        d = L_.Ddpm()
        d.x, d.x_dup = self._x_rows(B, cfg_on)
        d.eps, d.cfg, d.scale = self._guidance(cfg_on, scale)
        d.pred_x0, d.noise, d.coef, d.step = pred_x0 or None, noise, _ptr(coef), _ptr(self.step)
        d.T, d.B, d.C, d.L = T, B, self.engine.cfg.unet.in_channels, self.Lz
        d.clip = int(bool(clip))
        return d

    def dpm(self, B: int, S: int, cfg_on: bool, scale: float, pred_x0: int, ring: torch.Tensor, coef: torch.Tensor) -> L_.Dpm:
        """the mugd_sample_dpm descriptor of an S-step request for B samples: the update reads eps (both halves under
        classifier-free guidance) and ``coef`` (the request's [S, 8] coefficient rows), keeps the last three data predictions in
        ``ring`` ([3, B*Lz*C]), and writes the xin rows of both halves and pred_x0.  The caller keeps both tensors alive."""
        n = B * self.Lz * self.engine.cfg.unet.in_channels
        assert coef.shape == (S, 8) and coef.dtype == torch.float32 and coef.is_contiguous()
        assert ring.shape == (3, n) and ring.dtype == torch.float32 and ring.is_contiguous()
        d = L_.Dpm()
        d.x, d.x_dup = self._x_rows(B, cfg_on)
        d.eps, d.cfg, d.scale = self._guidance(cfg_on, scale)
        d.pred_x0, d.ring, d.coef, d.step = pred_x0 or None, _ptr(ring), _ptr(coef), _ptr(self.step)
        d.n, d.S = n, S
        return d

    def dpm_ex(self, dpm: L_.Dpm, stage: Optional[L_.Stage] = None, B: int = 0, start: Optional[torch.Tensor] = None,
               order_coef: Optional[torch.Tensor] = None) -> L_.DpmEx:
        """the mugd_sample_dpm_ex descriptor around ``dpm``: with ``stage`` (ddim_stage's, x0 / mask / q_noise / q_coef filled in) the
        inpainting blend runs in front of each step; with ``start`` ([B] int32, the first step of each chart) and ``order_coef``
        (the [S, 3, 8] per-order rows) every chart runs from its own step.  The caller keeps the stage and both tensors alive."""
        e = L_.DpmEx()
        e.dpm = dpm
        e.stage = C.addressof(stage) if stage is not None else None
        if start is not None:
            assert start.shape == (B,) and start.dtype == torch.int32 and start.is_contiguous()
            assert order_coef.shape == (dpm.S, 3, 8) and order_coef.dtype == torch.float32 and order_coef.is_contiguous()
            e.start, e.order_coef, e.B = _ptr(start), _ptr(order_coef), B
        return e

    def dpm_stop(self, dpm: L_.Dpm, B: int, stop: torch.Tensor) -> L_.DpmStop:
        """the mugd_sample_dpm_stop descriptor around ``dpm`` (an inversion schedule's rows): chart b runs steps 0 .. stop[b] - 1
        (``stop``: [B] int32 on the device).  The caller keeps the tensor alive."""
        assert stop.shape == (B,) and stop.dtype == torch.int32 and stop.is_contiguous()
        e = L_.DpmStop()
        e.dpm, e.stop, e.B = dpm, _ptr(stop), B
        return e

    def unipc(self, B: int, S: int, cfg_on: bool, scale: float, pred_x0: int, ring: torch.Tensor, coef: torch.Tensor, xc: torch.Tensor,
              corr: torch.Tensor) -> L_.Unipc:
        """the mugd_sample_unipc descriptor of an S-step request for B samples: ``dpm``'s with the predictor rows ``coef`` ([S, 8]), plus
        the corrector rows ``corr`` ([S, 8]) and the corrected latent ``xc`` ([B*Lz*C]).  The caller keeps the tensors alive."""
        assert corr.shape == (S, 8) and corr.dtype == torch.float32 and corr.is_contiguous()
        u = L_.Unipc()
        u.dpm = self.dpm(B, S, cfg_on, scale, pred_x0, ring, coef)
        assert xc.numel() == u.dpm.n and xc.dtype == torch.float32 and xc.is_contiguous()
        u.xc, u.corr = _ptr(xc), _ptr(corr)
        return u

    def unipc_ex(self, u: L_.Unipc, stage: Optional[L_.Stage] = None, B: int = 0, start: Optional[torch.Tensor] = None,
                 order_coef: Optional[torch.Tensor] = None, order_corr: Optional[torch.Tensor] = None) -> L_.UnipcEx:
        """the mugd_sample_unipc_ex descriptor around ``u``: with ``stage`` (ddim_stage's, x0 / mask / q_noise / q_coef filled in) the
        inpainting blend runs in front of each step; with ``start`` ([B] int32, the first step of each chart) and ``order_coef`` /
        ``order_corr`` (the [S, 3, 8] per-order predictor and corrector rows) every chart runs from its own step.  The caller keeps
        the stage and the tensors alive."""
        e = L_.UnipcEx()
        e.unipc = u
        e.stage = C.addressof(stage) if stage is not None else None
        if start is not None:
            S = u.dpm.S
            assert start.shape == (B,) and start.dtype == torch.int32 and start.is_contiguous()
            for t in (order_coef, order_corr):
                assert t.shape == (S, 3, 8) and t.dtype == torch.float32 and t.is_contiguous()
            e.start, e.order_coef, e.order_corr, e.B = _ptr(start), _ptr(order_coef), _ptr(order_corr), B
        return e

    def unipc_stop(self, u: L_.Unipc, B: int, stop: torch.Tensor) -> L_.UnipcStop:
        """the mugd_sample_unipc_stop descriptor around ``u`` (an inversion schedule's rows): chart b runs iterations 0 .. stop[b] - 1
        (``stop``: [B] int32 on the device).  The caller keeps the tensor alive."""
        assert stop.shape == (B,) and stop.dtype == torch.int32 and stop.is_contiguous()
        e = L_.UnipcStop()
        e.unipc, e.stop, e.B = u, _ptr(stop), B
        return e

    def ddim_tail(self, B: int, S: int, cfg_on: bool, scale: float, temperature: float, pred_x0: int, noise: int = 0) -> OpList:
        """the ops that follow each evaluation of an S-step request for B samples: the DDIM update of the xin rows (both halves
        under classifier-free guidance) from eps, the coef row of the current step and, if ``noise`` is given, the noise rows;
        pred_x0 receives the predicted x0 rows.  Then the step counter advances."""
        upd = self.ddim_update(B, S, cfg_on, scale, temperature, pred_x0, noise)
        adv = L_.StepAdvance()
        adv.step = _ptr(self.step)
        tail = OpList()
        tail.add(L_.OP_DDIM_UPDATE, upd)
        tail.add(L_.OP_STEP_ADVANCE, adv)
        return tail

    def ddim_stage(self, B: int, cfg_on: bool, noise: int = 0) -> L_.Stage:
        """the stage of mugd_sample_staged over the rows ddim_tail updates (x, and its copy under classifier-free guidance);
        ``noise`` = the tail's noise rows.  The caller fills in x0 / mask / q_noise / q_coef and the noise table."""
        s = L_.Stage()
        s.x, s.x_dup = self._x_rows(B, cfg_on)
        s.noise_rows = noise or None
        s.B, s.C, s.L = B, self.engine.cfg.unet.in_channels, self.Lz
        return s

    def join(self, B: int, cfg_on: bool, x_latent: int, join: int) -> L_.Join:
        """the mugd_sample_join descriptor over the rows ddim_tail updates (x, and its copy under classifier-free guidance):
        ``x_latent`` = the device address of the [B, C, Lz] start latents, ``join`` = that of the [B] int32 join iterations"""
        j = L_.Join()
        j.x, j.x_dup = self._x_rows(B, cfg_on)
        j.x_latent, j.join = x_latent, join
        j.B, j.C, j.L = B, self.engine.cfg.unet.in_channels, self.Lz
        return j

    def set_step(self, value: int):
        L_.check(self.engine.lib.mugd_fill_i32(_ptr(self.step), value, _stream()), "fill_i32")


class DecoderSession:
    def __init__(self, engine: MugEngine, B: int, Lz: int, ragged: bool = False):
        self.engine, self.B, self.Lz = engine, B, Lz
        comp = DecoderCompiler(engine.cfg.decoder, engine.blob, engine.wbase, engine.tc_map)
        # ragged: valid rows per sample at every length multiplier of the blocks ([n_mul, B] int32, row k = muls[k] * L_b)
        self.muls = sorted({b.mul for b in comp.seq} | {b.mul * 2 for b in comp.seq if b.kind == "up"}) if ragged else []
        self.valid = torch.zeros(len(self.muls), B, dtype=torch.int32, device=engine.device) if ragged else None
        valid = {m: _ptr(self.valid[k]) for k, m in enumerate(self.muls)} if ragged else None
        self.arena_t, res, self.plan = compile_sized(engine, lambda arena: comp.compile(arena, B, Lz, valid), batch=(B, 1))
        self.zin, self.logits, self.Lout = res["inp"], res["out"], res["Lout"]

    def notes(self, frame_ms: float, key_count: int = 4):
        """Note extraction on the logits of the last ``decode`` (still resident, channels-last): returns
        (count [B,K], start_ms [B,K,T], end_ms [B,K,T]) as CPU int32 tensors; only count and the used prefixes matter."""
        eng = self.engine
        B, T, K = self.B, self.Lout, key_count
        assert 4 * K == eng.cfg.decoder.x_channels
        cnt = torch.zeros(B, K, dtype=torch.int32, device=eng.device)
        st = torch.full((B, K, T), -1, dtype=torch.int32, device=eng.device)
        en = torch.full((B, K, T), -1, dtype=torch.int32, device=eng.device)
        d = L_.Notes()
        d.logits, d.ld = self.logits.ptr, self.logits.ld
        d.count, d.start_ms, d.end_ms = _ptr(cnt), _ptr(st), _ptr(en)
        d.frame_ms, d.B, d.T, d.K = float(frame_ms), B, T, K
        ops = OpList()
        ops.add(L_.OP_NOTES, d)
        eng.run_ops(ops)
        cnt_c = cnt.cpu()
        nmax = int(cnt_c.max()) if cnt_c.numel() else 0
        return cnt_c, st[:, :, :max(nmax, 1)].cpu(), en[:, :, :max(nmax, 1)].cpu()

    def set_lengths(self, lens: Sequence[int]):
        """a ragged session's latent length of each chart (its logits are valid for mul * L_b rows at multiplier mul)"""
        assert self.valid is not None and len(lens) == self.B and all(32 <= int(v) <= self.Lz for v in lens), lens
        t = torch.tensor([[m * int(v) for v in lens] for m in self.muls], dtype=torch.int32)
        self.valid.copy_(t.to(self.engine.device))

    def decode(self, z: torch.Tensor, lens: Optional[Sequence[int]] = None) -> torch.Tensor:
        """logits [B, x_channels, Lout] of the latents z [B, z_channels, Lz]; a ragged session takes each chart's length ``lens`` and
        returns logits that are 0 past Lout / Lz * lens[b]"""
        eng = self.engine
        cfg = eng.cfg.decoder
        if self.valid is not None:
            self.set_lengths(lens)
        z = z.to(eng.device, torch.float32)
        if cfg.scale != 1.0:
            z = z / cfg.scale                 # autoencoder.py:76
        eng.ncl_to_rows(z.contiguous(), self.zin)
        self.plan.launch()
        return eng.rows_to_ncl(self.logits, self.B, cfg.x_channels, self.Lout)


class EncoderSession:
    """Compiled chart encoder (Encoder.forward, autoencoder.py:244-265) for B note arrays of ``frames`` = 2^(levels-1) * Lz frames."""

    def __init__(self, engine: MugEngine, B: int, Lz: int):
        self.engine, self.B, self.Lz = engine, B, Lz
        self.cfg = engine.encoder_cfg
        comp = EncoderCompiler(self.cfg, engine.blob, engine.wbase, engine.tc_map)
        self.frames = Lz * comp.seq[0].mul
        self.arena_t, res, self.plan = compile_sized(engine, lambda arena: comp.compile(arena, B, Lz), batch=(B, 1))
        self.notes_rows, self.moments = res["inp"], res["out"]

    def encode(self, notes: torch.Tensor) -> "DiagonalGaussianDistribution":
        """notes [B, x_channels, frames] -> the posterior of AutoencoderKL.encode (autoencoder.py:67-73)"""
        eng = self.engine
        cfg = self.cfg
        x = notes.to(eng.device, torch.float32).contiguous()
        assert x.shape == (self.B, cfg.x_channels, self.frames), (tuple(x.shape), (self.B, cfg.x_channels, self.frames))
        eng.ncl_to_rows(x, self.notes_rows)
        self.plan.launch()
        params = eng.rows_to_ncl(self.moments, self.B, 2 * cfg.z_channels, self.Lz)
        return DiagonalGaussianDistribution(eng, params, cfg.scale)


class DiagonalGaussianDistribution:
    """The encoder's posterior with the surface callers use of the reference class of the same name (autoencoder.py:356-387):
    ``parameters`` [B, 2Z, L], ``mean`` / ``logvar`` (clamped to [-10, 20]) / ``std`` / ``var`` [B, Z, L], ``mode()`` and ``sample()``.
    All are device tensors; mean, logvar, std, mode() and sample() come from the posterior kernel (MUGD_OP_POSTERIOR)."""

    def __init__(self, engine: MugEngine, parameters: torch.Tensor, scale: float):
        self.engine, self.parameters, self.scale = engine, parameters, float(scale)
        B, C2, L = parameters.shape
        self.mean, self.logvar, self.std = (torch.empty(B, C2 // 2, L, device=parameters.device) for _ in range(3))
        self._var: Optional[torch.Tensor] = None
        self._run(mean=self.mean, logvar=self.logvar, std=self.std)

    def _run(self, noise: Optional[torch.Tensor] = None, **outs: torch.Tensor):
        B, Z, L = self.mean.shape
        d = L_.Posterior()
        d.params, d.noise = _ptr(self.parameters), _ptr(noise) if noise is not None else None
        for name, t in outs.items():
            setattr(d, name, _ptr(t))
        d.scale, d.B, d.Z, d.L = self.scale, B, Z, L
        ops = OpList()
        ops.add(L_.OP_POSTERIOR, d)
        with self.engine.lock:
            self.engine.run_ops(ops)

    @property
    def var(self) -> torch.Tensor:
        """exp(logvar) (autoencoder.py:365); only the KL term reads it, so it is formed on first use"""
        if self._var is None:
            self._var = torch.exp(self.logvar)
        return self._var

    def mode(self) -> torch.Tensor:
        """mean * scale (autoencoder.py:386-387)"""
        z = torch.empty_like(self.mean)
        self._run(z=z)
        return z

    def sample(self) -> torch.Tensor:
        """(mean + std * n) * scale with n = torch.randn(mean.shape) drawn on the CPU generator, as the reference draws it
        (autoencoder.py:370-372): after torch.manual_seed(s) the result matches the reference's for the same s."""
        noise = torch.randn(self.mean.shape).to(self.mean.device)
        z = torch.empty_like(self.mean)
        self._run(noise, z=z)
        return z


_NODE_CACHE: Dict[int, torch.Tensor] = {}


def s4_fft_nodes(L_int: int) -> torch.Tensor:
    """omega_f for f = 0..L/2 evaluated the way the reference does (SSKernelNPLR._omega, s4.py:586-604):
    a complex64 base raised to integer powers on the host.  This is a parameter-free constant table like the
    timestep sinusoid; feeding the same nodes to the fp64 kernel generator reproduces the reference's kernel
    to ~2e-6 instead of ~1e-4 (the complex64 power drifts by up to 5e-6 at f = L/2).  Returns [L/2+1, 2] fp32."""
    t = _NODE_CACHE.get(L_int)
    if t is None:
        base = torch.tensor(np.exp(-2j * np.pi / L_int), dtype=torch.complex64)
        t = torch.view_as_real(base ** torch.arange(0, L_int // 2 + 1)).contiguous()
        _NODE_CACHE[L_int] = t
    return t


def hit_object_lines(count, start_ms, end_ms, key_count: int):
    """Per chart: the .osu hit-object lines of OsuManiaConvertor.array_to_objects (convertor.py:257-264) from the
    compact (column, frame-ordered) note lists the GPU produced; sorted by start time with a stable sort, like the reference."""
    width = int(512 / key_count)
    charts = []
    for b in range(count.shape[0]):
        items = []
        for col in range(key_count):
            n = int(count[b, col])
            x = int(round((col + 0.5) * width))
            for s_, e_ in zip(start_ms[b, col, :n].tolist(), end_ms[b, col, :n].tolist()):
                line = f"{x},192,{s_},1,0,0:0:0:0:" if e_ == -1 else f"{x},192,{s_},128,0,{e_}:0:0:0:0:"
                items.append((line, s_))
        items.sort(key=lambda t: t[1])
        charts.append([t[0] for t in items])
    return charts
