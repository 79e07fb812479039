"""B200Whisper: device-resident Whisper weights packed for the sm_90a kernels + thin call wrappers.

Mirrors the model-object protocol the reference touches (SURVEY.md section 8b "B2": ``dims``, ``device``,
``is_multilingual``, ``num_languages``, ``alignment_heads``), but the forward passes are the C-ABI entry points of
libstablets_b200.so, not nn.Modules.  PyTorch only owns memory and streams.

Weight layout handed to the kernels (all caller-owned torch tensors kept alive in ``self._keep``):
  * every GEMM weight as split-fp16 planes (hi = fp16(W), lo = fp16(W - hi)), K-major [out][in];
  * q/k/v fused to one [3d][d] matrix (k bias = 0), cross k/v fused to [2d][d];
  * conv weights [out][in][3] re-ordered to [out][tap*in + c] so the convs are GEMMs over overlapping rows;
  * LayerNorm / bias / positional tables in fp32; token embedding both fp32 (gather) and split (logits GEMM).
"""
import ctypes
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

import functools

from . import _lib as L
from .shim import WhisperProtocol


def _on_device(fn):
    """Run a kernel-launching method with the model's device current: the launches go to torch's current stream OF THAT
    DEVICE (a model on cuda:1 must not enqueue on cuda:0's stream when the caller's current device differs)."""
    @functools.wraps(fn)
    def wrapped(self, *a, **k):
        with torch.cuda.device(self.device):
            return fn(self, *a, **k)
    return wrapped


@dataclass
class ModelDimensions:
    n_mels: int
    n_audio_ctx: int
    n_audio_state: int
    n_audio_head: int
    n_audio_layer: int
    n_vocab: int
    n_text_ctx: int
    n_text_state: int
    n_text_head: int
    n_text_layer: int


def _split(w: torch.Tensor, want_lo: bool):
    w = w.float().contiguous()
    hi = w.half()
    lo = (w - hi.float()).half() if want_lo else None
    return hi, lo


def mel_filterbank(n_mels: int) -> np.ndarray:
    """librosa-style Slaney mel filterbank (sr 16 kHz, n_fft 400), the matrix whisper ships as mel_filters.npz."""
    def hz2mel(f):
        f = np.asarray(f, dtype=np.float64)
        return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-10) / 1000.0) / (np.log(6.4) / 27.0), f / (200.0 / 3))

    def mel2hz(m):
        m = np.asarray(m, dtype=np.float64)
        return np.where(m >= 15.0, 1000.0 * np.exp((np.log(6.4) / 27.0) * (m - 15.0)), (200.0 / 3) * m)

    freqs = np.linspace(0.0, 8000.0, 201)
    pts = mel2hz(np.linspace(hz2mel(0.0), hz2mel(8000.0), n_mels + 2))
    fdiff = np.diff(pts)
    ramps = pts[:, None] - freqs[None, :]
    lower = -ramps[:-2] / fdiff[:-1, None]
    upper = ramps[2:] / fdiff[1:, None]
    w = np.maximum(0.0, np.minimum(lower, upper))
    w *= (2.0 / (pts[2:] - pts[:-2]))[:, None]
    return w.astype(np.float32)


class B200Whisper(WhisperProtocol):
    """Whisper weights on one H100 + the kernel entry points.  ``precision``: "fp16x3" (parity mode) or "fp16".
    ``WhisperProtocol`` (shim.py) adds the whisper model-object surface (``encoder`` / ``decoder`` / hooks / kv-cache
    protocol / ``detect_language``) that the unmodified reference code drives."""

    def __init__(self, dims, state_dict: Dict[str, torch.Tensor], device: Union[str, torch.device] = "cuda",
                 precision: str = "fp16x3", alignment_heads: Optional[Sequence[Tuple[int, int]]] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("B200Whisper needs a CUDA device (there is no CPU fallback)")
        self.dims = ModelDimensions(**{k: int(getattr(dims, k)) for k in ModelDimensions.__dataclass_fields__})
        self.device = torch.device(device)
        self.precision = precision
        self._prec = {"fp16x3": L.STB_PREC_FP16X3, "fp16": L.STB_PREC_FP16}[precision]
        self._want_lo = self._prec == L.STB_PREC_FP16X3
        self._keep: List[torch.Tensor] = []
        self._ws: Dict[str, torch.Tensor] = {}
        self.graph_kernel_launches = 0     # kernels executed by CUDA-graph replays (the library counter only sees captures)
        self._lib = L.lib()
        d = L.Dims(**self.dims.__dict__)
        h = ctypes.c_void_p()
        L.check(self._lib.stb_model_create(ctypes.byref(d), self._prec, ctypes.byref(h)))
        self._h = h
        if alignment_heads is None:           # whisper default: all heads of the last half of the decoder layers
            alignment_heads = [(l, hh) for l in range(self.dims.n_text_layer // 2, self.dims.n_text_layer)
                               for hh in range(self.dims.n_text_head)]
        self.alignment_head_pairs = [(int(a), int(b)) for a, b in alignment_heads]
        self.missing_alignment_heads = False
        self.random_init = False
        with torch.cuda.device(self.device):
            self._pack(state_dict)
            self._frontend_tables()
        self._init_protocol()

    def set_alignment_heads(self, pairs_or_mask):
        """(layer, head) pairs or a bool [n_text_layer, n_text_head] mask (whisper's ``set_alignment_heads`` takes the
        base85 dump of such a mask)."""
        if torch.is_tensor(pairs_or_mask) or isinstance(pairs_or_mask, np.ndarray):
            m = torch.as_tensor(pairs_or_mask).to_dense() if getattr(pairs_or_mask, "is_sparse", False) else torch.as_tensor(pairs_or_mask)
            pairs_or_mask = m.nonzero().tolist()
        self.alignment_head_pairs = [(int(a), int(b)) for a, b in pairs_or_mask]
        self.missing_alignment_heads = False

    # ---- reference model-protocol bits ----
    @property
    def is_multilingual(self) -> bool:
        return self.dims.n_vocab >= 51865

    @property
    def num_languages(self) -> int:
        return self.dims.n_vocab - 51765 - int(self.is_multilingual)

    @property
    def alignment_heads(self) -> torch.Tensor:
        m = torch.zeros(self.dims.n_text_layer, self.dims.n_text_head, dtype=torch.bool)
        for l, h in self.alignment_head_pairs:
            m[l, h] = True
        return m.to_sparse()

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._lib.stb_model_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- packing ----
    def _dev(self, t: torch.Tensor) -> torch.Tensor:
        t = t.detach().to(self.device).contiguous()
        self._keep.append(t)
        return t

    def _set(self, tid: int, is_dec: int, layer: int, p0: torch.Tensor, p1: Optional[torch.Tensor] = None):
        L.check(self._lib.stb_model_set_tensor(self._h, tid, is_dec, layer, L.ptr(p0), L.ptr(p1)))

    def _set_split(self, tid, is_dec, layer, w: torch.Tensor):
        hi, lo = _split(w.to(self.device), self._want_lo)
        hi = self._dev(hi)
        lo = self._dev(lo) if lo is not None else None
        self._set(tid, is_dec, layer, hi, lo)

    def _set_f32(self, tid, is_dec, layer, w: torch.Tensor):
        self._set(tid, is_dec, layer, self._dev(w.float()))

    def _pack(self, sd: Dict[str, torch.Tensor]):
        D = self.dims
        g = lambda k: sd[k].detach().float()
        B = L.T_LAYER_BASE
        # encoder stem
        self._set_split(L.T_ENC_CONV1_W, 0, 0, g("encoder.conv1.weight").permute(0, 2, 1).reshape(D.n_audio_state, -1))
        self._set_f32(L.T_ENC_CONV1_B, 0, 0, g("encoder.conv1.bias"))
        self._set_split(L.T_ENC_CONV2_W, 0, 0, g("encoder.conv2.weight").permute(0, 2, 1).reshape(D.n_audio_state, -1))
        self._set_f32(L.T_ENC_CONV2_B, 0, 0, g("encoder.conv2.bias"))
        self._set_f32(L.T_ENC_POS, 0, 0, g("encoder.positional_embedding"))
        self._set_f32(L.T_ENC_LNPOST_G, 0, 0, g("encoder.ln_post.weight"))
        self._set_f32(L.T_ENC_LNPOST_B, 0, 0, g("encoder.ln_post.bias"))

        def block(prefix: str, is_dec: int, l: int, d: int):
            p = f"{prefix}.blocks.{l}."
            z = torch.zeros(d)
            self._set_f32(B + L.L_ATTN_LN_G, is_dec, l, g(p + "attn_ln.weight"))
            self._set_f32(B + L.L_ATTN_LN_B, is_dec, l, g(p + "attn_ln.bias"))
            self._set_split(B + L.L_QKV_W, is_dec, l, torch.cat([g(p + "attn.query.weight"), g(p + "attn.key.weight"),
                                                                 g(p + "attn.value.weight")]))
            self._set_f32(B + L.L_QKV_B, is_dec, l, torch.cat([g(p + "attn.query.bias"), z, g(p + "attn.value.bias")]))
            self._set_split(B + L.L_OUT_W, is_dec, l, g(p + "attn.out.weight"))
            self._set_f32(B + L.L_OUT_B, is_dec, l, g(p + "attn.out.bias"))
            self._set_f32(B + L.L_MLP_LN_G, is_dec, l, g(p + "mlp_ln.weight"))
            self._set_f32(B + L.L_MLP_LN_B, is_dec, l, g(p + "mlp_ln.bias"))
            self._set_split(B + L.L_FC1_W, is_dec, l, g(p + "mlp.0.weight"))
            self._set_f32(B + L.L_FC1_B, is_dec, l, g(p + "mlp.0.bias"))
            self._set_split(B + L.L_FC2_W, is_dec, l, g(p + "mlp.2.weight"))
            self._set_f32(B + L.L_FC2_B, is_dec, l, g(p + "mlp.2.bias"))
            if is_dec:
                self._set_f32(B + L.L_CROSS_LN_G, 1, l, g(p + "cross_attn_ln.weight"))
                self._set_f32(B + L.L_CROSS_LN_B, 1, l, g(p + "cross_attn_ln.bias"))
                self._set_split(B + L.L_CQ_W, 1, l, g(p + "cross_attn.query.weight"))
                self._set_f32(B + L.L_CQ_B, 1, l, g(p + "cross_attn.query.bias"))
                self._set_split(B + L.L_CKV_W, 1, l, torch.cat([g(p + "cross_attn.key.weight"),
                                                                g(p + "cross_attn.value.weight")]))
                self._set_f32(B + L.L_CKV_B, 1, l, torch.cat([z, g(p + "cross_attn.value.bias")]))
                self._set_split(B + L.L_COUT_W, 1, l, g(p + "cross_attn.out.weight"))
                self._set_f32(B + L.L_COUT_B, 1, l, g(p + "cross_attn.out.bias"))

        for l in range(D.n_audio_layer):
            block("encoder", 0, l, D.n_audio_state)
        for l in range(D.n_text_layer):
            block("decoder", 1, l, D.n_text_state)
        emb = g("decoder.token_embedding.weight")
        self._set_f32(L.T_DEC_TOKEMB_F32, 0, 0, emb)
        self._set_split(L.T_DEC_TOKEMB, 0, 0, emb)
        self._set_f32(L.T_DEC_POS, 0, 0, g("decoder.positional_embedding"))
        self._set_f32(L.T_DEC_LN_G, 0, 0, g("decoder.ln.weight"))
        self._set_f32(L.T_DEC_LN_B, 0, 0, g("decoder.ln.bias"))

    def _frontend_tables(self):
        n = np.arange(400, dtype=np.float64)
        window = (0.5 - 0.5 * np.cos(2.0 * np.pi * n / 400.0)).astype(np.float32)        # periodic Hann
        ang = 2.0 * np.pi * n / 400.0
        dft = np.stack([np.cos(ang), np.sin(ang)], axis=1).astype(np.float32)
        self._window = self._dev(torch.from_numpy(window))
        self._dft = self._dev(torch.from_numpy(dft))
        self._filters = self._dev(torch.from_numpy(mel_filterbank(self.dims.n_mels)))

    # ---- buffers ----
    def _buf(self, name: str, nbytes: int) -> torch.Tensor:
        t = self._ws.get(name)
        if t is None or t.numel() < nbytes:
            if t is not None:
                del self._ws[name]
            t = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=self.device)
            self._ws[name] = t
        return t

    # ---- a1 ----
    @_on_device
    def log_mel(self, audio: torch.Tensor, padded_samples: Optional[int] = None, batch_global_max: bool = False
                ) -> torch.Tensor:
        """audio fp32 [B, n] (device) -> mel fp32 [B, n_mels, 3000].  padded_samples=None pads to 30 s (align path)."""
        if audio.ndim == 1:
            audio = audio[None]
        audio = audio.to(self.device, torch.float32).contiguous()
        B, n = audio.shape
        if n > 480000:
            audio, n = audio[:, :480000].contiguous(), 480000
        padded = 480000 if padded_samples is None else int(padded_samples)
        mel = torch.empty(B, self.dims.n_mels, L.N_FRAMES, dtype=torch.float32, device=self.device)
        ws = self._buf("logmel", B * 376 * 4)
        L.check(self._lib.stb_logmel(L.ptr(audio), B, n, padded, self.dims.n_mels, L.ptr(self._filters), L.ptr(self._window),
                                     L.ptr(self._dft), int(batch_global_max), L.ptr(mel), L.ptr(ws), ws.numel(),
                                     L.stream_ptr()))
        return mel

    # ---- a2 ----
    @_on_device
    def encode(self, mel: torch.Tensor) -> Dict[str, torch.Tensor]:
        """mel fp32 [B, n_mels, 3000] -> {"f32": [B,1500,d], "hi": fp16 [B*1500,d], "lo": ...}."""
        if mel.ndim == 2:
            mel = mel[None]
        mel = mel.to(self.device, torch.float32).contiguous()
        B = mel.shape[0]
        d = self.dims.n_audio_state
        xa = torch.empty(B, L.N_AUDIO_CTX, d, dtype=torch.float32, device=self.device)
        hi = torch.empty(B * L.N_AUDIO_CTX, d, dtype=torch.float16, device=self.device)
        lo = torch.empty_like(hi) if self._want_lo else None
        ws = self._buf("enc", self._lib.stb_encoder_ws_bytes(self._h, B))
        L.check(self._lib.stb_encoder_forward(self._h, L.ptr(mel), B, L.ptr(xa), L.ptr(hi), L.ptr(lo), L.ptr(ws), ws.numel(),
                                              L.stream_ptr()))
        return {"f32": xa, "hi": hi, "lo": lo, "B": B}

    @_on_device
    def cross_kv(self, enc: Dict[str, torch.Tensor], decode: bool = False, reuse: bool = False) -> torch.Tensor:
        """Cross-attention K / V^T of every decoder layer; ``decode=True`` also lays V out for the KV-cached decode step.
        ``reuse=True`` writes into a buffer owned by the model (overwritten by the next such call): a batch of 120
        large-v3 windows is an 82 GB block, and returning it to the caching allocator every step costs ~1 s."""
        B = enc["B"]
        nbytes = self._lib.stb_cross_kv_bytes(self._h, B)
        out = self._buf("cross_kv", nbytes) if reuse else torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        L.check(self._lib.stb_cross_kv(self._h, L.ptr(enc["hi"]), L.ptr(enc["lo"]), B, int(decode), L.ptr(out), L.stream_ptr()))
        return out

    # ---- a3 ----
    @_on_device
    def decode_forced(self, tokens: torch.Tensor, ckv: torch.Tensor, want_logits: bool = True,
                      heads: Union[None, str, Sequence[Tuple[int, int]]] = None, reuse: bool = False):
        """tokens int [B, M] -> (logits fp32 [B, M, V] view or None, qk fp32 [B, n_sel, M, 1504] or None).
        ``reuse=True``: both outputs live in model-owned buffers (valid until the next such call)."""
        tokens = tokens.to(self.device, torch.int32).contiguous()
        B, M = tokens.shape
        V = self.dims.n_vocab
        ldv = (V + 7) // 8 * 8
        def out(name, *shape):
            n = 1
            for v in shape:
                n *= v
            if reuse:
                return self._buf(name, 4 * n)[: 4 * n].view(torch.float32).view(*shape)
            return torch.empty(*shape, dtype=torch.float32, device=self.device)
        logits = out("dec_logits", B * M, ldv) if want_logits else None
        qk, sel, n_sel = None, None, 0
        if heads is not None:
            if isinstance(heads, str):
                assert heads == "all"
                n_sel = -1
                n_tot = self.dims.n_text_layer * self.dims.n_text_head
            else:
                flat = [int(v) for pair in heads for v in pair]
                sel = (ctypes.c_int32 * len(flat))(*flat)
                n_sel = n_tot = len(heads)
            qk = out("dec_qk", B, n_tot, M, L.KPAD)
        ws = self._buf("dec", self._lib.stb_decoder_ws_bytes(self._h, B, M))
        L.check(self._lib.stb_decoder_forward(self._h, L.ptr(tokens), B, M, L.ptr(ckv), L.ptr(logits), ldv, L.ptr(qk), sel,
                                              n_sel, L.ptr(ws), ws.numel(), L.stream_ptr()))
        lv = logits.view(B, M, ldv)[:, :, :V] if want_logits else None
        return lv, qk

    # ---- a4 / a10 ----
    @_on_device
    def token_probs(self, logits_rows: torch.Tensor, n_classes: int, targets: torch.Tensor, want_rank: bool = False):
        """logits_rows fp32 [n, >=n_classes] (row-strided view ok) -> (prob fp32 [n], rank int32 [n] | None)."""
        assert logits_rows.stride(-1) == 1
        n = logits_rows.shape[0]
        targets = targets.to(self.device, torch.int32).contiguous()
        prob = torch.empty(n, dtype=torch.float32, device=self.device)
        rank = torch.empty(n, dtype=torch.int32, device=self.device) if want_rank else None
        L.check(self._lib.stb_token_probs(L.ptr(logits_rows), logits_rows.stride(0), n, int(n_classes), L.ptr(targets),
                                          L.ptr(prob), L.ptr(rank), L.stream_ptr()))
        return prob, rank

    @_on_device
    def softmax_probs(self, logits_rows: torch.Tensor, n_classes: int) -> torch.Tensor:
        """logits_rows fp32 [n, >=n_classes] (row-strided view ok) -> probabilities fp32 [n, n_classes] (device)."""
        assert logits_rows.stride(-1) == 1
        n = logits_rows.shape[0]
        out = torch.empty(n, int(n_classes), dtype=torch.float32, device=self.device)
        L.check(self._lib.stb_softmax_probs(L.ptr(logits_rows), logits_rows.stride(0), n, int(n_classes), L.ptr(out),
                                            int(n_classes), L.stream_ptr()))
        return out

    # ---- a5 ----
    @_on_device
    def qk_postprocess(self, qk: torch.Tensor, S: int, F: int, R: Optional[int] = None, qk_scale: float = 1.0,
                       medfilt_width: int = 7) -> torch.Tensor:
        """qk fp32 [B, A, M, ld] -> matrix fp32 [B, R, F]; R defaults to M-1-S (the reference's [S:-1] slice)."""
        B, A, M, ld = qk.shape
        assert qk.is_contiguous()
        R = M - 1 - S if R is None else int(R)
        ldm = (F + 3) // 4 * 4
        out = torch.empty(B, R, ldm, dtype=torch.float32, device=self.device)
        ws = self._buf("qkpost", self._lib.stb_qkpost_ws_bytes(B, A, R, F))
        L.check(self._lib.stb_qk_postprocess(L.ptr(qk), B, A, M, ld, S, R, F, float(qk_scale), medfilt_width, L.ptr(out),
                                             ldm, L.ptr(ws), ws.numel(), L.stream_ptr()))
        return out[:, :, :F]

    @_on_device
    def qk_postprocess_dynamic(self, qk_all: torch.Tensor, S: int, F: int, R: Optional[int] = None, count: int = 6,
                               prev_jumps: Optional[torch.Tensor] = None, reuse_softmax: bool = False,
                               qk_scale: float = 1.0, medfilt_width: int = 7) -> torch.Tensor:
        """Per-token dynamic head selection (timing.py:85-103): qk_all fp32 [B, L*H, M, ld] -> matrix [B, R, F]."""
        B, LH, M, ld = qk_all.shape
        assert qk_all.is_contiguous()
        R = M - 1 - S if R is None else int(R)
        ldm = (F + 3) // 4 * 4
        out = torch.empty(B, R, ldm, dtype=torch.float32, device=self.device)
        ws = self._buf("qkpost_dyn", self._lib.stb_qkpost_dynamic_ws_bytes(B, LH, R, F, count))
        pj = None if prev_jumps is None else prev_jumps.to(self.device, torch.int32).contiguous()
        L.check(self._lib.stb_qk_postprocess_dynamic(L.ptr(qk_all), B, LH, M, ld, S, R, F, float(qk_scale), medfilt_width,
                                                     int(count), L.ptr(pj), int(reuse_softmax), L.ptr(out), ldm, L.ptr(ws),
                                                     ws.numel(), L.stream_ptr()))
        return out[:, :, :F]

    @_on_device
    def qk_postprocess_new(self, qk_all: torch.Tensor, S: int, F: int, R: Optional[int] = None, topk: int = 20,
                           w_colnorm: float = 1.0, w_rownorm: float = 1.0, w_coverage: float = 0.0, qk_scale: float = 1.0,
                           medfilt_width: int = 7) -> torch.Tensor:
        """The "new" aligner's head scoring (timing.py:115-163): qk_all fp32 [B, L*H, M, ld] -> matrix [B, R, F]."""
        B, LH, M, ld = qk_all.shape
        assert qk_all.is_contiguous()
        R = M - 1 - S if R is None else int(R)
        ldm = (F + 3) // 4 * 4
        out = torch.empty(B, R, ldm, dtype=torch.float32, device=self.device)
        ws = self._buf("qkpost_new", self._lib.stb_qkpost_new_ws_bytes(B, LH, M, F, topk))
        L.check(self._lib.stb_qk_postprocess_new(L.ptr(qk_all), B, LH, M, ld, S, R, F, float(qk_scale), medfilt_width, int(topk),
                                                 float(w_colnorm), float(w_rownorm), float(w_coverage), L.ptr(out), ldm,
                                                 L.ptr(ws), ws.numel(), L.stream_ptr()))
        return out[:, :, :F]

    @_on_device
    def scale_add(self, y: torch.Tensor, x: torch.Tensor, a: float, b: float) -> torch.Tensor:
        """y = a * x + b * y in place for two matrices returned by ``qk_postprocess*`` (same shape: the views' padded base
        buffers are combined whole).  Used to average the attention matrices of ``extra_models`` (timing.py:177-189)."""
        yb = y._base if y._base is not None else y
        xb = x._base if x._base is not None else x
        assert y.shape == x.shape and yb.shape == xb.shape and yb.is_contiguous() and xb.is_contiguous()
        L.check(self._lib.stb_axpby(L.ptr(yb), L.ptr(xb.to(self.device)), float(a), float(b), yb.numel(), L.stream_ptr()))
        return y

    # ---- a6 ----
    @_on_device
    def dtw(self, matrix: torch.Tensor, negate: bool = True, want_path: bool = False):
        """matrix fp32 [B, R, F] (row-strided view ok) -> jumps int32 [B, R] (+ path int32 [B, 2, R+F], len [B])."""
        B, R, F = matrix.shape
        assert matrix.stride(2) == 1 and matrix.stride(0) == R * matrix.stride(1)
        jumps = torch.empty(B, R, dtype=torch.int32, device=self.device)
        path = torch.empty(B, 2, R + F, dtype=torch.int32, device=self.device) if want_path else None
        plen = torch.empty(B, dtype=torch.int32, device=self.device) if want_path else None
        ws = self._buf("dtw", self._lib.stb_dtw_ws_bytes(B, R, F))
        L.check(self._lib.stb_dtw(L.ptr(matrix), B, R, F, matrix.stride(1), int(negate), L.ptr(jumps), L.ptr(path),
                                  L.ptr(plen), L.ptr(ws), ws.numel(), L.stream_ptr()))
        return (jumps, path, plen) if want_path else jumps


def from_oracle(model, device="cuda", precision="fp16x3") -> B200Whisper:
    """Build from any object with ``dims`` + ``state_dict()`` using openai-whisper key names (tests / loaders)."""
    pairs = None
    ah = getattr(model, "alignment_heads", None)
    if ah is not None:
        idx = ah.indices().T.tolist() if ah.is_sparse else ah.nonzero().tolist()
        pairs = [(int(a), int(b)) for a, b in idx]
    return B200Whisper(model.dims, model.state_dict(), device=device, precision=precision, alignment_heads=pairs)
