"""Drop-in ``Clair3_P`` / ``Clair3_F`` for the reference's callers, backed by the sm_90a kernels.

Mirrors the module protocol the reference uses (HKU-BAL/Clair3 paths):

    m = Clair3_P|Clair3_F(add_indel_length, predict=True, input_channels)   clair3/CallVariantsFromCffi.py:230-243
    m.to(device); m.eval(); m.load_state_dict(state_dict)                    clair3/CallVariantsFromCffi.py:19-28,246-248
    Y = m(X)    # X int8/int32/float tensor [B,33,18] or [B,D,33,C]; Y float32 [B,24|90] on X's device   :48-52

Constructor arguments, state_dict keys (strict), output head order and dtype are the reference's
(``clair3/model.py:58-161`` and ``:282-416``).  Everything numeric happens in ``libclair3b200.so``; there is no
PyTorch or CPU implementation behind these classes, and constructing one without an H100 raises.
"""
from __future__ import annotations

import numpy as np
import torch

from ._ffi import CONSTANTS as K
from ._ffi import C3BError, check, ffi, lib

_DT = {torch.int8: K["C3B_DT_I8"], torch.int32: K["C3B_DT_I32"], torch.float32: K["C3B_DT_F32"]}

# c3b_call (include/clair3_b200.h) as a numpy record
CALL_DTYPE = np.dtype([("dp", "<i8"), ("support", "<i8"), ("ref_count", "<i8"), ("prob", "<f4"), ("ref_len", "<i4"),
                       ("alt_len", "<i4"), ("n_ad", "<i4"), ("flags", "<u2"), ("genotype", "u1"), ("printed", "u1"),
                       ("status", "u1"), ("pad", "u1", (3,))])
assert CALL_DTYPE.itemsize == ffi.sizeof("c3b_call")


def call_config(output_config):
    """(C3B_CALL_* bits, maximum_variant_length_that_need_infer) of an object with the reference's OutputConfig fields."""
    bits = 0
    for name, bit in (("is_show_reference", "C3B_CALL_SHOW_REF"), ("is_haploid_precise_mode_enabled", "C3B_CALL_HAPLOID_PRECISE"),
                      ("is_haploid_sensitive_mode_enabled", "C3B_CALL_HAPLOID_SENSITIVE"),
                      ("enable_long_indel", "C3B_CALL_LONG_INDEL"), ("keep_iupac_bases", "C3B_CALL_KEEP_IUPAC")):
        if getattr(output_config, name):
            bits |= K[bit]
    max_len = output_config.maximum_variant_length_that_need_infer
    if isinstance(max_len, bool) or not isinstance(max_len, (int, np.integer)):
        raise C3BError("maximum_variant_length_that_need_infer must be an integer, got %r" % (max_len,))
    return bits, int(np.clip(int(max_len), -(1 << 62), 1 << 62))


class _C3BModule:
    _kind = None
    _default_channels = None

    def __init__(self, add_indel_length=False, predict=False, input_channels=None):
        self.add_indel_length = bool(add_indel_length)
        self.predict = bool(predict)
        self.input_channels = int(input_channels) if input_channels is not None else self._default_channels
        self.output_label_split = [21, 3, 33, 33]
        self.training = False
        self._device = None
        self._handle = None
        self._state = None
        self._by_broadcast = False
        self._options = {}

    # ---- torch.nn.Module-shaped surface used by the reference callers
    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise C3BError("clair3_b200 runs only on a CUDA (sm_90a) device; there is no CPU path "
                           "(requested device: %s)" % device)
        index = device.index if device.index is not None else torch.cuda.current_device()
        if self._handle is not None and self._device is not None and self._device.index == index:
            return self
        self._release()
        out = ffi.new("c3b_model **")
        check(lib().c3b_create(out, self._kind, self.input_channels, int(self.add_indel_length), index))
        self._handle = out[0]
        self._device = torch.device("cuda", index)
        for k, v in self._options.items():
            check(lib().c3b_set_option(self._handle, k.encode(), int(v)))
        if self._state is not None:
            self._upload(self._state)
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", device if device is not None else torch.cuda.current_device()))

    def eval(self):
        self.training = False
        return self

    def train(self, mode=True):
        if mode:
            raise C3BError("clair3_b200 implements the inference forward only (reference training is clair3/Train.py)")
        return self

    def state_dict(self):
        if self._by_broadcast:
            raise C3BError("this rank received packed weight images by broadcast; the state_dict lives on the source rank")
        return dict(self._state or {})

    def load_state_dict(self, state_dict, strict=True):
        sd = {}
        for k, v in state_dict.items():
            t = v.detach().cpu() if isinstance(v, torch.Tensor) else torch.as_tensor(np.asarray(v))
            sd[k] = t
        self._state = sd
        if self._handle is None:
            if torch.cuda.is_available():
                self.to(torch.device("cuda"))
            else:
                raise C3BError("no CUDA device: clair3_b200 has no CPU fallback")
        else:
            self._upload(sd)
        return self

    def set_option(self, name, value):
        """Kernel options: precision (0 fp16 tensor cores | 1 fp32 debug), chunk_sites, lstm_tile, lstm_wg, lstm2_split, profile,
        taps."""
        self._options[name] = int(value)
        if self._handle is not None:
            check(lib().c3b_set_option(self._handle, name.encode(), int(value)))
        return self

    def _upload(self, sd):
        L = lib()
        for key, t in sd.items():
            if t.dtype == torch.int64:
                arr = t.contiguous().numpy()
                dt = K["C3B_DT_I64"]
            else:
                arr = t.to(torch.float32).contiguous().numpy()
                dt = K["C3B_DT_F32"]
            dims = list(t.shape)                         # 0-d tensors (num_batches_tracked) keep ndim = 0
            shape = ffi.new("int64_t[]", dims or [0])
            check(L.c3b_set_param(self._handle, key.encode(), ffi.cast("void *", arr.ctypes.data), dt, shape, len(dims)))
        check(L.c3b_finalize(self._handle))

    @property
    def out_dim(self):
        return 90 if self.add_indel_length else 24

    def _check_input(self, x, who):
        """Shape / dtype / handle validation shared by every forward entry (the C-ABI trusts batch, depth and dtype)."""
        if self._handle is None:
            raise C3BError("model has no device/weights yet: call .to(device) and .load_state_dict() first")
        want_nd = 3 if self._kind == K["C3B_PILEUP"] else 4
        if x.ndim != want_nd or x.shape[-1] != self.input_channels or x.shape[-2] != 33:
            raise C3BError("%s: expected input [B,%s33,%d], got %s" % (who, "" if want_nd == 3 else "depth,", self.input_channels,
                                                                       tuple(x.shape)))
        return x.shape[0], (x.shape[1] if want_nd == 4 else 0)

    def forward(self, x):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(x)
        batch, depth = self._check_input(x, "forward")
        if x.dtype not in _DT:
            x = x.to(torch.int32) if not x.dtype.is_floating_point else x.to(torch.float32)
        x = x.contiguous()
        on_dev = x.device.type == "cuda"
        if on_dev and x.device.index != self._device.index:
            raise C3BError("input is on %s but the model is on %s" % (x.device, self._device))
        y = torch.empty((batch, self.out_dim), dtype=torch.float32, device=x.device if on_dev else "cpu")
        if batch == 0:
            return self._split(y)
        stream = torch.cuda.current_stream(self._device).cuda_stream
        check(lib().c3b_forward(self._handle, ffi.cast("void *", x.data_ptr()), _DT[x.dtype], int(on_dev), batch, depth,
                                ffi.cast("float *", y.data_ptr()), int(on_dev), ffi.cast("void *", stream)))
        return self._split(y)

    __call__ = forward

    def forward_into(self, x, y):
        """``forward`` on device tensors with a caller-provided output (no allocation per call; asynchronous on the current
        stream).  x, y on the model's device, y float32 [B, out_dim] contiguous."""
        batch, depth = self._check_input(x, "forward_into")
        if x.device != self._device or y.device != self._device or x.dtype not in _DT or not x.is_contiguous():
            raise C3BError("forward_into: contiguous int8/int32/float32 x and y on %s" % self._device)
        if tuple(y.shape) != (batch, self.out_dim) or y.dtype != torch.float32 or not y.is_contiguous():
            raise C3BError("forward_into: y must be contiguous float32 [batch, %d]" % self.out_dim)
        stream = torch.cuda.current_stream(self._device).cuda_stream
        check(lib().c3b_forward(self._handle, ffi.cast("void *", x.data_ptr()), _DT[x.dtype], 1, batch, depth,
                                ffi.cast("float *", y.data_ptr()), 1, ffi.cast("void *", stream)))
        return y

    def forward_async(self, x_host, y_host):
        """Stream-ordered forward on PINNED host tensors (H2D -> kernels -> D2H on the current CUDA stream, no host
        synchronisation; ``c3b_forward_async``): the double-buffered caller of SURVEY.md §8f N1.  The caller synchronises the
        stream before reading ``y_host`` and must keep both tensors alive until then."""
        batch, depth = self._check_input(x_host, "forward_async")
        if not (x_host.is_pinned() and y_host.is_pinned()):
            raise C3BError("forward_async needs pinned host tensors")
        if x_host.dtype not in _DT or not x_host.is_contiguous() or y_host.dtype != torch.float32 or not y_host.is_contiguous():
            raise C3BError("forward_async: x must be contiguous int8/int32/float32, y contiguous float32")
        if tuple(y_host.shape) != (batch, self.out_dim):
            raise C3BError("forward_async: y must be [batch, %d]" % self.out_dim)
        stream = torch.cuda.current_stream(self._device).cuda_stream
        check(lib().c3b_forward_async(self._handle, ffi.cast("void *", x_host.data_ptr()), _DT[x_host.dtype], batch, depth,
                                      ffi.cast("float *", y_host.data_ptr()), ffi.cast("void *", stream)))
        return y_host

    def forward_windows(self, cols, starts, y=None, sync=True, bounds=None):
        """Pileup only: ``c3b_forward_windows``.  ``cols`` is the per-column count matrix [n_cols, 18] (int64 = libclair3's
        ``plp_data.matrix``, or int32 / int8 / float32), ``starts`` the int64 first row of every candidate's 33-row window
        (``preprocess/CreateTensorPileupFromCffi.py:359``: ``offset = pos - flanking - first_pos - 1``); both on the host
        or both on the model's device.  ``bounds`` (optional, int64 [len(starts), 2] on the same side; pinned with
        ``sync=False``): window b reads only rows [bounds[b, 0], bounds[b, 1]) and zeros elsewhere
        (``c3b_forward_windows_bounded``) - the reference's zero padding outside a candidate's contiguous run (:374-391), as
        ``PileupCounter.window_bounds()`` gives it.  Returns float32 [len(starts), 24|90] on the same side."""
        if self._handle is None:
            raise C3BError("model has no device/weights yet: call .to(device) and .load_state_dict() first")
        if self._kind != K["C3B_PILEUP"]:
            raise C3BError("forward_windows is a pileup feature")
        if isinstance(cols, np.ndarray):
            cols = torch.from_numpy(cols)
        if isinstance(starts, np.ndarray):
            starts = torch.from_numpy(starts)
        if cols.ndim != 2 or cols.shape[1] != self.input_channels:
            raise C3BError("forward_windows: cols must be [n_cols, %d], got %s" % (self.input_channels, tuple(cols.shape)))
        dt = dict(_DT)
        dt[torch.int64] = K["C3B_DT_I64"]
        if cols.dtype not in dt:
            raise C3BError("forward_windows: cols dtype %s (int64/int32/int8/float32)" % cols.dtype)
        if starts.ndim != 1 or cols.device != starts.device:
            raise C3BError("forward_windows: starts must be 1-D and on the same device as cols")
        cols = cols.contiguous()
        starts = starts.to(torch.int64).contiguous()
        on_dev = cols.device.type == "cuda"
        batch = starts.shape[0]
        if bounds is not None:
            if isinstance(bounds, np.ndarray):
                bounds = torch.from_numpy(bounds)
            if tuple(bounds.shape) != (batch, 2) or bounds.device != starts.device:
                raise C3BError("forward_windows: bounds must be [len(starts), 2] on the same device as starts")
            bounds = bounds.to(torch.int64).contiguous()
        if y is None:
            y = torch.empty((batch, self.out_dim), dtype=torch.float32, device=cols.device)
        if tuple(y.shape) != (batch, self.out_dim) or y.dtype != torch.float32 or not y.is_contiguous():
            raise C3BError("forward_windows: y must be contiguous float32 [batch, %d]" % self.out_dim)
        if not sync and not on_dev and not (cols.is_pinned() and starts.is_pinned() and y.is_pinned()
                                            and (bounds is None or bounds.is_pinned())):
            raise C3BError("forward_windows(sync=False) needs pinned host tensors")
        if batch == 0:
            return y
        stream = torch.cuda.current_stream(self._device).cuda_stream
        bptr = ffi.NULL if bounds is None else ffi.cast("int64_t *", bounds.data_ptr())
        check(lib().c3b_forward_windows_bounded(self._handle, ffi.cast("void *", cols.data_ptr()), dt[cols.dtype], cols.shape[0],
                                                ffi.cast("int64_t *", starts.data_ptr()), bptr, int(on_dev), batch,
                                                ffi.cast("float *", y.data_ptr()), int(y.device.type == "cuda"), int(bool(sync)),
                                                ffi.cast("void *", stream)))
        return y

    def decode_stage1(self, y, ref_gt21):
        """``c3b_decode_stage1``: the data-parallel first stage of the reference's ``batch_output`` (``clair3/CallVariants.py:
        510-576,1069-1116``) on the GPU.  ``y`` [B, out_dim] float32 and ``ref_gt21`` [B] uint8 (gt21 index of ref+ref:
        A 0, C 4, G 7, T 9) on the same device (cuda: asynchronous on the current stream; cpu: complete on return).
        Returns a dict of tensors: is_ref, ref_prob, argmax [B,heads], maxprob, qual (float64), nonref_idx, n_nonref."""
        if self._handle is None:
            raise C3BError("model has no device yet")
        if isinstance(y, np.ndarray):
            y = torch.from_numpy(y)
        if isinstance(ref_gt21, np.ndarray):
            ref_gt21 = torch.from_numpy(ref_gt21)
        if y.ndim != 2 or y.shape[1] != self.out_dim or y.dtype != torch.float32:
            raise C3BError("decode_stage1: y must be float32 [B, %d]" % self.out_dim)
        ref_gt21 = ref_gt21.to(torch.uint8)
        if ref_gt21.shape != (y.shape[0],) or ref_gt21.device != y.device:
            raise C3BError("decode_stage1: ref_gt21 must be [B] on y's device")
        if ref_gt21.numel() and int(ref_gt21.max()) > 20:
            raise C3BError("decode_stage1: ref_gt21 holds gt21 indices (0..20)")
        y = y.contiguous()
        ref_gt21 = ref_gt21.contiguous()
        B, nh, dev = y.shape[0], (4 if self.add_indel_length else 2), y.device
        out = {"is_ref": torch.empty(B, dtype=torch.uint8, device=dev), "ref_prob": torch.empty(B, dtype=torch.float32, device=dev),
               "argmax": torch.empty((B, nh), dtype=torch.int32, device=dev), "maxprob": torch.empty((B, nh), dtype=torch.float32, device=dev),
               "qual": torch.empty(B, dtype=torch.float64, device=dev), "nonref_idx": torch.empty(B, dtype=torch.int32, device=dev),
               "n_nonref": torch.zeros(1, dtype=torch.int32, device=dev)}
        stream = torch.cuda.current_stream(self._device).cuda_stream
        c = ffi.cast
        check(lib().c3b_decode_stage1(self._handle, c("float *", y.data_ptr()), c("uint8_t *", ref_gt21.data_ptr()), B,
                                      int(dev.type == "cuda"), c("uint8_t *", out["is_ref"].data_ptr()),
                                      c("float *", out["ref_prob"].data_ptr()), c("int32_t *", out["argmax"].data_ptr()),
                                      c("float *", out["maxprob"].data_ptr()), c("double *", out["qual"].data_ptr()),
                                      c("int32_t *", out["nonref_idx"].data_ptr()), c("int32_t *", out["n_nonref"].data_ptr()),
                                      c("void *", stream)))
        return out

    def decode_stage2(self, y, ref_gt21, sites=None, n_sites=None, k=16):
        """``c3b_decode_stage2``: each listed site's genotype outcomes in the order the reference's ``output_from`` tries them
        (``clair3/CallVariants.py:676-1012``), first ``k`` (1..1024) entries, ending at homo_Ref.  ``y`` / ``ref_gt21`` as for
        ``decode_stage1``; ``sites`` int32 [S] row indices (default: every row) and ``n_sites`` int32 [1] how many of them are
        listed (default S) - stage 1's ``nonref_idx`` / ``n_nonref`` chain in with no host synchronisation.  All on y's device
        (cuda: asynchronous on the current stream; cpu: complete on return).  Returns a dict of tensors: cat uint8 [S,k]
        (0 homo_Ref .. 9 hetero_InsDel, 255 unused), idx int16 [S,k] (index in the category's list), prob float32 [S,k],
        tie_mask int16 [S,k] (bit c: the is_* flag of category c if this attempt succeeds), count int32 [S], complete uint8 [S]."""
        if self._handle is None:
            raise C3BError("model has no device yet")
        if isinstance(y, np.ndarray):
            y = torch.from_numpy(y)
        if isinstance(ref_gt21, np.ndarray):
            ref_gt21 = torch.from_numpy(ref_gt21)
        if isinstance(sites, np.ndarray):
            sites = torch.from_numpy(sites)
        if isinstance(n_sites, np.ndarray):
            n_sites = torch.from_numpy(n_sites)
        if y.ndim != 2 or y.shape[1] != self.out_dim or y.dtype != torch.float32:
            raise C3BError("decode_stage2: y must be float32 [B, %d]" % self.out_dim)
        ref_gt21 = ref_gt21.to(torch.uint8)
        if ref_gt21.shape != (y.shape[0],) or ref_gt21.device != y.device:
            raise C3BError("decode_stage2: ref_gt21 must be [B] on y's device")
        if ref_gt21.numel() and int(ref_gt21.max()) > 20:
            raise C3BError("decode_stage2: ref_gt21 holds gt21 indices (0..20)")
        if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= int(k) <= 1024:
            raise C3BError("decode_stage2: k must be an integer in [1, 1024], got %r" % (k,))
        k = int(k)
        if sites is not None:
            if sites.ndim != 1 or sites.device != y.device or sites.dtype not in (torch.int32, torch.int64):
                raise C3BError("decode_stage2: sites must be a 1-D int32 tensor on y's device")
            sites = sites.to(torch.int32).contiguous()
        if n_sites is not None:
            if n_sites.numel() != 1 or n_sites.device != y.device or n_sites.dtype != torch.int32:
                raise C3BError("decode_stage2: n_sites must be one int32 on y's device")
            n_sites = n_sites.reshape(1).contiguous()
        y = y.contiguous()
        ref_gt21 = ref_gt21.contiguous()
        B, dev = y.shape[0], y.device
        S = B if sites is None else sites.shape[0]
        out = {"cat": torch.empty((S, k), dtype=torch.uint8, device=dev), "idx": torch.empty((S, k), dtype=torch.int16, device=dev),
               "prob": torch.empty((S, k), dtype=torch.float32, device=dev),
               "tie_mask": torch.empty((S, k), dtype=torch.int16, device=dev),
               "count": torch.zeros(S, dtype=torch.int32, device=dev), "complete": torch.zeros(S, dtype=torch.uint8, device=dev)}
        if S == 0:
            return out
        stream = torch.cuda.current_stream(self._device).cuda_stream
        c = ffi.cast
        ptr = lambda t, ty: c(ty, t.data_ptr()) if t is not None else ffi.NULL          # noqa: E731
        check(lib().c3b_decode_stage2(self._handle, c("float *", y.data_ptr()), c("uint8_t *", ref_gt21.data_ptr()), B,
                                      ptr(sites, "int32_t *"), ptr(n_sites, "int32_t *"), S, k, int(dev.type == "cuda"),
                                      c("uint8_t *", out["cat"].data_ptr()), c("uint16_t *", out["idx"].data_ptr()),
                                      c("float *", out["prob"].data_ptr()), c("uint16_t *", out["tie_mask"].data_ptr()),
                                      c("int32_t *", out["count"].data_ptr()), c("uint8_t *", out["complete"].data_ptr()),
                                      c("void *", stream)))
        return out

    def decode_calls(self, y, ref_base, alt_bytes, alt_offsets, config, k=16):
        """``c3b_decode_calls``: every site's call as data - stage 1, stage 2 (first ``k`` entries), the walk of each
        non-reference site's ranked outcomes against its alt_info, the full re-rank of the sites whose k entries run out, and
        what ``output_with`` reads for the row (``clair3_b200.decode.format_row`` without the QUAL, FILTER and AF text).
        ``y`` float32 [B, out_dim]; ``ref_base`` uint8 [B] the raw reference character at each window's centre;
        ``alt_bytes`` uint8 [N] the alt_info strings concatenated, site s at ``alt_bytes[alt_offsets[s]:alt_offsets[s + 1]]``
        (``alt_offsets`` int64 [B + 1]); all on y's device (cuda: asynchronous on the current stream; cpu: complete on
        return).  ``config``: an object with the reference's ``OutputConfig`` field names.  Returns a dict of tensors:
        ``calls`` uint8 [B, 48] (``CALL_DTYPE`` records), ``text`` uint8 and ``ad`` int64, both [2 N + 8 B] (site s's REF,
        ALT and allele counts from index ``2 * alt_offsets[s] + 8 * s``)."""
        if self._handle is None:
            raise C3BError("model has no device yet")
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)) if isinstance(a, np.ndarray) else a      # noqa: E731
        y, ref_base, alt_bytes, alt_offsets = t(y), t(ref_base), t(alt_bytes), t(alt_offsets)
        if y.ndim != 2 or y.shape[1] != self.out_dim or y.dtype != torch.float32:
            raise C3BError("decode_calls: y must be float32 [B, %d]" % self.out_dim)
        B, dev = y.shape[0], y.device
        if ref_base.shape != (B,) or ref_base.dtype != torch.uint8 or ref_base.device != dev:
            raise C3BError("decode_calls: ref_base must be uint8 [B] on y's device")
        if alt_bytes.ndim != 1 or alt_bytes.dtype != torch.uint8 or alt_bytes.device != dev:
            raise C3BError("decode_calls: alt_bytes must be a 1-D uint8 tensor on y's device")
        if alt_offsets.shape != (B + 1,) or alt_offsets.dtype != torch.int64 or alt_offsets.device != dev:
            raise C3BError("decode_calls: alt_offsets must be int64 [B + 1] on y's device")
        if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= int(k) <= 1024:
            raise C3BError("decode_calls: k must be an integer in [1, 1024], got %r" % (k,))
        if bool(config.add_indel_length) != self.add_indel_length:
            raise C3BError("decode_calls: config.add_indel_length must match the model")
        bits, max_len = call_config(config)
        y, ref_base, alt_bytes, alt_offsets = y.contiguous(), ref_base.contiguous(), alt_bytes.contiguous(), alt_offsets.contiguous()
        N = alt_bytes.shape[0]
        out = {"calls": torch.zeros((B, CALL_DTYPE.itemsize), dtype=torch.uint8, device=dev),
               "text": torch.zeros(2 * N + 8 * B, dtype=torch.uint8, device=dev),
               "ad": torch.zeros(2 * N + 8 * B, dtype=torch.int64, device=dev)}
        if B == 0:
            return out
        stream = torch.cuda.current_stream(self._device).cuda_stream
        c = ffi.cast
        check(lib().c3b_decode_calls(self._handle, c("float *", y.data_ptr()), c("uint8_t *", ref_base.data_ptr()), B,
                                     c("char *", alt_bytes.data_ptr()), c("int64_t *", alt_offsets.data_ptr()), N, bits, max_len,
                                     int(k), int(dev.type == "cuda"), c("c3b_call *", out["calls"].data_ptr()),
                                     c("char *", out["text"].data_ptr()), c("int64_t *", out["ad"].data_ptr()), c("void *", stream)))
        return out

    def predict_stream(self, batches, streams=8):
        """Pipelined ``_torch_predict`` (``clair3/CallVariantsFromCffi.py:48-52,300-331``): consume an iterable of host batches
        (numpy arrays or CPU tensors, ragged sizes allowed) and yield one float32 numpy ``Y`` per batch, in order, while up to
        ``streams`` batches are in flight - H2D, kernels and D2H of consecutive batches overlap on as many CUDA streams, each
        with its own activation workspace and pinned staging buffers.  A caller written as
        ``for X, ... in generator: Y = _torch_predict(m, device, X)`` becomes ``for Y in m.predict_stream(X for X, ... in generator)``."""
        if self._handle is None:
            raise C3BError("model has no device/weights yet: call .to(device) and .load_state_dict() first")
        n = max(1, int(streams))
        with torch.cuda.device(self._device):
            cu = [torch.cuda.Stream(self._device) for _ in range(n)]
        slots = [{"x": None, "y": None, "ev": None, "batch": 0} for _ in range(n)]
        pending = []                       # slot indices in issue order

        def finish(i):
            sl = slots[i]
            sl["ev"].synchronize()
            return sl["y"][:sl["batch"]].numpy().copy()

        k = 0
        for xb in batches:
            if isinstance(xb, np.ndarray):
                xb = torch.from_numpy(xb)
            if xb.dtype not in _DT:
                xb = xb.to(torch.int32) if not xb.dtype.is_floating_point else xb.to(torch.float32)
            batch, depth = self._check_input(xb, "predict_stream")
            i = k % n
            if len(pending) == n:          # the slot about to be reused is the oldest in flight
                yield finish(pending.pop(0))
            sl = slots[i]
            if batch:
                if xb.is_pinned() and xb.is_contiguous():
                    xp = xb
                else:
                    need = xb.numel()
                    if sl["x"] is None or sl["x"].numel() < need or sl["x"].dtype != xb.dtype:
                        sl["x"] = torch.empty(max(need, 1), dtype=xb.dtype).pin_memory()
                    xp = sl["x"][:need].view(xb.shape)
                    xp.copy_(xb)
                if sl["y"] is None or sl["y"].shape[0] < batch:
                    sl["y"] = torch.empty((max(batch, 1), self.out_dim), dtype=torch.float32).pin_memory()
                with torch.cuda.stream(cu[i]):
                    check(lib().c3b_forward_async(self._handle, ffi.cast("void *", xp.data_ptr()), _DT[xp.dtype], batch, depth,
                                                  ffi.cast("float *", sl["y"].data_ptr()), ffi.cast("void *", cu[i].cuda_stream)))
                    sl["ev"] = torch.cuda.Event()
                    sl["ev"].record(cu[i])
                sl["keep"] = xp
            else:
                if sl["y"] is None:
                    sl["y"] = torch.empty((1, self.out_dim), dtype=torch.float32).pin_memory()
                sl["ev"] = torch.cuda.Event()
                sl["ev"].record(cu[i])
            sl["batch"] = batch
            pending.append(i)
            k += 1
        while pending:
            yield finish(pending.pop(0))

    def _split(self, y):
        if self.predict:
            return y
        sizes = self.output_label_split[:4 if self.add_indel_length else 2]
        return list(torch.split(y, sizes, dim=1))

    # ---- extras
    def tap(self, name):
        """Intermediate activation of the last forward as float32 numpy (debug/parity; set_option("taps", 1) first)."""
        cnt = ffi.new("int64_t *", 0)
        lib().c3b_get_tap(self._handle, name.encode(), ffi.NULL, cnt)
        n = int(cnt[0])
        if n <= 0:
            raise C3BError(ffi.string(lib().c3b_last_error()).decode())
        out = np.empty(n, dtype=np.float32)
        cnt[0] = n
        check(lib().c3b_get_tap(self._handle, name.encode(), ffi.cast("float *", out.ctypes.data), cnt))
        return out[:int(cnt[0])]

    def weight_blob(self, which=0):
        """(device_ptr, nbytes) of a packed weight image (the broadcast units of clair3_b200.sharding):
        0 = everything the default fp16 tensor-core forward reads (operand images, biases, head weights), 1 = the weights
        only the fp32 debug path (precision=1) reads.  The fp32 path reads both images."""
        p = ffi.new("void **")
        n = ffi.new("size_t *")
        check(lib().c3b_weight_blob(self._handle, int(which), p, n))
        return int(ffi.cast("uintptr_t", p[0])), int(n[0])

    @property
    def launch_count(self):
        return int(lib().c3b_launch_count(self._handle)) if self._handle is not None else 0

    def _release(self):
        if self._handle is not None:
            lib().c3b_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass


class Clair3_P(_C3BModule):
    """Pileup network forward (reference: clair3/model.py:58-161)."""
    _kind = K["C3B_PILEUP"]
    _default_channels = 18      # shared/param_p.py:31-36


class Clair3_F(_C3BModule):
    """Full-alignment network forward (reference: clair3/model.py:282-416)."""
    _kind = K["C3B_FULL_ALIGNMENT"]
    _default_channels = 8       # shared/param_f.py:23-30
