"""The Python bases of the library's region workspaces: ``_Handle`` (the pileup counter, the full-alignment builder and the BAM
reader) and ``_Workspace`` (the counter and the builder: the reference bases of a call, the all_alt_info text stage and the
call path behind it)."""
from __future__ import annotations

import numpy as np
import torch

from ._ffi import C3BError, check, ffi
from .records import DeviceBamRecords


class _Handle:
    """A library workspace on one CUDA device, created by ``<_API>_create`` and released by ``<_API>_destroy``, whose calls run
    on the device's current torch stream (``PileupCounter``, ``FullAlignmentBuilder``, ``bam_decode.BamDecoder``)."""

    _API = None                      # "c3b_plp" / "c3b_fa" / "c3b_bam"

    def __init__(self, device):
        dev = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        if dev.type != "cuda":
            raise C3BError("%s needs a CUDA device (no CPU fallback)" % type(self).__name__)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self._device = dev
        out = ffi.new(self._API + " **")
        check(self._entry("_create")(out, dev.index or 0))
        self._h = out[0]

    def _lib(self):
        """The library as the module that defines the workspace's class binds it, so that every call a workspace makes goes
        through one binding."""
        raise NotImplementedError

    def _entry(self, name):
        """The workspace's entry point ``<_API><name>``."""
        return getattr(self._lib(), self._API + name)

    def _stream(self):
        return ffi.cast("void *", torch.cuda.current_stream(self._device).cuda_stream)

    def _timing(self, fn):
        ms, n = ffi.new("float *"), ffi.new("int *")
        check(fn(self._h, ms, n))
        return float(ms[0]), int(n[0])

    def last_ms(self):
        """(device milliseconds, kernel launches) of the last call, between CUDA events on its stream."""
        return self._timing(self._entry("_last_ms"))

    def close(self):
        if getattr(self, "_h", None) is not None:
            self._entry("_destroy")(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _Workspace(_Handle):
    """What ``PileupCounter`` and ``FullAlignmentBuilder`` share beyond the workspace itself: the reference bases of a call, and
    the all_alt_info text stage with the call path behind it."""

    @staticmethod
    def _reference(ref_seq, rec, who):
        """(pointer, length, object that owns the bytes) of a call's reference bases: str / bytes on the host, or with device
        records a uint8 tensor on their device (default: the one ``to_device`` was given)."""
        if isinstance(rec, DeviceBamRecords):
            if ref_seq is None:
                ref_seq = rec.ref
            if not (isinstance(ref_seq, torch.Tensor) and ref_seq.dtype == torch.uint8 and ref_seq.device == rec.device):
                raise C3BError("%s: device records need the reference bases as a uint8 tensor on the same device" % who)
            ref = ref_seq.contiguous()
            return ffi.cast("const char *", ref.data_ptr()), ref.numel(), ref
        ref = ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq)
        return ffi.cast("const char *", ffi.from_buffer(ref)), len(ref), ref

    # The all_alt_info text stage and the call path behind it, the same for both workspaces.  Each class states what differs:
    # _text_max_indel (whether a text stage can follow the last call, and its default max_indel_length), _text_queued (what a
    # queued text stage makes stale), _n_cand (the candidate count without a wait beyond the one ``sizes()`` makes), _network
    # (the network its candidates go through), _queue_forward (how that network is queued) and _call_fields (what ``call``
    # returns beside the decoder's results).
    _OWNER = None                    # "counter" / "builder", in the errors

    def alt_text(self, max_indel_length=None):
        """Enqueues the text stage (``<_API>_alt_text``) behind the last count / build, on its stream and without a host wait:
        the ``all_alt_info`` string of every candidate and what the decoder takes of it, formatted on the device.
        ``max_indel_length``: as the reference's (default: what the count / build was given).  Device-resident records must stay
        alive until the text has been fetched."""
        default = self._text_max_indel()
        if max_indel_length is None:
            max_indel_length = default
        if isinstance(max_indel_length, bool) or not isinstance(max_indel_length, (int, np.integer)):
            raise C3BError("alt_text: max_indel_length must be an integer, got %r" % (max_indel_length,))
        check(self._entry("_alt_text")(self._h, int(max_indel_length)))
        self._text_queued()
        return self

    def _text_queued(self):
        pass

    def alt_text_sizes(self):
        """(bytes of all text strings, bytes of all decoder strings) of the last ``alt_text``."""
        a, b = ffi.new("int64_t *"), ffi.new("int64_t *")
        check(self._entry("_alt_text_sizes")(self._h, a, b))
        return int(a[0]), int(b[0])

    def alt_text_fetch(self):
        """dict: ``text`` (the ``all_alt_info`` strings, one per candidate), ``decoder`` (the ``"depth-alt"`` strings the
        reference passes on with each candidate), ``ref_base`` uint8 [n_cand], ``position`` int64 [n_cand] (1-based).  Waits for
        the text stage."""
        nk = self._n_cand()
        nt, nd = self.alt_text_sizes()
        text, dec = np.zeros(max(nt, 1), np.uint8), np.zeros(max(nd, 1), np.uint8)
        toff, doff = np.zeros(nk + 1, np.int64), np.zeros(nk + 1, np.int64)
        rb, pos = np.zeros(nk, np.uint8), np.zeros(nk, np.int64)
        c = ffi.cast
        check(self._entry("_fetch_alt_text")(self._h, c("char *", text.ctypes.data), c("int64_t *", toff.ctypes.data),
                                             c("char *", dec.ctypes.data), c("int64_t *", doff.ctypes.data),
                                             c("uint8_t *", rb.ctypes.data), c("int64_t *", pos.ctypes.data)))
        tb, db = text.tobytes(), dec.tobytes()
        return {"text": [tb[toff[j]:toff[j + 1]].decode("latin-1") for j in range(nk)],
                "decoder": [db[doff[j]:doff[j + 1]].decode("latin-1") for j in range(nk)], "ref_base": rb, "position": pos}

    def alt_text_device(self):
        """The text stage's results as tensors that alias the workspace (valid until the next count / build / ``alt_text``):
        ``text`` uint8 [n_text_bytes], ``text_off`` int64 [n_cand + 1], ``decoder`` uint8 [n_decoder_bytes], ``decoder_off``
        int64 [n_cand + 1], ``ref_base`` uint8 [n_cand], ``position`` int64 [n_cand]; ``decoder`` / ``decoder_off`` /
        ``ref_base`` are ``decode_calls``' ``alt_bytes`` / ``alt_offsets`` / ``ref_base``.  Waits (``sizes()``) only when
        nothing has waited since the last count / build / ``alt_text``; after that wait it touches the stream no more."""
        nk = self._n_cand()
        nt, nd = self.alt_text_sizes()
        p = [ffi.new("const char **"), ffi.new("const int64_t **"), ffi.new("const char **"), ffi.new("const int64_t **"),
             ffi.new("const uint8_t **"), ffi.new("const int64_t **")]
        check(self._entry("_alt_text_device")(self._h, *p))
        shapes = (("text", nt, torch.uint8), ("text_off", nk + 1, torch.int64), ("decoder", nd, torch.uint8),
                  ("decoder_off", nk + 1, torch.int64), ("ref_base", nk, torch.uint8), ("position", nk, torch.int64))
        return {name: _device_view(int(ffi.cast("uintptr_t", q[0])), n, dt, self._device) for (name, n, dt), q in zip(shapes, p)}

    def alt_text_last_ms(self):
        """Device time and kernel launches of the last ``alt_text`` (``last_ms`` reports the count / build alone)."""
        return self._timing(self._entry("_alt_text_last_ms"))

    def call(self, model, output_config, ctg_name, k=16):
        """The candidates of the last count / build from records to call records on the current stream: the text stage, the
        network over every candidate and ``model.decode_calls`` on the device views, with one host wait (the sizes) before the
        network is queued.  Returns ``decode.batch_calls``' dict (``chromosome``, ``position``, ``calls``, ``text``, ``ad``,
        ``start``; ``decode.calls_text`` formats it) plus ``Y``, the probabilities, on the device, and for the counter
        ``cand_ok`` uint8 [n_cand].  Every candidate is decoded, as the reference decodes every full-alignment candidate;
        ``cand_ok == 0``: the reference drops that pileup candidate, ignore its row.  ``device`` holds the same results where
        they are on the device, for stream-ordered work that follows (``cascade.select_device``): ``calls``, ``text``,
        ``decoder_off``, ``position`` and for the counter ``cand_ok``; ``decoder_off``, ``position`` and ``cand_ok`` alias the
        workspace and are valid until its next count / build / ``alt_text``.  Raises what ``batch_calls`` raises on an
        alt_info string the decoder rejects."""
        from . import decode
        decode._check_config(output_config)
        self._check_model(model, "call")
        if bool(output_config.add_indel_length) != model.add_indel_length:
            raise C3BError("call: output_config.add_indel_length must match the model")
        self.alt_text()
        self.sizes()                                       # the one wait: the count / build and the text together
        v = self.alt_text_device()
        nk = self._n_cand()
        y = torch.empty((nk, model.out_dim), dtype=torch.float32, device=self._device)
        self._forward_into(model, y)
        out = model.decode_calls(y, v["ref_base"], v["decoder"], v["decoder_off"], output_config, k=k)
        fields = self._call_fields()
        res = decode.calls_result(decode._numpy(out), [ctg_name] * nk, v["position"].cpu().numpy(), v["decoder_off"].cpu().numpy())
        res.update(fields, Y=y)
        res.setdefault("device", {}).update(calls=out["calls"], text=out["text"], decoder_off=v["decoder_off"],
                                            position=v["position"])
        return res

    def _call_fields(self):
        return {}

    def _check_model(self, model, who):
        if getattr(model, "_handle", None) is None:
            raise C3BError("%s: the model has no device / weights yet (.to(device), .load_state_dict())" % who)
        kind, channels, name = self._network()
        if getattr(model, "input_channels", channels) != channels or model._kind != kind:
            raise C3BError("%s: needs %s" % (who, name))
        if torch.device(model._device) != self._device:
            raise C3BError("%s: the model lives on %s, the %s on %s" % (who, model._device, self._OWNER, self._device))

    def _forward_into(self, model, y):
        """The network over every candidate into y, stream-ordered."""
        if len(y):
            self._queue_forward(model, y)


class _DeviceArray:
    def __init__(self, ptr, n, dtype):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": {torch.uint8: "|u1", torch.int64: "<i8"}[dtype],
                                         "data": (ptr, False), "version": 2}


def _device_view(ptr, n, dtype, device):
    """A tensor over n elements of workspace memory at ptr (no copy; the workspace owns the memory)."""
    if n == 0:
        return torch.empty(0, dtype=dtype, device=device)
    return torch.as_tensor(_DeviceArray(ptr, n, dtype), device=device)
