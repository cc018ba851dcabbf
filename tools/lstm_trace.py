"""Per-step SM-cycle breakdown of the two recurrent kernels (lstm1, lstm2) of one pileup forward.

    python tools/lstm_trace.py [--batch 1024] [--lstm-wg 1|2] [--lstm-tile 16|32|64] [--lstm2-split 0|1|2] [--per-step]

Builds a ``Clair3_P`` from the seeded synthetic weights (``clair3_b200.synth``), turns on the debug option ``lstm_trace`` and
runs one device-resident forward after a warm-up forward. Thread 0 of CTA (0, 0) of each LSTM kernel stamps ``clock64`` at four
points of every step (``c3b_debug_lstm_trace``): operands ready, first accumulator ready, cell math of the step done, h_t in
the operand buffer. In LSTM2's split kernel (option ``lstm2_split`` 1: 32 sites per CTA, 2: 48 sites, one operand buffer) that
thread is in warpgroup 0, so the stamps follow block pair 0 of the CTA's sites; with one buffer, ``h_store`` includes the wait
for every warpgroup's chain and copy-out before h_t overwrites h_{t-1}. Printed per layer, as medians over the steps (and per step with ``--per-step``):

    period      operands ready of step s -> operands ready of step s + 1
    first_acc   operands ready -> the first block pair's accumulators are in registers
    epilogue    first accumulators -> the step's last cell math is done
    h_store     last cell math -> h_t stored into the operand buffer

The values are SM clock cycles, so they do not depend on the clock the GPU runs at. Needs an H100.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from clair3_b200 import synth  # noqa: E402
from clair3_b200._ffi import check, ffi, lib  # noqa: E402
from clair3_b200.model import Clair3_P  # noqa: E402

T = 33
FIELDS = ("period", "first_acc", "epilogue", "h_store")


def breakdown(st):
    """st: [33][4] clock64 stamps of one layer -> dict of per-step cycle counts (period has 32 entries)."""
    st = st.astype(np.int64)
    return {"period": st[1:, 0] - st[:-1, 0], "first_acc": st[:, 1] - st[:, 0], "epilogue": st[:, 2] - st[:, 1],
            "h_store": st[:, 3] - st[:, 2], "total": int(st[-1, 3] - st[0, 0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--lstm-wg", type=int, default=0, help="warpgroups per LSTM CTA (0 = library default)")
    ap.add_argument("--lstm-tile", type=int, default=0, help="sites per LSTM1 sub-tile (0 = library choice)")
    ap.add_argument("--lstm2-split", type=int, default=-1, help="LSTM2 split by block pair: 0 | 1 | 2 (-1 = library default)")
    ap.add_argument("--per-step", action="store_true")
    args = ap.parse_args()

    m = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    m.to("cuda")
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=0).items()})
    if args.lstm_wg:
        m.set_option("lstm_wg", args.lstm_wg)
    if args.lstm_tile:
        m.set_option("lstm_tile", args.lstm_tile)
    if args.lstm2_split >= 0:
        m.set_option("lstm2_split", args.lstm2_split)
    m.set_option("lstm_trace", 1)
    x = torch.from_numpy(synth.pileup_inputs(args.batch, seed=0)).cuda()
    m(x)                                   # warm-up: module load, cold L2
    m(x)
    torch.cuda.synchronize()
    buf = np.zeros(2 * T * 4, dtype=np.int64)
    check(lib().c3b_debug_lstm_trace(m._handle, ffi.cast("int64_t *", buf.ctypes.data)))
    stamps = buf.reshape(2, T, 4)

    print("# %s, batch %d, lstm_wg %s, lstm_tile %s, lstm2_split %s: SM cycles (clock64) of thread 0 of CTA (0, 0)"
          % (torch.cuda.get_device_name(), args.batch, args.lstm_wg or "default", args.lstm_tile or "default",
             "default" if args.lstm2_split < 0 else args.lstm2_split))
    for layer in range(2):
        b = breakdown(stamps[layer])
        med = {f: float(np.median(b[f])) for f in FIELDS}
        print("lstm%d: %s, whole recurrence %d" % (layer + 1, ", ".join("%s %.0f" % (f, med[f]) for f in FIELDS), b["total"]))
        if args.per_step:
            print("  step " + " ".join("%9s" % f for f in FIELDS))
            for s in range(T):
                per = ["%9d" % b["period"][s] if s < T - 1 else "%9s" % "-"] + ["%9d" % b[f][s] for f in FIELDS[1:]]
                print("  %4d " % s + " ".join(per))


if __name__ == "__main__":
    main()
