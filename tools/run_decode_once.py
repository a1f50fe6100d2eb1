#!/usr/bin/env python
"""Tiny driver for ncu captures: build the decoder for a workload and run a few positions.

The persistent engine decodes `--start` positions in launch #1 (unprofiled context build-up) and
`--steps` positions in launch #2; capture the SECOND launch, it is short and sits at the context
length you asked for (ncu replays a kernel ~40 times, so keep --steps small):

    ncu --set full --clock-control none --import-source on -k regex:decode_megakernel \
        --launch-skip 1 -c 1 -o mega python tools/run_decode_once.py --steps 8 --start 504

(without --launch-skip the capture is launch #1: --start tokens, bytes per token = total / start.)
"""
import argparse
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="tinyllama-1.1b")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--start", type=int, default=0, help="positions decoded (unprofiled) before the profiled launch")
    a = ap.parse_args()
    import torch
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    shape = SHAPES[a.workload]
    dec = Decoder(shape, synth_weights(shape, "cuda", 1235))
    print("engine", dec.engine)
    tok = 1
    if a.start:
        ids = dec.generate(1, 0, a.start)
        tok = ids[-1]
    torch.cuda.synchronize()
    ids = dec.generate(tok, a.start, a.steps)
    print(ids)


if __name__ == "__main__":
    main()
