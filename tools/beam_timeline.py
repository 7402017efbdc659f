"""In-kernel clock64 timeline of the fused forward scan + beam search (chunk 0, blocks 100..107) through the decode test hook.
state_len 4 or 5 only: the state_len 3 decode (one warp per chunk) carries no timeline.
usage: python tools/beam_timeline.py [state_len] [N]"""
import os, sys, numpy as np
os.environ["B200_DEBUG_BEAM_TIMELINE"] = "1"
sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
from conftest import synthetic_scores
from dorado_b200 import lib as L
sl = int(sys.argv[1]) if len(sys.argv) > 1 else 4
if sl not in (4, 5):
    sys.exit("beam_timeline: state_len must be 4 or 5 (the state_len 3 decode has no timeline)")
N = int(sys.argv[2]) if len(sys.argv) > 2 else 512
scores = synthetic_scores(N, 1666, sl, seed=1, scale=1.9)
L.decode_scores(scores, clamp_val=5.0)
