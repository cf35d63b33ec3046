"""Per-level, per-phase profile of wl_fused2 from its globaltimer stamps: median and max over CTAs, in us.

    python tools/prof_wl_phases.py [n_graphs]      (default 10 000 = bench.py config 2; 28 284 = several tiles per CTA)

The verification instance follows GRAKEL_B200_WL_PAYLOAD as in the library.  Phases of a level >= 1 (stamp indices of
wl_fused2.cuh in brackets): [A] signatures (0 -> 10), [A] insert + row copy-out (10 -> 1), barrier wait (1 -> 2),
[B] representative + verification (2 -> 4), label write-back (4 -> 5), feature count/emit (5 -> 3), table clear +
partials flush (3 -> 6).  The stamps inside a tile loop keep the last tile's value, so with several tiles per CTA
'signatures' also holds the earlier tiles' [A] and 'verify' their [B] + emit; the [A], wait and [B]+emit totals
(0 -> 1, 1 -> 2, 2 -> 3) are exact on every route.
"""
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from bench import H, pack_workload  # noqa: E402
from grakel_b200 import _lib  # noqa: E402

PHASES = [("signatures", 0, 10), ("insert", 10, 1), ("barrier wait", 1, 2), ("verify", 2, 4), ("write-back", 4, 5),
          ("count/emit", 5, 3), ("clear+flush", 3, 6), ("[A]", 0, 1), ("[B]+emit", 2, 3), ("level", 0, 6)]
PHASES0 = [("stage+emit", 0, 2), ("clear", 2, 3), ("flush", 3, 6), ("level", 0, 6)]


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
    eng = _lib.get_engine()
    eng.pack(*pack_workload(n))
    ms = []
    for _ in range(8):
        ms.append(eng.wl_features(H).ms_features)
    st = eng.wl_features(H)
    fd, path = tempfile.mkstemp(suffix=".bin")
    os.close(fd)
    os.environ["GRAKEL_B200_PROF"] = "1"
    os.environ["GRAKEL_B200_PROF_OUT"] = path
    try:
        eng.wl_features(H)
        raw = np.fromfile(path, dtype=np.int64)
    finally:
        del os.environ["GRAKEL_B200_PROF"], os.environ["GRAKEL_B200_PROF_OUT"]
        os.unlink(path)
    L = H + 1
    q = raw.reshape(-1, L, 16).astype(np.float64) / 1e3  # [CTA][level][stamp], us
    print(f"graphs {n}  CTAs {q.shape[0]}  payload {os.environ.get('GRAKEL_B200_WL_PAYLOAD', '1')}  "
          f"ms_features (unprofiled, median of 8) {np.median(ms[2:]):.4f}  level dims {[st.level_dims[i] for i in range(L)]}")
    print("median over CTAs (max), us")
    for lv in range(L):
        ph = PHASES0 if lv == 0 else PHASES
        cells = []
        for name, a, b in ph:
            d = q[:, lv, b] - q[:, lv, a]
            cells.append(f"{name} {np.median(d):.1f} ({d.max():.1f})")
        print(f"  level {lv}: " + " | ".join(cells))
    span = q[:, L - 1, 6].max() - q[:, 0, 0].min()
    print(f"  kernel span (first stamp to last): {span:.1f} us")


if __name__ == "__main__":
    main()
