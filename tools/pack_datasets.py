#!/usr/bin/env python
"""Pack the reference's shipped Monte-Carlo runs into compact .npz files for the dataset replay (tools/replay_datasets.py).

    python tools/pack_datasets.py            (needs the rpng/cpi checkout, CPI_REFERENCE, by default /root/reference; writes tests/golden/_datasets/replay_<rate>.npz)

Only what the preintegration path consumes is kept: per run the IMU stream of imu_data_meas.dat ("wx wy wz ax ay az <unused> t_ms",
sim/SimParser.h:148-175) and the camera stamps of camera_data_meas.dat (last column, ms).  The output directory is git-ignored
(it is ~100 MB of the reference's data, not source of this repository)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("CPI_REFERENCE", "/root/reference") + "/cpi_simulation"
OUT = os.path.join(ROOT, "tests", "golden", "_datasets")


def main():
    os.makedirs(OUT, exist_ok=True)
    for rate in (100, 200, 400):
        d = {}
        runs = sorted(x for x in os.listdir(f"{REF}/GAZEBO_FREQ_{rate}") if x.startswith("rawdata_"))
        for r in runs:
            base = f"{REF}/GAZEBO_FREQ_{rate}/{r}"
            imu = np.loadtxt(f"{base}/imu_data_meas.dat")
            cam = np.array([float(l.split()[-1]) for l in open(f"{base}/camera_data_meas.dat") if l.strip()])
            d[f"{r}/imu"] = np.concatenate([imu[:, 0:6], 1e-3 * imu[:, 7:8]], axis=1)      # [w(3) a(3) t_seconds]
            d[f"{r}/cam"] = 1e-3 * cam
        np.savez_compressed(os.path.join(OUT, f"replay_{rate}.npz"), **d)
        print(rate, len(runs), "runs", os.path.getsize(os.path.join(OUT, f"replay_{rate}.npz")) >> 20, "MiB")


if __name__ == "__main__":
    sys.exit(main())
