"""Binary PCD v0.7 files of the 48-byte pcl::PointXYZINormal records (liinit_cloud_download, capi.LiInitGpu.cloud): what the node's
pcd_save writes with pcl::PCDWriter::writeBinary (laserMapping.cpp:183-187, 594-613). And the map-sharpness cloud of the assessment
(liinit_assess_cloud, capi.LiInitGpu.assess_cloud): 8 float fields per record (write_assess).

The header lists the fields sorted by offset, with the padding bytes as `_` fields, so that the binary body is the records as they
are. The padding floats are written as they come (0 in the library's records).
"""
from __future__ import annotations

import numpy as np

HEADER = ("# .PCD v0.7 - Point Cloud Data file format\n"
          "VERSION 0.7\n"
          "FIELDS x y z _ normal_x normal_y normal_z _ intensity curvature _\n"
          "SIZE 4 4 4 1 4 4 4 1 4 4 1\n"
          "TYPE F F F U F F F U F F U\n"
          "COUNT 1 1 1 4 1 1 1 4 1 1 8\n"
          "WIDTH {n}\n"
          "HEIGHT 1\n"
          "VIEWPOINT 0 0 0 1 0 0 0\n"
          "POINTS {n}\n"
          "DATA binary\n")


def write_binary(path: str, rec12) -> int:
    """Writes [n, 12] float32 records as a binary PCD file; returns the number of points."""
    a = np.ascontiguousarray(rec12, dtype="<f4").reshape(-1, 12)
    with open(path, "wb") as f:
        f.write(HEADER.format(n=len(a)).encode("ascii"))
        f.write(a.tobytes())
    return len(a)


ASSESS_FIELDS = ("x", "y", "z", "entropy", "plane_variance", "neighbors", "points", "valid")
ASSESS_HEADER = ("# .PCD v0.7 - Point Cloud Data file format\n"
                 "VERSION 0.7\n"
                 "FIELDS " + " ".join(ASSESS_FIELDS) + "\n"
                 "SIZE 4 4 4 4 4 4 4 4\n"
                 "TYPE F F F F F F F F\n"
                 "COUNT 1 1 1 1 1 1 1 1\n"
                 "WIDTH {n}\n"
                 "HEIGHT 1\n"
                 "VIEWPOINT 0 0 0 1 0 0 0\n"
                 "POINTS {n}\n"
                 "DATA binary\n")


def write_assess(path: str, rec8) -> int:
    """Writes [n, 8] float32 assessment records (x y z entropy plane_variance neighbors points valid) as a binary PCD file; returns
    the number of records. A viewer colours the cloud by any field, e.g. entropy."""
    a = np.ascontiguousarray(rec8, dtype="<f4").reshape(-1, 8)
    with open(path, "wb") as f:
        f.write(ASSESS_HEADER.format(n=len(a)).encode("ascii"))
        f.write(a.tobytes())
    return len(a)
