"""lio_pcd_write_xyzi: the binary PCD v0.7 that pcl::PCDWriter::writeBinary writes for pcl::PointXYZI (src/save_bag_to_pcd.cc:156-160),
on host arrays and without a device."""
import numpy as np
import pytest

from lio_mapping_b200 import _lib, write_pcd

HEADER = (b"# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\n"
          b"COUNT 1 1 1 1\nWIDTH %d\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS %d\nDATA binary\n")


@pytest.mark.parametrize("n", [0, 1, 1000])
def test_header_bytes_and_records(tmp_path, n):
    rng = np.random.default_rng(n)
    pts = rng.normal(0, 30, (n, 4)).astype(np.float32)
    if n:
        pts[0] = [np.nan, np.inf, -0.0, 1e-40]   # every bit pattern goes through
    path = tmp_path / "cloud.pcd"
    write_pcd(path, pts)
    data = path.read_bytes()
    head = HEADER % (n, n)
    assert data[:len(head)] == head
    assert len(data) == len(head) + 16 * n
    assert np.array_equal(np.frombuffer(data[len(head):], "<u4").reshape(-1, 4), pts.view(np.uint32))


def test_unwritable_path(tmp_path):
    L = _lib.lib()
    pts = np.zeros((1, 4), np.float32)
    assert L.lio_pcd_write_xyzi(str(tmp_path / "missing" / "cloud.pcd").encode(), pts, 1) == -2   # LIO_ERR_INVALID
    assert b"No such file" in L.lio_last_error()
    assert L.lio_pcd_write_xyzi(str(tmp_path).encode(), pts, 1) == -2                             # a directory
    assert L.lio_pcd_write_xyzi(None, pts, 1) == -2 and L.lio_pcd_write_xyzi(b"x.pcd", pts, -1) == -2
    with pytest.raises(_lib.LioError):
        write_pcd(tmp_path / "missing" / "cloud.pcd", pts)
