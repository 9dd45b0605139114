"""The caller's side of the mesh's change feed (immesh_mesh_changes) for the tests: a mirror that starts from snapshot() and is fed only
the rows, checking every row against what it holds (a removal of a live triangle, an addition of a dead one, a flip row that changes
the flip) and the order of the rows inside a frame."""
import numpy as np


def code_of(exc):
    return int(str(exc.value).split("code ")[1].split(":")[0])


class Mirror:
    """the caller's copy of the mesh: snapshot() at the start, then only the rows"""

    def __init__(self, mesh):
        mesh.wait()
        v, t, f = mesh.snapshot()
        self.v = v.copy()
        self.tri = {tuple(r): int(x) for r, x in zip(t.tolist(), f.tolist())}
        self.newest = mesh.changes_newest()
        self.codes = np.zeros(6, np.int64)
        self.rows = {}   # frame -> its rows

    def apply(self, ch):
        fr, rows = ch["frames"], ch["rows"]
        if len(fr):
            assert fr[0, 1] == len(self.v), "the first frame's vertices do not follow the mirror's"
            assert np.all(fr[1:, 1] == fr[:-1, 2]), "vertex ranges are not contiguous"
            assert len(ch["vertices"]) == fr[-1, 2] - fr[0, 1]
            self.v = np.concatenate([self.v, ch["vertices"]])
        r0 = 0
        for f, _, _, r1 in fr.tolist():
            seg = rows[r0:r1]
            if len(seg) > 1:   # ascending, distinct triples inside a frame
                k = seg[:, 0].astype(np.int64) << 42 | seg[:, 1].astype(np.int64) << 21 | seg[:, 2].astype(np.int64)
                assert np.all(np.diff(k) > 0), f"frame {f}: rows not in ascending triple order"
            self.rows[f] = seg.copy()
            for a, b, c, code in seg.tolist():
                key = (a, b, c)
                self.codes[code] += 1
                if code == 0:
                    assert key in self.tri, f"frame {f}: removal of a triangle the mirror does not hold {key}"
                    del self.tri[key]
                elif code in (2, 3):
                    assert key not in self.tri, f"frame {f}: addition of a live triangle {key}"
                    self.tri[key] = code & 1
                elif code in (4, 5):
                    assert self.tri.get(key, -1) == 1 - (code & 1), f"frame {f}: flip row of {key} changes nothing"
                    self.tri[key] = code & 1
                else:
                    raise AssertionError(f"frame {f}: row code {code}")
            r0 = r1
        assert r0 == len(rows)
        self.newest = ch["newest"]

    def sync(self, mesh):
        self.apply(mesh.changes(self.newest))

    def check(self, mesh, what=""):
        mesh.wait()
        self.check_state(*mesh.snapshot(), what)

    def check_state(self, v, t, f, what=""):
        assert v.shape == self.v.shape and np.array_equal(v.view(np.uint32), self.v.view(np.uint32)), f"{what}: vertices"
        keys = sorted(self.tri)
        assert t.shape == (len(keys), 3) and np.array_equal(t, np.array(keys, np.int32).reshape(-1, 3)), f"{what}: triangle set"
        assert np.array_equal(f, np.array([self.tri[k] for k in keys], np.int32)), f"{what}: flips"
