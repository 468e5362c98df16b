"""An independent NumPy restatement of a binary_little_endian PLY file of columns (tinyply 2.x's layout, as the
reference writes it through WriteCollectionToPLY): the header text, then per element a packed structured array.
TEST INFRASTRUCTURE."""
import numpy as np

TYPE = {1: ("char", "<i1"), 2: ("uchar", "<u1"), 3: ("short", "<i2"), 4: ("ushort", "<u2"), 5: ("int", "<i4"),
        6: ("uint", "<u4"), 7: ("float", "<f4"), 8: ("double", "<f8")}


def convert(values, ply_dtype):
    """static_cast<ply type> of every value; float -> integer truncates and saturates, NaN -> 0"""
    a = np.asarray(values)
    dt = np.dtype(TYPE[ply_dtype][1])
    if a.dtype.kind == "f" and dt.kind in "iu":
        info = np.iinfo(dt)
        x = a.astype(np.float64)
        t = np.clip(np.trunc(np.nan_to_num(x, nan=0.0, posinf=info.max, neginf=info.min)), info.min, info.max)
        return t.astype(np.int64).astype(dt)
    return a.astype(dt)


def header(elements):
    """elements: [(name, count, [(property, ply_dtype), ...]), ...]"""
    h = "ply\nformat binary_little_endian 1.0\n"
    for name, count, props in elements:
        h += "element %s %d\n" % (name, count)
        h += "".join("property %s %s\n" % (TYPE[t][0], p) for p, t in props)
    return (h + "end_header\n").encode()


def ply_file(columns, num_items):
    """columns: [(element, name, ply_dtype code, values)] with values broadcast to num_items; bytes"""
    order = []
    for elem, _, _, _ in columns:
        if elem not in order:
            order.append(elem)
    elements, body = [], b""
    for elem in order:
        cols = [c for c in columns if c[0] == elem]
        rec = np.zeros(num_items, dtype=np.dtype([("f%d" % i, TYPE[c[2]][1]) for i, c in enumerate(cols)]))
        for i, c in enumerate(cols):
            rec["f%d" % i] = convert(np.broadcast_to(np.asarray(c[3]), (num_items,)), c[2])
        elements.append((elem, num_items, [(c[1], c[2]) for c in cols]))
        body += rec.tobytes()
    return header(elements) + body
