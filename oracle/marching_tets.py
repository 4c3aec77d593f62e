"""Torch restatement of marching tetrahedra (kaolin/ops/conversions/tetmesh.py:57-168) and
subdivide_tetmesh (kaolin/ops/mesh/tetmesh.py:85-181) for any batch, in float32 or float64, with
autograd to the vertices, the sdf and the features.

  edges     the tets' corner pairs 01, 02, 03, 12, 13, 23, sorted, made unique in lexicographic order
            (E of them, self-loops of degenerate tets included); tet_edge (T, 6) their ids
  occ       sdf > 0
  vertices  per view, the edges with occ(a) != occ(b), in edge order, at
            (x_a (-s_b) + x_b s_a) / (s_a + (-s_b))
  faces     case c = sum_k occ(corner k) 2^k; the faces of one-triangle tets in tet order, then both
            faces of each two-triangle tet in tet order; each face's vertices are the edges of the
            case's corner pairs
  subdivide edge e becomes vertex V + e at the mean of its ends (positions and features); the eight
            children of each tet, block by block
The case table is not restated here: ``case_table`` reads it off the reference's own outputs for one
tetrahedron in corner order 0123 under all 16 sign patterns (tests/golden/marching_tets.npz).
Structures are built with numpy; the arithmetic is torch, in the dtype of the vertices.
``marching_on_device`` gives the same results with the reference's per-view structure kept on the
device (torch ops only, ``unique`` over the valid tets' edges): the benchmark times it as the baseline.
"""
import numpy as np
import torch

PAIRS = np.array([[0, 1], [0, 2], [0, 3], [1, 2], [1, 3], [2, 3]])
# children of a tet over (v0, v1, v2, v3, m01, m02, m03, m12, m13, m23), in the reference's block order
CHILDREN = np.array([[0, 4, 5, 6], [1, 7, 4, 8], [2, 5, 7, 9], [3, 6, 9, 8],
                     [4, 5, 6, 8], [4, 5, 8, 7], [9, 5, 8, 6], [9, 5, 7, 8]])


def topology(num_vertices, tets):
    """-> (edges (E, 2) int64, tet_edge (T, 6) int64)."""
    tets = np.asarray(tets, np.int64).reshape(-1, 4)
    V = int(num_vertices)
    if len(tets) and (tets.min() < 0 or tets.max() >= V):
        raise IndexError("tet index outside [0, V)")
    pe = np.sort(tets[:, PAIRS], -1).reshape(-1, 2)
    key = pe[:, 0] * max(V, 1) + pe[:, 1]
    uniq, inverse = np.unique(key, return_inverse=True)
    edges = np.stack([uniq // max(V, 1), uniq % max(V, 1)], 1).astype(np.int64)
    return edges, inverse.reshape(-1, 6).astype(np.int64)


def case_table(single_faces, single_nf):
    """The (16, 2, 3) edge slots (0..5 for pairs 01 .. 23; -1 unused) of each case, from the faces the
    reference gives for one tet with corners 0123 under the 16 patterns (view c: pattern c)."""
    table = -np.ones((16, 2, 3), np.int64)
    start = 0
    for c in range(16):
        occ = [(c >> k) & 1 for k in range(4)]
        sign = [s for s, (a, b) in enumerate(PAIRS) if occ[a] != occ[b]]     # vertex id -> slot
        f = np.asarray(single_faces[start:start + single_nf[c]])
        start += single_nf[c]
        for k, tri in enumerate(f):
            table[c, k] = [sign[v] for v in tri]
    return table


def marching(vertices, tets, sdf, table, topo=None):
    """-> per view: (vertices (nv, 3), faces (nf, 3) int64, tet_idx (nf,) int64), for vertices (B, V, 3)
    and sdf (B, V) of any dtype.  ``topo``: ``topology(V, tets)``, if already built."""
    tets = np.asarray(tets, np.int64).reshape(-1, 4)
    edges, tet_edge = topology(vertices.shape[1], tets) if topo is None else topo
    ntri = np.array([0 if n in (0, 4) else 2 if n == 2 else 1 for n in (bin(c).count("1") for c in range(16))])
    dev = vertices.device
    out = []
    for b in range(vertices.shape[0]):
        s = sdf[b]
        occ = (s > 0).cpu().numpy()
        sel = np.nonzero(occ[edges[:, 0]] != occ[edges[:, 1]])[0]
        vid = -np.ones(len(edges), np.int64)
        vid[sel] = np.arange(len(sel))
        ia, ib = (torch.from_numpy(edges[sel, k]).to(dev) for k in (0, 1))
        sa, nb = s[ia][:, None], -s[ib][:, None]
        verts = (vertices[b, ia] * nb + vertices[b, ib] * sa) / (sa + nb)
        case = (occ[tets] * (1 << np.arange(4))).sum(1) if len(tets) else np.zeros(0, np.int64)
        ones, twos = np.nonzero(ntri[case] == 1)[0], np.nonzero(ntri[case] == 2)[0]
        f1 = vid[tet_edge[ones[:, None], table[case[ones], 0]]]
        f2 = vid[tet_edge[twos[:, None, None], table[case[twos]]]].reshape(-1, 3)
        faces = np.concatenate([f1.reshape(-1, 3), f2])
        assert (faces >= 0).all()
        tet_idx = np.concatenate([ones, np.repeat(twos, 2)])
        out.append((verts, torch.from_numpy(faces), torch.from_numpy(tet_idx)))
    return out


def marching_on_device(vertices, tets, sdf, table):
    """The reference's per-view structure with every step a torch op on the inputs' device: the corner
    occupancies, the valid-tet mask, ``torch.unique(dim=0)`` over the valid tets' sorted edges, the
    sign-change mask over the unique edges, and the boolean gathers of the one- and two-triangle tets.
    Same results as ``marching``; used as the timing baseline of the reference's structure."""
    dev = vertices.device
    tets = torch.as_tensor(tets, device=dev).reshape(-1, 4)
    slots = torch.as_tensor(table, device=dev)
    ntri = torch.tensor([0 if n in (0, 4) else 2 if n == 2 else 1 for n in (bin(c).count("1") for c in range(16))],
                        device=dev)
    pairs = torch.as_tensor(PAIRS, device=dev)
    bits = 1 << torch.arange(4, device=dev)
    out = []
    for b in range(vertices.shape[0]):
        s = sdf[b]
        occ = s > 0
        corner = occ[tets]
        inside = corner.sum(1)
        valid = (inside > 0) & (inside < 4)
        edges = tets[valid][:, pairs].reshape(-1, 2).sort(1).values
        uniq, inverse = torch.unique(edges, dim=0, return_inverse=True)
        crossing = occ[uniq[:, 0]] != occ[uniq[:, 1]]
        vid = torch.full((len(uniq),), -1, dtype=torch.int64, device=dev)
        vid[crossing] = torch.arange(int(crossing.sum()), device=dev)
        ends = uniq[crossing]
        sa, nb = s[ends[:, 0]][:, None], -s[ends[:, 1]][:, None]
        verts = (vertices[b, ends[:, 0]] * nb + vertices[b, ends[:, 1]] * sa) / (sa + nb)
        tet_vid = vid[inverse].reshape(-1, 6)
        case = (corner[valid] * bits).sum(1)
        n = ntri[case]
        one, two = n == 1, n == 2
        f1 = tet_vid[one].gather(1, slots[case[one], 0])
        f2 = tet_vid[two].gather(1, slots[case[two]].reshape(-1, 6)).reshape(-1, 3)
        idx = torch.arange(len(tets), device=dev)[valid]
        out.append((verts, torch.cat([f1, f2]), torch.cat([idx[one], idx[two].repeat_interleave(2)])))
    return out


def subdivide(vertices, tets, features=None):
    """subdivide_tetmesh for vertices (B, V, 3) and features (B, V, D) or None of any dtype ->
    (vertices (B, V + E, 3), tets (8T, 4) int64, features (B, V + E, D) or None)."""
    tets = np.asarray(tets, np.int64).reshape(-1, 4)
    V = vertices.shape[1]
    edges, tet_edge = topology(V, tets)
    pf = vertices if features is None else torch.cat([vertices, features], -1)
    ia, ib = (torch.from_numpy(edges[:, k]).to(vertices.device) for k in (0, 1))
    new = torch.cat([pf, (pf[:, ia] + pf[:, ib]) / 2], 1)
    table = np.concatenate([tets, V + tet_edge], 1)
    new_tets = np.concatenate([table[:, c] for c in CHILDREN]) if len(tets) else np.zeros((0, 4), np.int64)
    return new[..., :3], torch.from_numpy(np.ascontiguousarray(new_tets)), None if features is None else new[..., 3:]
