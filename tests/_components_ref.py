"""CPU oracle of small-component removal (nm_mesh_components, DESIGN 4.9).

Components: the connected components of the vertex graph whose edges are the face edges (scipy.sparse.csgraph); a
component's id is its smallest vertex index, its size its number of faces (np.bincount over the faces' labels).  The filter
keeps the vertices and faces of components with >= m faces, both in their original order, faces re-indexed."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def labels_and_sizes(V, faces):
    """(labels (V,) int64: the smallest vertex index of each vertex's component, sizes (V,) int64: faces per label)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if V == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    rows = np.concatenate([f[:, 0], f[:, 0]])
    cols = np.concatenate([f[:, 1], f[:, 2]])
    g = coo_matrix((np.ones(rows.size, np.int32), (rows, cols)), shape=(V, V))
    n, lab = connected_components(g, directed=False)
    first = np.full(n, V, np.int64)
    np.minimum.at(first, lab, np.arange(V))
    labels = first[lab]
    sizes = np.bincount(labels[f[:, 0]], minlength=V).astype(np.int64)
    return labels, sizes


def remove_small_components(verts, normals, faces, m):
    """(verts, normals, faces int32, counts, labels int32) like Engine.mesh_components; counts = (kept vertices, kept faces,
    components with >= 1 face, kept components)."""
    v, n = np.asarray(verts, np.float32).reshape(-1, 3), np.asarray(normals, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    labels, sizes = labels_and_sizes(len(v), f)
    vkeep = sizes[labels] >= m
    fkeep = vkeep[f[:, 0]] if len(f) else np.zeros(0, bool)
    new = np.cumsum(vkeep) - 1
    roots = labels == np.arange(len(v))
    counts = (int(vkeep.sum()), int(fkeep.sum()), int((roots & (sizes > 0)).sum()), int((roots & (sizes > 0) & (sizes >= m)).sum()))
    return v[vkeep], n[vkeep], new[f[fkeep]].astype(np.int32).reshape(-1, 3), counts, labels.astype(np.int32)


def bfs_labels(V, faces):
    """Plain breadth-first search over an adjacency list: the yard-stick of labels_and_sizes."""
    adj = [[] for _ in range(V)]
    for a, b, c in np.asarray(faces, np.int64).reshape(-1, 3).tolist():
        for x, y in ((a, b), (b, c), (a, c)):
            adj[x].append(y)
            adj[y].append(x)
    labels = [-1] * V
    for s in range(V):                       # in index order: the first vertex reached is the component's smallest
        if labels[s] >= 0:
            continue
        labels[s] = s
        queue = [s]
        while queue:
            x = queue.pop()
            for y in adj[x]:
                if labels[y] < 0:
                    labels[y] = s
                    queue.append(y)
    return np.asarray(labels, np.int64)
