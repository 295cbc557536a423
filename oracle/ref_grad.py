"""The gradient-branch outputs of the UNMODIFIED reference `get_mesh_udf_fast` under oracle/ref_post.py -- test
infrastructure.

`run_grad` is `ref_post.run_post` (the runner's two calls of get_mesh_udf_fast under the trimesh stub, then its last
Trimesh(...)) with the staged function wrapped so that the tuple of the call that returned is kept.  It adds to run_post's
dict the gradient branch's `new_verts` (fp32 NumPy [V,3], out[0]) and `next_indices` (int64 [7V], out[4]), and `mesh`:
the vertices and faces of the returned mesh (out[2]), the mesh that branch saw.  ref_post itself is not modified.
"""
import numpy as np

from oracle import ref_post


def run_grad(*args, **kwargs):
    """ref_post.run_post(*args, **kwargs) plus `new_verts`, `next_indices` and `mesh` of the call that returned"""
    returned = []
    load = ref_post.load_extract_mesh

    def load_recording():
        em = load()
        gmuf = em.get_mesh_udf_fast

        def recording(*a, **k):
            out = gmuf(*a, **k)
            returned.append(out)
            return out

        em.get_mesh_udf_fast = recording
        return em

    ref_post.load_extract_mesh = load_recording
    try:
        r = ref_post.run_post(*args, **kwargs)
    finally:
        ref_post.load_extract_mesh = load
    out = returned[-1]
    r.update(new_verts=out[0].detach().cpu().numpy(), next_indices=np.asarray(out[4]),
             mesh=(np.asarray(out[2].vertices), np.asarray(out[2].faces)))
    return r
