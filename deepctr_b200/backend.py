"""The part of ``tf.keras.backend`` the reference's builders call inside their ``Lambda`` layers (ONN's
``K.sum(element_wise_prod, axis=-1)``, deepctr/models/onn.py:95-96).  A builder imported as a drop-in reaches it
as ``tensorflow.keras.backend``.  Each function works on a runtime Var (on the package's kernels, through ``ops``)
and on the shape probe ``Lambda`` uses to learn its output shape while the graph is built."""
from . import engine as E
from . import ops


def sum(x, axis=None, keepdims=False):
    if axis is None:
        raise NotImplementedError("sum over all axes: only a reduction over one axis is supported")
    if isinstance(x, E._ShapeProbe):
        nd = len(x.shape)
        ax = axis if axis >= 0 else nd + axis
        if not 0 < ax < nd:
            raise ValueError("sum: axis %r out of range for a %d-D tensor" % (axis, nd))
        return E._ShapeProbe(x.shape[:ax] + ((1,) if keepdims else ()) + x.shape[ax + 1:],
                             summed_from=None if keepdims else (x, ax))
    return ops.reduce(x, "sum", axis, keepdims)
