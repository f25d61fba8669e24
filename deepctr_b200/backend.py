"""The part of ``tf.keras.backend`` (and of ``tensorflow``) the reference's builders call inside their ``Lambda``
layers: ONN's ``K.sum(element_wise_prod, axis=-1)`` (deepctr/models/onn.py:95-96) and CCPM's
``tf.expand_dims(x, axis=3)`` (deepctr/models/ccpm.py:59-60).  A builder imported as a drop-in reaches them as
``tensorflow.keras.backend`` and ``tensorflow``.  Each function works on a runtime Var (on the package's kernels, through ``ops``)
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


def expand_dims(x, axis=-1):
    """A unit axis inserted at ``axis`` (not the batch axis): a zero-copy view, a window of the gather buffer
    stays one."""
    nd = len(x.shape) + 1
    ax = axis if axis >= 0 else nd + axis
    if not 0 < ax < nd:
        raise ValueError("expand_dims: axis %r out of range for a %d-D result (the batch axis is not supported)"
                         % (axis, nd))
    shape = tuple(x.shape[:ax]) + (1,) + tuple(x.shape[ax:])
    if isinstance(x, E._ShapeProbe):
        return E._ShapeProbe(shape)
    return ops.reshape(x, (None,) + shape[1:])
