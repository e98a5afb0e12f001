"""
Utilities used by the FFTPower path (subset of nbodykit/utils.py):
JSON (de)serialisation compatible with the reference's result files (utils.py:381-489),
`attrs_to_dict` (:372-379), `timer` (:491-511), `get_data_bounds` (:23-82).
"""
import json

import numpy


def attrs_to_dict(obj, prefix):
    if not hasattr(obj, 'attrs'):
        return {}
    return {prefix + k: v for k, v in obj.attrs.items()}


class JSONEncoder(json.JSONEncoder):
    """numpy arrays -> {'__dtype__', '__shape__', '__data__'}; complex -> {'__complex__': [re, im]};
    numpy scalars -> python scalars; a Cosmology -> {'__cosmo__': pars}.  Same wire format as the reference
    (utils.py:381-433)."""

    def default(self, obj):
        from .cosmology import Cosmology
        if isinstance(obj, Cosmology):
            return {'__cosmo__': obj.pars.copy()}
        if isinstance(obj, (complex, numpy.complexfloating)):
            return {'__complex__': [float(obj.real), float(obj.imag)]}
        if isinstance(obj, numpy.ndarray):
            dt = obj.dtype
            return {'__dtype__': dt.str if dt.names is None else dt.descr,
                    '__shape__': obj.shape,
                    '__data__': obj.tolist()}
        if isinstance(obj, numpy.floating):
            return float(obj)
        if isinstance(obj, numpy.integer):
            return int(obj)
        if isinstance(obj, numpy.bool_):
            return bool(obj)
        return json.JSONEncoder.default(self, obj)


class JSONDecoder(json.JSONDecoder):
    """inverse of JSONEncoder (utils.py:435-489)"""

    @staticmethod
    def hook(value):
        if '__dtype__' in value:
            dtype = value['__dtype__']
            shape = value['__shape__']
            data = value['__data__']
            if isinstance(dtype, list):      # structured: innermost records must be tuples
                dtype = [tuple([str(f[0]), str(f[1])] + list(f[2:])) for f in dtype]
                nfield = len(dtype)

                def records(d, depth):
                    if depth > 0:
                        return [records(x, depth - 1) for x in d]
                    assert len(d) == nfield
                    return tuple(d)
                data = records(data, len(shape))
            return numpy.array(data, dtype=dtype)
        if '__complex__' in value:
            re, im = value['__complex__']
            return re + 1j * im
        if '__cosmo__' in value:
            from .cosmology import Cosmology
            return Cosmology.from_dict(value['__cosmo__'])
        return value

    def __init__(self, *args, **kwargs):
        kwargs['object_hook'] = JSONDecoder.hook
        json.JSONDecoder.__init__(self, *args, **kwargs)


def timer(start, end):
    """elapsed time as hours:minutes:seconds"""
    hours, rem = divmod(end - start, 3600)
    minutes, seconds = divmod(rem, 60)
    return "{:0>2}:{:0>2}:{:05.2f}".format(int(hours), int(minutes), seconds)


def get_data_bounds(data, comm, selection=None):
    """global (min, max) along axis 0 of a (n, ...) column over all ranks (utils.py:23-82);
    `data` may be a numpy array or a torch tensor (device reductions, tiny all-gather)"""
    import torch
    t = data if isinstance(data, torch.Tensor) else torch.as_tensor(numpy.asarray(data))
    if selection is not None:
        s = selection if isinstance(selection, torch.Tensor) else torch.as_tensor(numpy.asarray(selection))
        t = t[s.to(t.device).bool()]
    shape = tuple(t.shape[1:])
    if t.shape[0] == 0:
        dmin = numpy.full(shape, numpy.inf)
        dmax = numpy.full(shape, -numpy.inf)
    else:
        dmin = t.min(dim=0).values.double().cpu().numpy()
        dmax = t.max(dim=0).values.double().cpu().numpy()
    dmin = numpy.min(numpy.asarray(comm.allgather(dmin)), axis=0)
    dmax = numpy.max(numpy.asarray(comm.allgather(dmax)), axis=0)
    return dmin, dmax
