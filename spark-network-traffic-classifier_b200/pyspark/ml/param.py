"""Minimal pyspark.ml.param: keyword params with defaults, setX()/getX() accessors (setters return self), and Param objects
(`est.numTrees`) for param maps keyed the pyspark way (ParamGridBuilder, fit(df, {est.maxDepth: 8}))."""
import uuid


class Param:
    """a declared param of one Params instance; equal when the owner's uid and the name are equal (as in pyspark)."""

    def __init__(self, parent, name, doc=""):
        self.parent, self.name, self.doc = parent.uid, name, doc

    def __eq__(self, other):
        return isinstance(other, Param) and self.parent == other.parent and self.name == other.name

    def __hash__(self):
        return hash((self.parent, self.name))

    def __repr__(self):
        return "%s__%s" % (self.parent, self.name)

    __str__ = __repr__


class Params:
    _defaults = {}

    def __init__(self, **kwargs):
        self._paramMap = {}
        self._set(**kwargs)

    @property
    def uid(self):
        """a stable identity that copies share (pyspark: type name + random suffix)."""
        u = self.__dict__.get("_uid")
        if u is None:
            u = self.__dict__["_uid"] = "%s_%s" % (type(self).__name__, uuid.uuid4().hex[-12:])
        return u

    def _set(self, **kwargs):
        for k, v in kwargs.items():
            if k not in self._all_defaults():
                raise TypeError("%s got an unexpected keyword argument %r" % (type(self).__name__, k))
            if v is not None:
                self._paramMap[k] = v
        return self

    @classmethod
    def _all_defaults(cls):
        d = {}
        for klass in reversed(cls.__mro__):
            d.update(klass.__dict__.get("_defaults", {}))
        return d

    def _param_name(self, param):
        """a name, or a Param of this instance -> the name"""
        if isinstance(param, Param):
            if param.parent != self.uid:
                raise ValueError("Param %r does not belong to %s." % (param, self.uid))
            return param.name
        return param

    def _named(self, extra):
        """a param map keyed by names and / or Params -> {name: value}; Params of other instances are skipped (pyspark's
        copy applies only the params an instance owns, so one map can address several pipeline stages)."""
        return {(k.name if isinstance(k, Param) else k): v for k, v in extra.items()
                if not isinstance(k, Param) or k.parent == self.uid}

    def hasParam(self, name):
        return name in self._all_defaults()

    def getOrDefault(self, name):
        name = self._param_name(name)
        if name in self._paramMap:
            return self._paramMap[name]
        return self._all_defaults()[name]

    def isSet(self, name):
        return self._param_name(name) in self._paramMap

    def setParams(self, **kwargs):
        return self._set(**kwargs)

    def copy(self, extra=None):
        import copy as _copy
        c = _copy.copy(self)
        c._paramMap = dict(self._paramMap)
        if extra:
            c._set(**self._named(extra))
        return c

    def explainParams(self):
        return "\n".join("%s: (default: %r%s)" % (k, v, ", current: %r" % self._paramMap[k] if k in self._paramMap else "")
                         for k, v in sorted(self._all_defaults().items()))

    def __getattr__(self, name):
        # setFoo(value) / getFoo() for every declared param; the bare name is its Param object
        if name.startswith("set") and len(name) > 3:
            p = name[3].lower() + name[4:]
            if p in self._all_defaults():
                return lambda value: self._set(**{p: value})
        if name.startswith("get") and len(name) > 3:
            p = name[3].lower() + name[4:]
            if p in self._all_defaults():
                return lambda: self.getOrDefault(p)
        if not name.startswith("_") and name in self._all_defaults():
            return Param(self, name)
        raise AttributeError("%s has no attribute %r" % (type(self).__name__, name))
