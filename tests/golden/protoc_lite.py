"""A small .proto (proto3) reader: turns the reference's own protocol files into protobuf descriptors at run time.

This image has the `protobuf` runtime but no protoc / grpc_tools, and the reference's plan messages
(ballista/core/proto/{datafusion_common,datafusion,ballista}.proto) are the only authoritative statement of the wire format
a Ballista task's plan bytes use (TaskDefinition.plan, ballista.proto:518-529).  Reading those files -- field numbers, types,
oneofs, enums -- and handing them to google.protobuf's descriptor pool gives the fixture generator real message classes, so
the bytes under tests/golden/proto_plans.json are what a conforming protobuf encoder produces for these schemas, not a
restatement of them.  Supports what the three files use: messages (nested), enums, oneof, repeated / optional, map<,>,
imports, packages, reserved, options (ignored), services (ignored).
"""
import os
import re

from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

_SCALARS = {
    "double": 1, "float": 2, "int64": 3, "uint64": 4, "int32": 5, "fixed64": 6, "fixed32": 7, "bool": 8, "string": 9,
    "bytes": 12, "uint32": 13, "sfixed32": 15, "sfixed64": 16, "sint32": 17, "sint64": 18,
}
_TOK = re.compile(r'"(?:[^"\\]|\\.)*"|[A-Za-z_][A-Za-z0-9_.]*|-?\d+|[{}=;<>,\[\]()]')


def _tokens(text):
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"//[^\n]*", " ", text)
    return _TOK.findall(text)


class _Parser:
    def __init__(self, name, text):
        self.t = _tokens(text)
        self.i = 0
        self.fd = descriptor_pb2.FileDescriptorProto()
        self.fd.name = name
        self.fd.syntax = "proto3"

    def peek(self):
        return self.t[self.i] if self.i < len(self.t) else None

    def next(self):
        tok = self.t[self.i]
        self.i += 1
        return tok

    def expect(self, tok):
        got = self.next()
        assert got == tok, f"{self.fd.name}: expected {tok!r}, got {got!r} near token {self.i}"

    def skip_statement(self):
        depth = 0
        while True:
            tok = self.next()
            if tok == "{":
                depth += 1
            elif tok == "}":
                depth -= 1
                if depth == 0:
                    return
            elif tok == ";" and depth == 0:
                return

    def skip_options(self):
        if self.peek() == "[":
            while self.next() != "]":
                pass

    def parse(self):
        while self.peek() is not None:
            tok = self.next()
            if tok == "syntax":
                self.skip_statement()
            elif tok == "package":
                self.fd.package = self.next()
                self.expect(";")
            elif tok == "import":
                if self.peek() in ("public", "weak"):
                    self.next()
                self.fd.dependency.append(self.next().strip('"'))
                self.expect(";")
            elif tok == "option":
                self.skip_statement()
            elif tok == "message":
                self.message(self.fd.message_type.add())
            elif tok == "enum":
                self.enum(self.fd.enum_type.add())
            elif tok == "service":
                self.skip_statement()
            elif tok == ";":
                pass
            else:
                raise AssertionError(f"{self.fd.name}: unexpected top-level token {tok!r}")
        return self.fd

    def enum(self, ed):
        ed.name = self.next()
        self.expect("{")
        while self.peek() != "}":
            tok = self.next()
            if tok in ("option", "reserved"):
                self.i -= 1
                self.next()
                while self.next() != ";":
                    pass
                continue
            v = ed.value.add()
            v.name = tok
            self.expect("=")
            v.number = int(self.next())
            self.skip_options()
            self.expect(";")
        self.expect("}")

    def field(self, md, label_tok, oneof_index=None):
        f = md.field.add()
        typ = label_tok
        f.label = 1
        if label_tok == "repeated":
            f.label = 3
            typ = self.next()
        elif label_tok == "optional":
            typ = self.next()
            f.proto3_optional = True
        if typ == "map":
            self.expect("<")
            kt = self.next()
            self.expect(",")
            vt = self.next()
            self.expect(">")
            f.name = self.next()
            entry = md.nested_type.add()
            entry.name = "".join(p.capitalize() for p in f.name.split("_")) + "Entry"
            entry.options.map_entry = True
            for nm, num, t in (("key", 1, kt), ("value", 2, vt)):
                ef = entry.field.add()
                ef.name, ef.number, ef.label = nm, num, 1
                self.set_type(ef, t)
            f.label = 3
            f.type = 11
            f.type_name = entry.name
            self.pending_maps.append((f, md))
        else:
            self.set_type(f, typ)
            f.name = self.next()
        self.expect("=")
        f.number = int(self.next())
        self.skip_options()
        self.expect(";")
        if oneof_index is not None:
            f.oneof_index = oneof_index
        return f

    def set_type(self, f, typ):
        if typ in _SCALARS:
            f.type = _SCALARS[typ]
        else:
            f.type = 11          # message or enum: resolved after all files are read
            f.type_name = typ

    pending_maps = []

    def message(self, md):
        md.name = self.next()
        self.expect("{")
        synthetic = []
        while self.peek() != "}":
            tok = self.next()
            if tok == "message":
                self.message(md.nested_type.add())
            elif tok == "enum":
                self.enum(md.enum_type.add())
            elif tok == "oneof":
                od = md.oneof_decl.add()
                od.name = self.next()
                idx = len(md.oneof_decl) - 1
                self.expect("{")
                while self.peek() != "}":
                    t2 = self.next()
                    if t2 == "option":
                        while self.next() != ";":
                            pass
                        continue
                    self.field(md, t2, idx)
                self.expect("}")
            elif tok in ("reserved", "option", "extensions"):
                while self.next() != ";":
                    pass
            elif tok == ";":
                pass
            else:
                f = self.field(md, tok)
                if f.proto3_optional:
                    synthetic.append(f)
        self.expect("}")
        for f in synthetic:   # proto3 optional = a synthetic one-field oneof, declared after the real ones
            od = md.oneof_decl.add()
            od.name = "_" + f.name
            f.oneof_index = len(md.oneof_decl) - 1


def _index(fd, names, prefix, container, kind_of):
    for m in container.message_type if hasattr(container, "message_type") else container.nested_type:
        full = prefix + "." + m.name
        kind_of[full] = 11
        _index(fd, names, full, m, kind_of)
    for e in container.enum_type:
        kind_of[prefix + "." + e.name] = 14


def _resolve(md, scope, kind_of, package):
    here = scope + "." + md.name
    for f in md.field:
        if f.type == 11 and f.type_name and not f.type_name.startswith("."):
            name = f.type_name
            # innermost scope outwards, then the name as a fully qualified one
            parts = here.split(".")
            found = None
            for k in range(len(parts), 0, -1):
                cand = ".".join(parts[:k]) + "." + name
                if cand in kind_of:
                    found = cand
                    break
            if found is None and "." + name in kind_of:
                found = "." + name
            assert found, f"cannot resolve type {name} in {here}"
            f.type_name = found
            f.type = kind_of[found]
    for n in md.nested_type:
        _resolve(n, here, kind_of, package)


def load(paths):
    """paths: [(import name, file path)] in dependency order -> {full message name: class}, pool."""
    fds = []
    for name, path in paths:
        with open(path) as fh:
            fds.append(_Parser(name, fh.read()).parse())
    kind_of = {}
    for fd in fds:
        _index(fd, None, "." + fd.package, fd, kind_of)
    for fd in fds:
        for m in fd.message_type:
            _resolve(m, "." + fd.package, kind_of, fd.package)
    pool = descriptor_pool.DescriptorPool()
    for fd in fds:
        pool.Add(fd)
    classes = {}
    for full in kind_of:
        if kind_of[full] == 11:
            try:
                classes[full[1:]] = message_factory.GetMessageClass(pool.FindMessageTypeByName(full[1:]))
            except Exception:   # map entries have no public class
                pass
    return classes, pool


def load_ballista(proto_dir=None):
    """The message classes of a datafusion-ballista checkout's ballista/core/proto (default: $BALLISTA_SRC/ballista/core/proto)."""
    if proto_dir is None:
        if not os.environ.get("BALLISTA_SRC"):
            raise RuntimeError("set BALLISTA_SRC to a datafusion-ballista checkout")
        proto_dir = os.path.join(os.environ["BALLISTA_SRC"], "ballista", "core", "proto")
    return load([("datafusion_common.proto", proto_dir + "/datafusion_common.proto"),
                 ("datafusion.proto", proto_dir + "/datafusion.proto"),
                 ("ballista.proto", proto_dir + "/ballista.proto")])
