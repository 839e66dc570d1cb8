"""The reference's SolverState / BlobProto / BlobShape messages (src/caffe/proto/caffe.proto:15-35,303-308, same field numbers), built
with google.protobuf at run time: an encoder and decoder of .solverstate files that shares no code with host/proto_wire.cpp."""
import numpy as np
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

FLOAT = 1        # caffe.proto Type.FLOAT, the raw_data_type NVCaffe writes


def _build():
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="caffe_state_test.proto", package="caffe_state_test", syntax="proto2")

    def msg(name, fields):
        m = fd.message_type.add(name=name)
        for fname, num, ftype, label, tname, packed in fields:
            f = m.field.add(name=fname, number=num, type=ftype, label=label)
            if tname:
                f.type_name = ".caffe_state_test." + tname
            if packed:
                f.options.packed = True

    opt, rep = F.LABEL_OPTIONAL, F.LABEL_REPEATED
    msg("BlobShape", [("dim", 1, F.TYPE_INT64, rep, None, True)])
    msg("BlobProto", [("shape", 7, F.TYPE_MESSAGE, opt, "BlobShape", False), ("data", 5, F.TYPE_FLOAT, rep, None, True),
                      ("raw_data_type", 10, F.TYPE_INT32, opt, None, False), ("raw_data", 12, F.TYPE_BYTES, opt, None, False)])
    msg("SolverState", [("iter", 1, F.TYPE_INT32, opt, None, False), ("learned_net", 2, F.TYPE_STRING, opt, None, False),
                        ("history", 3, F.TYPE_MESSAGE, rep, "BlobProto", False), ("current_step", 4, F.TYPE_INT32, opt, None, False)])
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    get = message_factory.GetMessageClass
    return get(pool.FindMessageTypeByName("caffe_state_test.SolverState"))


SolverState = _build()


def read_state(path):
    """(iter, current_step, learned_net, [history blobs as flat float32 arrays])."""
    st = SolverState()
    with open(path, "rb") as f:
        st.ParseFromString(f.read())
    blobs = []
    for b in st.history:
        if b.HasField("raw_data"):
            assert b.raw_data_type == FLOAT
            blobs.append(np.frombuffer(b.raw_data, np.float32).copy())
        else:
            blobs.append(np.array(b.data, np.float32))
    return st.iter, st.current_step, st.learned_net, blobs


def write_state(path, it, learned_net, history, shapes, current_step=0):
    """A .solverstate as the reference's BVLC-format writer lays it out (packed `data`, `shape`)."""
    st = SolverState(iter=it, current_step=current_step, learned_net=learned_net)
    for h, shp in zip(history, shapes):
        b = st.history.add()
        b.shape.dim.extend(int(d) for d in shp)
        b.data.extend(np.asarray(h, np.float32).reshape(-1).tolist())
    with open(path, "wb") as f:
        f.write(st.SerializeToString())
