"""Without a GPU: the packed string columns evg_intern_batch and evg_upload_strings take, and their argument guard."""
import ctypes as C

import numpy as np

from evergreen_b200 import _lib as L
from evergreen_b200 import soa as S


def test_string_cols_pack_bytes_and_text_alike():
    sc = S.StringCols.pack(np.array([0, 2, 3]), ["a", b"\x00\xff", "é"], ["v", "v", ""], ["", "g", "g"], [0, 1, 1],
                           np.array([0, 1, 1, 2]), [b"a", "é"])
    assert (sc.n_tasks, sc.n_distros) == (3, 2)
    assert bytes(sc.id[0]) == b"a\x00\xff\xc3\xa9" and sc.id[1].tolist() == [0, 1, 3, 5]
    st = sc.struct()
    assert st.n_tasks == 3 and st.n_distros == 2 and st.dep_id.off == L.ptr(sc.dep_id[1])
    out, outs = sc.intern_out()
    assert L.load().evg_intern_columns(C.byref(st), C.byref(outs), 1) == L.EVG_OK
    out = sc.trim(out)
    assert out["group_id"].tolist() == [-1, 0, 0] and out["dep_idx"].tolist() == [0, 0]
    assert out["group_first"].tolist() == [1, 2] and out["n_versions"].tolist() == [1, 1]


def test_device_interning_fails_a_null_context_before_reading_its_arguments():
    lib = L.load()
    sc = S.StringCols.pack(np.array([0, 1]), ["t"], ["v"], [""], [0], np.array([0, 0]), [])
    out, outs = sc.intern_out()
    assert lib.evg_intern_batch(None, C.byref(sc.struct()), C.byref(outs)) == L.EVG_ERR_INVALID
    assert L.last_error() == "evg_intern_batch: null context"
    assert lib.evg_upload_strings(None, None, C.byref(sc.struct()), None, None, None, None, C.byref(outs)) == L.EVG_ERR_INVALID
    assert L.last_error() == "evg_upload_strings: null context"
