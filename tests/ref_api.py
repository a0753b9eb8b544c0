"""The reference's own sources (oracle/_ref/libvxref.so, built by oracle/Makefile from the reference sources at VXS_REFERENCE_SRC (see oracle/Makefile) against the stand-in headers) behind the
same Python wrappers as the hand-written oracle: this module is tests/oracle_api.py executed a second time with BACKEND = "ref"."""
import os as _os

BACKEND = "ref"
exec(compile(open(_os.path.join(_os.path.dirname(_os.path.abspath(__file__)), "oracle_api.py")).read(), "oracle_api.py[ref]", "exec"))
