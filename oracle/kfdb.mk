# oracle/kfdb.mk -- builds the key-frame database oracle (test infrastructure; never linked into the product) from the
# reference's own sources, reusing the flags and objects of oracle/Makefile.  Built only where $(REF) exists; the GPU
# box uses the prebuilt files (oracle/_ref/ is git-ignored).
#   _ref/libkfdbsrc.so   src/KeyFrameDatabase.cc, unmodified, + the objects of target `ref` minus its harness (which
#                        stubs KeyFrameDatabase::erase) + kfdb_harness.cpp
#   _ref/libkfdbshim.so  src/Frame.cc, KeyFrame.cc, MapPoint.cc, Map.cc, unmodified, against the shims as in target
#                        `shim`, plus shim/KeyFrameDatabase.h force-included: include/KeyFrame.h includes its sibling
#                        include/KeyFrameDatabase.h by quote, which finds the sibling before any -I directory, so the
#                        shim has to own the KEYFRAMEDATABASE_H guard first.  The harness includes it ahead of KeyFrame.h.
include Makefile
.DEFAULT_GOAL := kfdb
kfdb: $(if $(wildcard $(REF)/src/KeyFrameDatabase.cc),_ref/libkfdbsrc.so _ref/libkfdbshim.so)
_ref/kfdb_harness.o: kfdb_harness.cpp $(wildcard standin/*.hpp standin/*.h standin/Thirdparty/DBoW2/DBoW2/*.h) ../include/b200orb.h
	@mkdir -p _ref
	$(CXX) $(REFFLAGS) -c $< -o $@
_ref/libkfdbsrc.so: $(REFSRCS:%=_ref/%.o) _ref/KeyFrameDatabase.o _ref/kfdb_harness.o
	$(CXX) -shared -pthread -o $@ $^ -Wl,--no-undefined -Wl,-Bsymbolic
KFDBSHIMFLAGS := $(SHIMFLAGS) -include $(SHIM)/KeyFrameDatabase.h
_ref/kfdbshim_%.o: $(REF)/src/%.cc $(wildcard $(SHIM)/*.h standin/*.hpp) ../include/b200orb.h
	@mkdir -p _ref
	$(CXX) $(KFDBSHIMFLAGS) -c $< -o $@
_ref/kfdbshim_harness.o: kfdb_harness.cpp $(wildcard $(SHIM)/*.h standin/*.hpp) ../include/b200orb.h
	@mkdir -p _ref
	$(CXX) $(SHIMFLAGS) -c $< -o $@
_ref/libkfdbshim.so: $(SHIMSRCS:%=_ref/kfdbshim_%.o) _ref/kfdbshim_harness.o $(PKG)/libb200orb.so
	$(CXX) -shared -pthread -o $@ $(SHIMSRCS:%=_ref/kfdbshim_%.o) _ref/kfdbshim_harness.o -L$(PKG) -lb200orb \
	    -Wl,-rpath,'$$ORIGIN/../../orb_slam2_ssd_semantic_b200' -Wl,--no-undefined -Wl,-Bsymbolic
