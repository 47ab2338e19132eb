# oracle/homo.mk -- the perfect tree's point-pair SearchByProjection (TrackHomo) oracle and the perfect tree's sources
# against the shims (test infrastructure; never linked into the product), reusing the flags and objects of
# oracle/Makefile.  Built only where $(REF)/perfect exists; the GPU box uses the prebuilt files (oracle/_ref/ is
# git-ignored).
#   _ref/libhomoref.so      the objects of target `perfect` (perfect/src/Frame.cc, KeyFrame.cc, MapPoint.cc, Map.cc,
#                           ORBextractor.cc, ORBmatcher.cc, unmodified) + homo_harness.cpp (exports refperfect_homo_*)
#   _ref/libshimperfect.so  perfect/src/Frame.cc (plain + masked RGB-D constructors), KeyFrame.cc, MapPoint.cc, Map.cc,
#                           unmodified, against the shims with the include path and the three force-includes that
#                           INTEGRATION.md prescribes (shim/ORBextractor.h, shim/ORBVocabulary.h, shim/KeyFrameDatabase.h:
#                           perfect/include/KeyFrame.h also includes its sibling KeyFrameDatabase.h by quote), plus
#                           homo_harness.cpp (exports shimperfect_homo_*), linked against libb200orb.so.  Like target
#                           `perfect`, the build adds what only the stand-ins need: <fstream> and standin/Converter.h
#                           force-included (perfect/include/Map.h includes Converter.h, which needs Eigen + g2o).
include Makefile
.DEFAULT_GOAL := homo
homo: $(if $(wildcard $(REF)/perfect/src/Frame.cc),_ref/libhomoref.so _ref/libshimperfect.so)
_ref/homoref_harness.o: homo_harness.cpp $(wildcard standin/*.hpp standin/*.h) ../include/b200orb.h
	@mkdir -p _ref
	$(CXX) $(PERFFLAGS) -c $< -o $@
_ref/libhomoref.so: $(PERFSRCS:%=_ref/perfect_%.o) _ref/homoref_harness.o
	$(CXX) -shared -pthread -o $@ $^ -Wl,--no-undefined -Wl,-Bsymbolic
SHIMPERFFLAGS := -O2 -march=x86-64-v3 -ffp-contract=off -std=c++14 -fPIC -w -pthread -DREFSRC_SHIM -include fstream \
                 -include standin/Converter.h -include $(SHIM)/ORBextractor.h -include $(SHIM)/ORBVocabulary.h \
                 -include $(SHIM)/KeyFrameDatabase.h -I$(SHIM) -I../include -Istandin -I$(REF)/perfect/include -I$(REF)/perfect
_ref/shimperfect_%.o: $(REF)/perfect/src/%.cc $(wildcard $(SHIM)/*.h standin/*.hpp standin/*.h) ../include/b200orb.h
	@mkdir -p _ref
	$(CXX) $(SHIMPERFFLAGS) -c $< -o $@
_ref/shimperfect_harness.o: homo_harness.cpp $(wildcard $(SHIM)/*.h standin/*.hpp standin/*.h) ../include/b200orb.h
	@mkdir -p _ref
	$(CXX) $(SHIMPERFFLAGS) -c $< -o $@
_ref/libshimperfect.so: $(SHIMSRCS:%=_ref/shimperfect_%.o) _ref/shimperfect_harness.o $(PKG)/libb200orb.so
	$(CXX) -shared -pthread -o $@ $(SHIMSRCS:%=_ref/shimperfect_%.o) _ref/shimperfect_harness.o -L$(PKG) -lb200orb \
	    -Wl,-rpath,'$$ORIGIN/../../orb_slam2_ssd_semantic_b200' -Wl,--no-undefined -Wl,-Bsymbolic
