# oracle/sem.mk -- builds oracle/libsem_oracle.so, the restatement of the semantic object clusters (sem_ref.cpp), with
# the flags of oracle/Makefile.  Test infrastructure; never linked into the product.
include Makefile
.DEFAULT_GOAL := sem
sem: libsem_oracle.so
libsem_oracle.so: sem_ref.cpp ../include/b200orb.h
	$(CXX) $(CXXFLAGS) -shared -o $@ sem_ref.cpp
