# oracle/somatic_indel.mk -- TEST INFRASTRUCTURE.  Builds the scalar restatement of the somatic indel model (libsindel_oracle.so),
# with the flags of oracle/Makefile's liboracle.so.
CXX ?= g++
CXXFLAGS = -std=gnu++14 -O3 -fomit-frame-pointer -ffp-contract=off -fPIC -Wall -I../include

libsindel_oracle.so: somatic_indel_oracle.cpp ../include/strelka_b200.h ../strelka_b200/csrc/sx_libm_mirror_d.h ../strelka_b200/csrc/sx_libm_mirror_d_tables.inc
	$(CXX) $(CXXFLAGS) -shared -o $@ somatic_indel_oracle.cpp

.PHONY: clean
clean:
	rm -f libsindel_oracle.so
