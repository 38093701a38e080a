# oracle/continuous.mk -- TEST INFRASTRUCTURE.  Builds the scalar restatement of the continuous-frequency site model
# (libcontinuous_oracle.so), with the flags of oracle/allele_groups.mk.
CXX ?= g++
CXXFLAGS = -std=gnu++17 -O3 -fomit-frame-pointer -ffp-contract=off -fPIC -Wall -I../include -I../strelka_b200/csrc

libcontinuous_oracle.so: continuous_oracle.cpp ../include/strelka_b200.h ../strelka_b200/csrc/k2c_core.cuh ../strelka_b200/csrc/sx_libm_mirror_d.h
	$(CXX) $(CXXFLAGS) -shared -o $@ continuous_oracle.cpp

.PHONY: clean
clean:
	rm -f libcontinuous_oracle.so
