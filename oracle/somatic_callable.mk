# oracle/somatic_callable.mk -- TEST INFRASTRUCTURE.  Builds the callable-mode restatement of the somatic SNV model
# (libsomatic_callable_oracle.so) on top of liboracle.so (oracle/Makefile), with its flags.
CXX ?= g++
CXXFLAGS = -std=gnu++14 -O3 -fomit-frame-pointer -ffp-contract=off -fPIC -Wall -I../include -I../strelka_b200/csrc

libsomatic_callable_oracle.so: somatic_callable_oracle.cpp liboracle.so strelka_oracle.h ../include/strelka_b200.h ../strelka_b200/csrc/sx_libm_mirror_d.h
	$(CXX) $(CXXFLAGS) -shared -o $@ somatic_callable_oracle.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'

.PHONY: clean
clean:
	rm -f libsomatic_callable_oracle.so
