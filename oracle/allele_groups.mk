# oracle/allele_groups.mk -- TEST INFRASTRUCTURE.  Builds the scalar restatement of the K6 -> K5 link (liballele_groups_oracle.so), with the
# flags of oracle/indel_reads.mk.
CXX ?= g++
CXXFLAGS = -std=gnu++14 -O3 -fomit-frame-pointer -ffp-contract=off -fPIC -Wall -I../include

liballele_groups_oracle.so: allele_groups_oracle.cpp ../include/strelka_b200.h
	$(CXX) $(CXXFLAGS) -shared -o $@ allele_groups_oracle.cpp

.PHONY: clean
clean:
	rm -f liballele_groups_oracle.so
