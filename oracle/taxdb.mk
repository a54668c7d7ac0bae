# oracle/taxdb.mk -- builds _ref/taxdb_ref: the reference's OWN taxdb.hpp (header-only), compiled in place from $(REF)
# behind the command-line front end ref_taxdb.cpp (nothing is copied).  Test infrastructure, like _ref/kseq_dump in
# oracle/Makefile; only built where $(REF) exists, the prebuilt tool travels with the tree.
REF ?= /root/reference/src/mash
CXX ?= g++

all:
	@if [ -d $(REF) ]; then $(MAKE) -f taxdb.mk _ref/taxdb_ref; else echo "reference sources absent: keeping prebuilt oracle/_ref (if any)"; fi

_ref/taxdb_ref: ref_taxdb.cpp $(REF)/taxdb.hpp
	mkdir -p _ref
	$(CXX) -O2 -std=c++14 -I$(REF) -o $@ ref_taxdb.cpp

.PHONY: all
