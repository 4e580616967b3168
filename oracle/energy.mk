# oracle/energy.mk -- builds the reference CRF's klDivergence (TEST INFRASTRUCTURE, not product code).
#
#   _ref/libdensecrf_energy_ref.so: the reference's OWN CRF sources (the list oracle/grad.mk compiles), unmodified and
#                                   in place, against oracle/eigen_shim, with a driver around DenseCRF::klDivergence
#                                   (ref_densecrf_energy_driver.cpp); only when $(REF) exists.  Only
#                                   tests/golden/make_crf_energy_golden.py uses it: the tests read the frozen golden
#
# Flags as in oracle/Makefile (the reference build's -O2, no FMA contraction, no -march).
REF ?= /root/reference
CXX ?= g++
CXXFLAGS = -O2 -ffp-contract=off -fPIC -shared -w

ref:
	@if [ -f $(REF)/CRF/src/densecrf.cpp ]; then \
	  mkdir -p _ref && \
	  $(CXX) $(CXXFLAGS) -Ieigen_shim -I$(REF)/CRF/include -o _ref/libdensecrf_energy_ref.so \
	      $(REF)/CRF/src/densecrf.cpp $(REF)/CRF/src/labelcompatibility.cpp $(REF)/CRF/src/pairwise.cpp \
	      $(REF)/CRF/src/permutohedral.cpp $(REF)/CRF/src/unary.cpp $(REF)/CRF/src/util.cpp \
	      ref_densecrf_energy_driver.cpp && \
	  echo "built _ref/libdensecrf_energy_ref.so from $(REF)/CRF/src/*.cpp"; \
	else echo "reference not present: keeping prebuilt _ref/ (if any)"; fi

clean:
	rm -f _ref/libdensecrf_energy_ref.so
.PHONY: ref clean
