# oracle/_ref/libvlcal_bag_ref.so: the reference's OWN per-scan code of `preprocess` -- extract_raw_points, TimeKeeper
# and the static integrator -- compiled where it lies (test infrastructure).
#   make -C oracle -f bag_ref.mk ref REF=<reference checkout>      (or VLCAL_REFERENCE in the environment)
# The stand-ins of ref_standin_bag/ come first on the include path (they shadow the reference's frame headers and
# the viewer); ref_standin/ supplies boost/format.hpp.  Flags: the reference's RelWithDebInfo (-O2 -g -std=c++17).
REF ?= $(VLCAL_REFERENCE)
CXX_REF = /usr/bin/g++
BAG_REF_SRCS = $(REF)/src/vlcal/common/time_keeper.cpp $(REF)/src/vlcal/preprocess/static_point_cloud_integrator.cpp
BAG_REF_FLAGS = -O2 -g -std=c++17 -fPIC -ffp-contract=off -w -Iref_standin_bag -Iref_standin -I$(REF)/include

ref: _ref/libvlcal_bag_ref.so
$(if $(filter ref,$(MAKECMDGOALS)),$(if $(REF),,$(error set REF=<reference checkout>)))

_ref/libvlcal_bag_ref.so: bag_ref_shim.cpp $(shell find ref_standin_bag -type f)
	mkdir -p _ref
	$(CXX_REF) $(BAG_REF_FLAGS) -shared -Wl,--no-undefined -o $@ bag_ref_shim.cpp $(BAG_REF_SRCS)
