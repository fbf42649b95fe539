# oracle/fps_ref.mk -- builds the reference's farthest point sampling as a checker. TEST INFRASTRUCTURE ONLY.
#
#   make -C oracle -f fps_ref.mk REF=<reference checkout>   -> _ref/libfps_ref.so
#
# compiled from the UNMODIFIED utils/dataset_tools/fps/src/farthest_point_sampling.cpp where it lies under $(REF),
# with the reference's own flags (fps/setup.py:3; no -march, so no FMA).  Its extern "C" functions are called
# through ctypes (oracle/fps_oracle.py).  The output is git-ignored like the rest of _ref/.
CXX := /usr/bin/g++
ifndef REF
$(error REF=<path of the reference checkout> is required)
endif
FPS := $(REF)/ffb6d/utils/dataset_tools/fps/src

_ref/libfps_ref.so: $(FPS)/farthest_point_sampling.cpp
	mkdir -p _ref
	$(CXX) -O2 -std=c++11 -fopenmp -fPIC -shared -o $@ $(FPS)/farthest_point_sampling.cpp
