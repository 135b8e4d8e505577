// Frame.h -- stand-in for the reference's include/Frame.h: refshim/ref_skeleton.h (pre-included) defines FRAME_H and the skeleton
// Frame the host units are compiled against, so the real header's body would be skipped as well.
#ifndef FRAME_H
#define FRAME_H
#endif
