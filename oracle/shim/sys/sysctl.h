/* Empty stand-in for <sys/sysctl.h>, which current glibc no longer ships.  Only the unmodified OpenCV 2 sources of the
 * reference sgbm binary include it (3rdparty/sgbm/parallel.cpp); nothing of it is used on Linux. */
